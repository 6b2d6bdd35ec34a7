"""sedumi_b200 -- H100-native normal-equations hot path behind SeDuMi's MEX boundary."""
__version__ = "0.1.0"
