"""Achieved HBM bandwidth of the Lorentz stream kernels (qblkmul, ddot, quadadd) at a size that does not fit
in L2: the HBM-bound rows of SURVEY 8d measured against a measured copy bandwidth (MEASURED_PEAKS.json: hbm_gbs) or else the H100 data sheet."""
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sedumi_b200 import device as sbdev  # noqa: E402

L = sbdev.lib()
sbdev.check(L.sb200_init(C.c_int(0)), "init")
dev = torch.device("cuda", 0)
stream = torch.cuda.ExternalStream(L.sb200_stream(), device=dev)
I64 = C.c_int64
p = lambda t: C.c_void_p(t.data_ptr())
peak, peak_source = 3350.0, "H100 SXM data sheet (HBM3, 3.35 TB/s)"
try:
    measured = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))).get("hbm_gbs")
    if measured:
        peak, peak_source = measured, "MEASURED_PEAKS.json hbm_gbs"
except (OSError, ValueError):
    pass
N, cone = 1 << 26, 64
nblk = N // cone
with torch.cuda.stream(stream):
    bs = torch.arange(0, N + 1, cone, dtype=torch.int64, device=dev)
    d = torch.randn(N, dtype=torch.float64, device=dev)
    x = torch.randn(N, dtype=torch.float64, device=dev)
    y = torch.empty(N, dtype=torch.float64, device=dev)
    lo = torch.randn(N, dtype=torch.float64, device=dev) * 1e-17
    mu = torch.randn(nblk, dtype=torch.float64, device=dev)
    dd = torch.empty(nblk, dtype=torch.float64, device=dev)
    zh = torch.empty(N, dtype=torch.float64, device=dev)
    zl = torch.empty(N, dtype=torch.float64, device=dev)
    cases = {
        "qblkmul": (lambda: L.sb200_qblkmul_dev(I64(nblk), p(bs), I64(N), p(mu), p(d), p(y)), 16.0 * N + 8.0 * nblk),
        "ddot (dense)": (lambda: L.sb200_ddot_dense_dev(I64(nblk), p(bs), p(d), p(x), I64(N), I64(1), p(dd)), 16.0 * N + 8.0 * nblk),
        "quadadd": (lambda: L.sb200_quadadd_dev(I64(N), p(x), p(lo), p(d), p(zh), p(zl)), 40.0 * N),
    }
    out = {}
    for name, (fn, nbytes) in cases.items():
        for _ in range(3):
            sbdev.check(fn(), name)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(10):
            sbdev.check(fn(), name)
        e1.record(stream)
        stream.synchronize()
        ms = e0.elapsed_time(e1) / 10
        gbs = nbytes / (ms * 1e-3) / 1e9
        out[name] = {"ms": ms, "GB/s": gbs, "frac_of_hbm_peak": gbs / peak, "peak_source": peak_source}
        print(f"{name:14s} N=2^26 doubles  {ms:7.3f} ms  {gbs:8.1f} GB/s  = {100 * gbs / peak:5.1f} % of {peak:.0f} GB/s")
print(json.dumps(out))
