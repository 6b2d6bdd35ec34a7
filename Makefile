# Top-level build: libmxshim.so, libsedumi_b200.so (sm_90a CUDA, H100) and the MEX stubs.
# `make oracle` additionally builds the reference MEX targets into oracle/_ref (needs a
# checkout of the reference, REF=<dir>; test infrastructure only).
NVCC     ?= /usr/local/cuda/bin/nvcc
CXX      ?= g++
ARCH     := -gencode arch=compute_90a,code=sm_90a
NVFLAGS  := $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Iinclude -Isedumi_b200/csrc --fmad=true $(if $(FUSED_PROF),-DSB200_FUSED_PROF)
CSRC     := $(wildcard sedumi_b200/csrc/*.cu)
COBJ     := $(CSRC:.cu=.o)
LIB      := sedumi_b200/libsedumi_b200.so
MEXSRC   := $(filter-out %mex_common.cpp,$(wildcard sedumi_b200/mex/*.cpp))
MEXSO    := $(MEXSRC:.cpp=.so)

.PHONY: all shim oracle clean
all: shim $(LIB) $(MEXSO)

shim:
	$(MAKE) -C mxshim

sedumi_b200/csrc/%.o: sedumi_b200/csrc/%.cu $(wildcard sedumi_b200/csrc/*.h sedumi_b200/csrc/*.cuh) include/sedumi_b200.h
	$(NVCC) $(NVFLAGS) -c -o $@ $<

$(LIB): $(COBJ)
	$(NVCC) $(ARCH) -shared -o $@ $(COBJ) -lcudart -ldl

sedumi_b200/mex/%.so: sedumi_b200/mex/%.cpp sedumi_b200/mex/mex_common.h include/sedumi_b200.h $(LIB) | shim
	$(CXX) -O2 -std=c++17 -fPIC -shared -Imxshim -Iinclude -o $@ $< -Lsedumi_b200 -lsedumi_b200 -Lmxshim -lmxshim \
	  -Wl,-rpath,'$$ORIGIN/..:$$ORIGIN/../../mxshim'

oracle: shim
	$(MAKE) -C oracle

clean:
	rm -f $(COBJ) $(LIB) $(MEXSO)
	$(MAKE) -C mxshim clean
