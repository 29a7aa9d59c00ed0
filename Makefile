# Builds the product library (sm_90a only) and the CPU oracle.
#   make            -> f2nerf_b200/libf2nerf_b200.so + oracle/libf2oracle.so
#   make ref        -> oracle/_ref/ref_driver (the unmodified reference, ~25 min; needs /root/reference)
NVCC    ?= /usr/local/cuda/bin/nvcc
ARCH    := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xptxas -v
CSRC    := f2nerf_b200/csrc
SRCS    := $(wildcard $(CSRC)/*.cu)
OBJS    := $(patsubst $(CSRC)/%.cu,build/%.o,$(SRCS))
DEFS    := $(if $(wildcard $(CSRC)/mlp_tc.cu),-DF2B_HAVE_TC,)

all: f2nerf_b200/libf2nerf_b200.so oracle/libf2oracle.so

build/%.o: $(CSRC)/%.cu $(wildcard $(CSRC)/*.cuh) include/f2nerf_b200.h
	@mkdir -p build
	$(NVCC) $(NVFLAGS) $(DEFS) -c $< -o $@ 2> build/$*.ptxas.log || (cat build/$*.ptxas.log; false)

f2nerf_b200/libf2nerf_b200.so: $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS)

oracle/libf2oracle.so: oracle/f2_oracle.c
	gcc -O2 -march=x86-64-v3 -fopenmp -ffp-contract=off -fno-fast-math -shared -fPIC $< -o $@ -lm

ref:
	$(MAKE) -f oracle/Makefile.ref -j8

clean:
	rm -rf build f2nerf_b200/libf2nerf_b200.so oracle/libf2oracle.so
.PHONY: all ref clean
