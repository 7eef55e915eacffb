# TEST INFRASTRUCTURE: host build of the product's BVH rebuild bodies (see bvh_build_host_emu.cu): make -C tests/emu -f bvh_build.mk.  Same floating-point contract as the
# device build the libraries link (csrc/Makefile: the strict object): no contraction.
NVCC ?= /usr/local/cuda/bin/nvcc
CSRC := ../../rtxpt_b200/csrc
BVHBUILDER := $(CSRC)/_build/bvh_builder.o
_build/libbvh_build_emu.so: bvh_build_host_emu.cu $(BVHBUILDER) $(CSRC)/bvh_build.cuh $(CSRC)/bvh8.h $(CSRC)/device_math.cuh
	@mkdir -p _build
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O2 -std=c++17 -fmad=false -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -o $@ bvh_build_host_emu.cu $(BVHBUILDER) -Xcompiler -fopenmp
$(BVHBUILDER): $(CSRC)/bvh_builder.cpp $(CSRC)/bvh8.h
	$(MAKE) -C $(CSRC) _build/bvh_builder.o
