# TEST INFRASTRUCTURE: host build of the traversal's node step (see slab_compare_host_emu.cu): make -C tests/emu -f slab_compare.mk.  No contraction: the reference formulation in
# that file and the product's function have to see the same plane distances.
NVCC ?= /usr/local/cuda/bin/nvcc
CSRC := ../../rtxpt_b200/csrc
_build/libslab_compare_emu.so: slab_compare_host_emu.cu $(CSRC)/traverse.cuh $(CSRC)/device_math.cuh $(CSRC)/scene_device.cuh
	@mkdir -p _build
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O2 -std=c++17 -fmad=false -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -o $@ slab_compare_host_emu.cu -Xcompiler -fopenmp
