# TEST INFRASTRUCTURE: host build of the approximate-MIS shade (see approximate_mis_host_emu.cu): make -C tests/emu -f approximate_mis.mk.  Same flags as libshade_emu.so
# (Makefile): no contraction.
NVCC ?= /usr/local/cuda/bin/nvcc
CSRC := ../../rtxpt_b200/csrc
_build/libapproximate_mis_emu.so: approximate_mis_host_emu.cu nee_full_samples_host_emu.cu shade_host_emu.cu $(CSRC)/shade.cuh $(CSRC)/realtime.cuh $(CSRC)/wavefront.cuh $(CSRC)/bsdf.cuh $(CSRC)/device_math.cuh $(CSRC)/neeat.cuh $(CSRC)/scene_device.cuh
	@mkdir -p _build
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O1 -std=c++17 -fmad=false -diag-suppress 20011,20014 -Xcompiler -fPIC,-ffp-contract=off -shared -o $@ approximate_mis_host_emu.cu
