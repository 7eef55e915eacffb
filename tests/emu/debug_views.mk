# TEST INFRASTRUCTURE: host build of the debug-view pixel functions (see debug_views_host_emu.cu): make -C tests/emu -f debug_views.mk.  No contraction, IEEE division and
# square root: what the strict library computes on the GPU.
NVCC ?= /usr/local/cuda/bin/nvcc
CSRC := ../../rtxpt_b200/csrc
_build/libdebug_views_emu.so: debug_views_host_emu.cu $(CSRC)/debug_views.cuh $(CSRC)/device_math.cuh
	@mkdir -p _build
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O2 -std=c++17 -fmad=false -prec-div=true -prec-sqrt=true -Xcompiler -fPIC,-ffp-contract=off -shared -o $@ debug_views_host_emu.cu
