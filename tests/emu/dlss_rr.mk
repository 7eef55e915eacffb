# TEST INFRASTRUCTURE: host build of the DLSS-RR input pass (see dlss_rr_host_emu.cu): make -C tests/emu -f dlss_rr.mk.  No contraction, IEEE division and square root: what the
# strict library computes on the GPU.
NVCC ?= /usr/local/cuda/bin/nvcc
CSRC := ../../rtxpt_b200/csrc
_build/libdlss_rr_emu.so: dlss_rr_host_emu.cu $(CSRC)/denoiser_iface.cuh $(CSRC)/debug_views.cuh $(CSRC)/wavefront.cuh $(CSRC)/device_math.cuh ../../include/rtxpt_b200.h dlss_rr.mk
	@mkdir -p _build
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O2 -std=c++17 -fmad=false -prec-div=true -prec-sqrt=true -Xcompiler -fPIC,-ffp-contract=off -shared -o $@ dlss_rr_host_emu.cu
