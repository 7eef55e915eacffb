# TEST INFRASTRUCTURE: host build of the ReBLUR pass bodies under panel settings (see reblur_settings_host_emu.cu): make -C tests/emu -f reblur_settings.mk.  Same floating-point
# contract as the oracle and libreblur_emu.so: no contraction.
NVCC ?= /usr/local/cuda/bin/nvcc
CSRC := ../../rtxpt_b200/csrc
_build/libreblur_settings_emu.so: reblur_settings_host_emu.cu reblur_settings.mk $(CSRC)/reblur_passes.cuh $(CSRC)/reblur.cuh $(CSRC)/reblur_host.h $(CSRC)/device_math.cuh ../../include/rtxpt_b200.h
	@mkdir -p _build
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O2 -std=c++17 -fmad=false -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -o $@ reblur_settings_host_emu.cu -Xcompiler -fopenmp
