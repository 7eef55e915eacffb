# TEST INFRASTRUCTURE: make -C tests/emu -f env_update.mk.  Two libraries for the tests of rtxpt_b200_update_env_map:
#   _build/libenv_update_emu.so  host build of the product's importance-map bodies (env_update_host_emu.cu); no contraction, as the strict object the libraries link
#   _build/liboracle_env.so      the oracle plus the entry points that replace a context's environment (oracle_env_update.cpp); the oracle's compiler and flags (oracle/Makefile)
NVCC ?= /usr/local/cuda/bin/nvcc
CXX  := $(shell command -v /usr/bin/g++ || echo g++)
CSRC := ../../rtxpt_b200/csrc
ORC  := ../../oracle

all: _build/libenv_update_emu.so _build/liboracle_env.so

_build/libenv_update_emu.so: env_update_host_emu.cu $(CSRC)/envbake.cuh $(CSRC)/device_math.cuh
	@mkdir -p _build
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O2 -std=c++17 -fmad=false -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -o $@ env_update_host_emu.cu -Xcompiler -fopenmp

_build/liboracle_env.so: oracle_env_update.cpp $(ORC)/oracle.cpp $(wildcard $(ORC)/*.h) ../../include/rtxpt_b200.h
	@mkdir -p _build
	$(CXX) -O2 -std=c++17 -fPIC -fopenmp -ffp-contract=off -fno-fast-math -fvisibility=hidden -Wno-unused-function -Wno-unused-variable -shared -o $@ oracle_env_update.cpp

.PHONY: all
