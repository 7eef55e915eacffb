# ORACLE build for stochastic texture filtering — test infrastructure only:
#   make -C oracle -f stf.mk         _build/stf/liboracle_stf.so: the oracle (same flags as liboracle.so) with pt_stf.h applied in loadSurface and oracle_set_texture_filtering; its
#                                    sources are written by stf_oracle.py from the committed pt_scene.h / oracle.cpp, which stay the trilinear oracle
#   make -C oracle -f stf.mk ref     (only when the reference tree is present) _ref/ref_kat_stf: the UNMODIFIED RTXTF headers (External/Rtxtf) as ref_stf_tu.sh streams them
#                                    behind ref_hlsl_shim.h, driven by ref_kat_stf_main.cpp; tests/golden/make_stf_golden.py runs it
SHELL       := /bin/bash
.SHELLFLAGS := -o pipefail -c
CXX    := $(shell command -v /usr/bin/g++ || echo g++)
REF    ?= /root/reference
CXXFLAGS ?= -O2 -std=c++17 -fPIC -fopenmp -ffp-contract=off -fno-fast-math -fvisibility=hidden -Wall -Wno-unused-function
HDRS   := $(wildcard *.h) ../include/rtxpt_b200.h
REFCXX := $(CXX) -x c++ -O1 -std=c++17 -fpermissive -w -ffp-contract=off -fno-fast-math -include string -I.

_build/stf/liboracle_stf.so: oracle.cpp stf_oracle.py stf.mk $(HDRS)
	python3 stf_oracle.py _build/stf
	$(CXX) $(CXXFLAGS) -I. -shared -o $@ _build/stf/oracle.cpp

ref:
	@if [ -d $(REF)/External/Rtxtf ]; then $(MAKE) -f stf.mk _ref/ref_kat_stf; else echo "reference tree absent: oracle/_ref not rebuilt"; fi

_ref/ref_kat_stf: ref_kat_stf_main.cpp ref_hlsl_shim.h ref_hlsl_tu.sh ref_stf_tu.sh stf.mk
	@mkdir -p _ref
	REF=$(REF) ./ref_stf_tu.sh | $(REFCXX) -o $@ -

.PHONY: ref
