# ORACLE build for approximate light-vs-BSDF MIS (RTXPT_USE_APPROXIMATE_MIS = 1, RtxptPathTracerConstants::useApproximateMIS) — test infrastructure only:
#   make -C oracle -f amis.mk            _build/amis/liboracle_amis.so: the oracle (same flags as liboracle.so) with the switch honoured; its sources are written by
#                                        amis_oracle.py from the committed pt_path.h / oracle.cpp, which stay the full-MIS oracle
#   make -C oracle -f amis.mk ref        (only when the reference tree is present) _ref/ref_kat_bsdf_amis, _ref/ref_kat_pt_build_amis, _ref/ref_kat_pt_fill_amis: the three passes of
#                                        the UNMODIFIED reference headers as Makefile builds them, with the macro switched to 1 in the stream ref_hlsl_tu.sh writes (nothing on disk);
#                                        tests/golden/make_hit_golden_amis.py runs them
SHELL       := /bin/bash
.SHELLFLAGS := -o pipefail -c
CXX      := $(shell command -v /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O2 -std=c++17 -fPIC -fopenmp -ffp-contract=off -fno-fast-math -fvisibility=hidden -Wall -Wno-unused-function
REF      ?= /root/reference
HDRS     := $(wildcard *.h) ../include/rtxpt_b200.h

_build/amis/liboracle_amis.so: oracle.cpp amis_oracle.py $(HDRS)
	python3 amis_oracle.py _build/amis
	$(CXX) $(CXXFLAGS) -I. -shared -o $@ _build/amis/oracle.cpp

# RTXPT_USE_APPROXIMATE_MIS 0 -> 1 in the translation unit; fails unless the define was found exactly once
AMIS_MACRO := awk '{ if ($$0 == "\#define RTXPT_USE_APPROXIMATE_MIS 0") { print "\#define RTXPT_USE_APPROXIMATE_MIS 1"; n++ } else print } END { exit n != 1 }'
REFCXX     := $(CXX) -x c++ -O1 -std=c++17 -fpermissive -w -ffp-contract=off -fno-fast-math -include string -I.

ref:
	@if [ -d $(REF)/Rtxpt/Shaders/PathTracer/Utils ]; then $(MAKE) -f amis.mk _ref/ref_kat_bsdf_amis _ref/ref_kat_pt_build_amis _ref/ref_kat_pt_fill_amis; else echo "reference tree absent: oracle/_ref not rebuilt"; fi

_ref/ref_kat_bsdf_amis: ref_kat_bsdf_main.cpp ref_hlsl_shim.h ref_hlsl_tu.sh ref_bridge_stub.h amis.mk
	@mkdir -p _ref
	REF=$(REF) ./ref_hlsl_tu.sh ref_kat_bsdf_main.cpp | $(AMIS_MACRO) | $(REFCXX) -o $@ -
_ref/ref_kat_pt_build_amis: ref_kat_bsdf_main.cpp ref_hlsl_shim.h ref_hlsl_tu.sh ref_bridge_stub.h amis.mk
	@mkdir -p _ref
	REF=$(REF) ./ref_hlsl_tu.sh ref_kat_bsdf_main.cpp | $(AMIS_MACRO) | $(REFCXX) -DPATH_TRACER_MODE=1 -o $@ -
_ref/ref_kat_pt_fill_amis: ref_kat_bsdf_main.cpp ref_hlsl_shim.h ref_hlsl_tu.sh ref_bridge_stub.h amis.mk
	@mkdir -p _ref
	REF=$(REF) ./ref_hlsl_tu.sh ref_kat_bsdf_main.cpp | $(AMIS_MACRO) | $(REFCXX) -DPATH_TRACER_MODE=2 -o $@ -

.PHONY: ref
