# ORACLE/_ref — RTXPT's DLSS-RR input pass (only when the reference tree is present):
#   make -C oracle -f dlss_rr_ref.mk ref   _ref/ref_kat_dlss_rr: the UNMODIFIED PostProcess.hlsl DENOISER_DLSS_RR pass and ComputeSpecularMotionVector as ref_dlss_rr_tu.sh streams
#                                         them behind ref_hlsl_shim.h and the path-tracer headers, driven by ref_kat_dlss_rr_main.cpp; tests/golden/make_dlss_rr_golden.py runs it
SHELL       := /bin/bash
.SHELLFLAGS := -o pipefail -c
CXX    := $(shell command -v /usr/bin/g++ || echo g++)
REF    ?= /root/reference
REFCXX := $(CXX) -x c++ -O1 -std=c++17 -fpermissive -w -ffp-contract=off -fno-fast-math -include string -I.

ref:
	@if [ -d $(REF)/Rtxpt/ProcessingPasses ] && [ -d $(REF)/Rtxpt/Shaders/PathTracer/Utils ]; then $(MAKE) -f dlss_rr_ref.mk _ref/ref_kat_dlss_rr; else echo "reference tree absent: oracle/_ref not rebuilt"; fi

_ref/ref_kat_dlss_rr: ref_kat_dlss_rr_main.cpp ref_hlsl_shim.h ref_hlsl_tu.sh ref_bridge_stub.h ref_dlss_rr_tu.sh dlss_rr_ref.mk
	@mkdir -p _ref
	REF=$(REF) ./ref_dlss_rr_tu.sh | $(REFCXX) -o $@ -

.PHONY: ref
