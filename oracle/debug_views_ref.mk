# ORACLE/_ref — debug-view colour functions (only when the reference tree is present):
#   make -C oracle -f debug_views_ref.mk ref   _ref/ref_kat_debug: the UNMODIFIED ColorFromHash / GradientHeatMap / Unpack_R11G11B10_FLOAT / StablePlaneDebugVizColor /
#                                             StablePlaneDebugVizFourWaySplitCoord / DbgShowNormalSRGB as ref_debug_tu.sh streams them behind ref_hlsl_shim.h, driven by
#                                             ref_kat_debug_main.cpp; tests/golden/make_debug_view_golden.py runs it
SHELL       := /bin/bash
.SHELLFLAGS := -o pipefail -c
CXX    := $(shell command -v /usr/bin/g++ || echo g++)
REF    ?= /root/reference
REFCXX := $(CXX) -x c++ -O1 -std=c++17 -fpermissive -w -ffp-contract=off -fno-fast-math -include string -I.

ref:
	@if [ -d $(REF)/Rtxpt/Shaders/PathTracer/Utils ]; then $(MAKE) -f debug_views_ref.mk _ref/ref_kat_debug; else echo "reference tree absent: oracle/_ref not rebuilt"; fi

_ref/ref_kat_debug: ref_kat_debug_main.cpp ref_hlsl_shim.h ref_hlsl_tu.sh ref_debug_tu.sh debug_views_ref.mk
	@mkdir -p _ref
	REF=$(REF) ./ref_debug_tu.sh | $(REFCXX) -o $@ -

.PHONY: ref
