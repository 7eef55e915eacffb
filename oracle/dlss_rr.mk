# ORACLE build with RTXPT's DLSS-RR input pass — test infrastructure only:
#   make -C oracle -f dlss_rr.mk    _build/dlss_rr/liboracle_dlss_rr.so: the committed oracle (same flags as liboracle.so) plus the entries of dlss_rr_oracle.cpp
CXX      := $(shell command -v /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O2 -std=c++17 -fPIC -fopenmp -ffp-contract=off -fno-fast-math -fvisibility=hidden -Wall -Wno-unused-function
HDRS     := $(wildcard *.h) ../include/rtxpt_b200.h

_build/dlss_rr/liboracle_dlss_rr.so: dlss_rr_oracle.cpp oracle.cpp dlss_rr.mk $(HDRS)
	@mkdir -p _build/dlss_rr
	$(CXX) $(CXXFLAGS) -I. -shared -o $@ dlss_rr_oracle.cpp
