# ORACLE build with RTXPT's debug views — test infrastructure only:
#   make -C oracle -f debug_views.mk    _build/debug_views/liboracle_debug_views.so: the committed oracle (same flags as liboracle.so) plus the entries of debug_views_oracle.cpp
CXX      := $(shell command -v /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O2 -std=c++17 -fPIC -fopenmp -ffp-contract=off -fno-fast-math -fvisibility=hidden -Wall -Wno-unused-function
HDRS     := $(wildcard *.h) ../include/rtxpt_b200.h

_build/debug_views/liboracle_debug_views.so: debug_views_oracle.cpp oracle.cpp debug_views.mk $(HDRS)
	@mkdir -p _build/debug_views
	$(CXX) $(CXXFLAGS) -I. -shared -o $@ debug_views_oracle.cpp
