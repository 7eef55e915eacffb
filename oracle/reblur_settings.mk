# ORACLE build with ReBLUR's panel settings — test infrastructure only:
#   make -C oracle -f reblur_settings.mk    _build/reblur_settings/liboracle_reblur_settings.so: the committed oracle (same flags as liboracle.so) plus the entries of reblur_settings_oracle.cpp
CXX      := $(shell command -v /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O2 -std=c++17 -fPIC -fopenmp -ffp-contract=off -fno-fast-math -fvisibility=hidden -Wall -Wno-unused-function
HDRS     := $(wildcard *.h) ../include/rtxpt_b200.h

_build/reblur_settings/liboracle_reblur_settings.so: reblur_settings_oracle.cpp oracle.cpp reblur_settings.mk $(HDRS)
	@mkdir -p _build/reblur_settings
	$(CXX) $(CXXFLAGS) -I. -shared -o $@ reblur_settings_oracle.cpp
