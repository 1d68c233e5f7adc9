# CPU ORACLE of the translation-averaging step (test infrastructure), a library of its own on top of
# liboracle_rotavg.so (whose bi-edge-connected component and dense Cholesky it reuses) and liboracle_relpose.so (Ceres'
# rotation conversions):
#   make -C oracle -f transavg.mk
# Same flags as the Makefile (-ffp-contract=off, no -ffast-math).
CXX := g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -fopenmp -ffp-contract=off -fno-fast-math -Wall -Wextra
OUT := _build/liboracle_transavg.so

all: $(OUT)

_build/liboracle_rotavg.so: FORCE
	$(MAKE) -f rotavg.mk

$(OUT): oracle_transavg.cpp oracle_transavg.h oracle_relpose.h oracle.h _build/liboracle_rotavg.so
	$(CXX) $(CXXFLAGS) -shared -o $@ oracle_transavg.cpp -L_build -loracle_rotavg -loracle_relpose -loracle -Wl,-rpath,'$$ORIGIN'

FORCE:
.PHONY: all FORCE
