# CPU ORACLE of the rotation-averaging step (test infrastructure), a library of its own on top of liboracle_relpose.so
# (whose Jacobi SVD and Ceres rotation conversions it reuses):
#   make -C oracle -f rotavg.mk
# Same flags as the Makefile (-ffp-contract=off, no -ffast-math): its triplet decisions must be reproducible.
CXX := g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -fopenmp -ffp-contract=off -fno-fast-math -Wall -Wextra
OUT := _build/liboracle_rotavg.so

all: $(OUT)

_build/liboracle_relpose.so: FORCE
	$(MAKE) -f relpose.mk

$(OUT): oracle_rotavg.cpp oracle_rotavg.h oracle_relpose.h oracle.h oracle_detmath.hpp _build/liboracle_relpose.so
	$(CXX) $(CXXFLAGS) -shared -o $@ oracle_rotavg.cpp -L_build -loracle_relpose -loracle -Wl,-rpath,'$$ORIGIN'

FORCE:
.PHONY: all FORCE
