# CPU ORACLE of the resection step (test infrastructure), a library of its own on top of liboracle.so:
#   make -C oracle -f resection.mk
# Same flags as the Makefile (-ffp-contract=off, no -ffast-math): its decisions must be reproducible.
CXX := g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -fopenmp -ffp-contract=off -fno-fast-math -Wall -Wextra
OUT := _build/liboracle_resection.so

all: $(OUT)

_build/liboracle.so: FORCE
	$(MAKE) -f Makefile

$(OUT): oracle_resection.cpp oracle_resection.h oracle.h oracle_detmath.hpp _build/liboracle.so
	$(CXX) $(CXXFLAGS) -shared -o $@ oracle_resection.cpp -L_build -loracle -Wl,-rpath,'$$ORIGIN'

FORCE:
.PHONY: all FORCE
