# CPU ORACLE of the relative-pose step (test infrastructure), a library of its own on top of liboracle.so:
#   make -C oracle -f relpose.mk
# Same flags as the Makefile (-ffp-contract=off, no -ffast-math): its decisions must be reproducible.
CXX := g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -fopenmp -ffp-contract=off -fno-fast-math -Wall -Wextra
OUT := _build/liboracle_relpose.so

all: $(OUT)

_build/liboracle.so: FORCE
	$(MAKE) -f Makefile

$(OUT): oracle_relpose.cpp oracle_relpose.h oracle.h _build/liboracle.so
	$(CXX) $(CXXFLAGS) -shared -o $@ oracle_relpose.cpp -L_build -loracle -Wl,-rpath,'$$ORIGIN'

FORCE:
.PHONY: all FORCE
