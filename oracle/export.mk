# CPU ORACLE of the colour plan, the coloured PLY and the undistortion (test infrastructure), a library of its own:
#   make -C oracle -f export.mk
# Same flags as the Makefile (-ffp-contract=off, no -ffast-math): its undistorted bytes must be reproducible.
CXX := g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -fopenmp -ffp-contract=off -fno-fast-math -Wall -Wextra
OUT := _build/liboracle_export.so

all: $(OUT)

$(OUT): oracle_export.cpp oracle_detmath.hpp
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -shared -o $@ oracle_export.cpp

.PHONY: all
