# CPU ORACLE of the Fast-AKAZE detector (test infrastructure), a library of its own:
#   make -C oracle -f akaze.mk
# Same flags as the Makefile (-ffp-contract=off, no -ffast-math): its arithmetic must be reproducible.
CXX := g++
CXXFLAGS ?= -O2 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wextra
OUT := _build/liboracle_akaze.so

all: $(OUT)

$(OUT): oracle_akaze.cpp
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -shared -o $@ oracle_akaze.cpp

.PHONY: all
