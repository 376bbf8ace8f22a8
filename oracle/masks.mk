# ORACLE — test infrastructure only. Builds libforma_oracle_masks.so, the oracle's layer coverage masks
# (forma_oracle_masks.cpp), with the flags of oracle/Makefile: the library works on compositions
# built by libforma_oracle.so, so both must see the same layouts.
#     make -C oracle -f masks.mk
CXX = /usr/bin/g++
CXXFLAGS = -std=c++17 -O3 -march=x86-64-v3 -ffp-contract=off -fno-fast-math -fopenmp -fPIC -Wall -Wextra -Wno-unused-parameter
HDRS = fmath.hpp path.hpp scene.hpp raster.hpp painter.hpp painter_masks.hpp

all: libforma_oracle_masks.so

libforma_oracle_masks.so: forma_oracle_masks.cpp $(HDRS)
	$(CXX) $(CXXFLAGS) -shared -o $@ forma_oracle_masks.cpp

clean:
	rm -f libforma_oracle_masks.so

.PHONY: all clean
