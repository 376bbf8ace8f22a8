# ORACLE — test infrastructure only. Builds libforma_oracle_stats.so, the oracle's layer statistics
# (forma_oracle_stats.cpp), with the flags of oracle/Makefile: the library works on compositions
# built by libforma_oracle.so, so both must see the same layouts.
#     make -C oracle -f stats.mk
CXX = /usr/bin/g++
CXXFLAGS = -std=c++17 -O3 -march=x86-64-v3 -ffp-contract=off -fno-fast-math -fopenmp -fPIC -Wall -Wextra -Wno-unused-parameter
HDRS = fmath.hpp path.hpp scene.hpp raster.hpp painter.hpp painter_ids.hpp painter_masks.hpp

all: libforma_oracle_stats.so

libforma_oracle_stats.so: forma_oracle_stats.cpp $(HDRS)
	$(CXX) $(CXXFLAGS) -shared -o $@ forma_oracle_stats.cpp

clean:
	rm -f libforma_oracle_stats.so

.PHONY: all clean
