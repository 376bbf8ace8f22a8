# ORACLE — test infrastructure only. Builds libforma_oracle_over.so, the oracle's frames over a
# background (forma_oracle_over.cpp), with the flags of oracle/Makefile: the library works on
# compositions built by libforma_oracle.so, so both must see the same layouts.
#     make -C oracle -f over.mk
CXX = /usr/bin/g++
CXXFLAGS = -std=c++17 -O3 -march=x86-64-v3 -ffp-contract=off -fno-fast-math -fopenmp -fPIC -Wall -Wextra -Wno-unused-parameter
HDRS = fmath.hpp path.hpp scene.hpp raster.hpp painter.hpp painter_over.hpp ../forma_b200/csrc/srgb_decode.h

all: libforma_oracle_over.so

libforma_oracle_over.so: forma_oracle_over.cpp $(HDRS)
	$(CXX) $(CXXFLAGS) -shared -o $@ forma_oracle_over.cpp

clean:
	rm -f libforma_oracle_over.so

.PHONY: all clean
