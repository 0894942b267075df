# Build recipe of the a-contrario RANSAC oracle (TEST INFRASTRUCTURE), with the flags of oracle/Makefile.  `make -f acransac.mk`
# builds the port; `ref REF=<AliceVision>/src` additionally compiles the reference's ACRansac.hpp, randSampling.hpp and
# polynomial.hpp (verbatim, through oracle/shim) into _ref/ (git-ignored).
CXX = g++
REF ?= $(ALICEVISION_SRC)
CXXFLAGS = -O3 -msse2 -std=c++17 -fPIC -ffp-contract=off

all: libport_acransac.so
ref: _ref/libref_acransac.so

libport_acransac.so: acransac_oracle.cpp ../alicevision_b200/csrc/acransac_math.h
	$(CXX) $(CXXFLAGS) -shared $< -o $@

_ref/libref_acransac.so: acransac_oracle.cpp ../alicevision_b200/csrc/acransac_math.h $(wildcard shim/*/* shim/*/*/*)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -shared -DACR_USE_REFERENCE -I shim -I $(REF) $< -o $@

clean:
	rm -f libport_acransac.so _ref/libref_acransac.so
