# Build recipe of the spherical a-contrario RANSAC oracle (TEST INFRASTRUCTURE), with the flags of oracle/acransac.mk.
# `make -f acransac_s.mk` builds the port; `ref REF=<AliceVision>/src` additionally compiles the reference's ACRansac.hpp,
# randSampling.hpp and polynomial.hpp (verbatim, through oracle/shim) into _ref/ (git-ignored).
CXX = g++
REF ?= $(ALICEVISION_SRC)
CXXFLAGS = -O3 -msse2 -std=c++17 -fPIC -ffp-contract=off

all: libport_acransac_s.so
ref: _ref/libref_acransac_s.so

libport_acransac_s.so: acransac_s_oracle.cpp ../alicevision_b200/csrc/acransac_math.h
	$(CXX) $(CXXFLAGS) -shared $< -o $@

_ref/libref_acransac_s.so: acransac_s_oracle.cpp ../alicevision_b200/csrc/acransac_math.h $(wildcard shim/*/* shim/*/*/*)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -shared -DACR_USE_REFERENCE -I shim -I $(REF) $< -o $@

clean:
	rm -f libport_acransac_s.so _ref/libref_acransac_s.so
