# Build recipe of the fundamental-matrix-with-distortion (F10) a-contrario RANSAC oracle (TEST INFRASTRUCTURE), with the flags of
# oracle/acransac.mk.  `make -f acransac_f10.mk` builds the port; `ref REF=<AliceVision>/src` additionally compiles the reference's
# ACRansac.hpp and randSampling.hpp (verbatim, through oracle/shim) into _ref/ (git-ignored).
CXX = g++
REF ?= $(ALICEVISION_SRC)
CXXFLAGS = -O3 -msse2 -std=c++17 -fPIC -ffp-contract=off

all: libport_acransac_f10.so
ref: _ref/libref_acransac_f10.so

libport_acransac_f10.so: acransac_f10_oracle.cpp ../alicevision_b200/csrc/acransac_math.h
	$(CXX) $(CXXFLAGS) -shared $< -o $@

_ref/libref_acransac_f10.so: acransac_f10_oracle.cpp ../alicevision_b200/csrc/acransac_math.h $(wildcard shim/*/* shim/*/*/*)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -shared -DACR_USE_REFERENCE -I shim -I $(REF) $< -o $@

clean:
	rm -f libport_acransac_f10.so _ref/libref_acransac_f10.so
