# Build recipe of the GeometricFilterMatrix_F_AC batch adaptor test with estimateDistortion (TEST INFRASTRUCTURE), with the flags of
# oracle/Makefile: `make -f distortion_filter.mk REF=<AliceVision>/src` compiles tests/cpp/distortion_filter_test.cpp against the
# reference's own headers (through shim/) and links the "ref" F10 a-contrario RANSAC and guided-matching oracles, into _ref/ (git-ignored).
CXX = g++
REF ?= $(ALICEVISION_SRC)
CXXFLAGS = -O3 -fopenmp -msse2 -std=c++17 -fPIC -ffp-contract=off

all: _ref/distortion_filter_test

_ref/distortion_filter_test: ../tests/cpp/distortion_filter_test.cpp ../alicevision_b200/adaptor/GeometricFilter_b200.hpp ../alicevision_b200/adaptor/RegionsMatcher_b200.hpp ../alicevision_b200/libb200match.so _ref/libref_acransac_f10.so _ref/libref_guided_fast.so
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -I shim -I $(REF) -I ../include -I ../alicevision_b200/adaptor $< -o $@ -L ../alicevision_b200 -lb200match -L _ref -lref_acransac_f10 -lref_guided_fast -Wl,-rpath,'$$ORIGIN/../../alicevision_b200' -Wl,-rpath,'$$ORIGIN'

clean:
	rm -f _ref/distortion_filter_test
