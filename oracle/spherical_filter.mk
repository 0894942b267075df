# Build recipe of the GeometricFilterMatrix_F_AC batch adaptor test on a list of planar and spherical pairs (TEST INFRASTRUCTURE), with
# the flags of oracle/Makefile: `make -f spherical_filter.mk REF=<AliceVision>/src` compiles tests/cpp/spherical_filter_test.cpp against
# the reference's own headers (through shim/) and links the "ref" planar and spherical a-contrario RANSAC and guided-matching oracles,
# into _ref/ (git-ignored).
CXX = g++
REF ?= $(ALICEVISION_SRC)
CXXFLAGS = -O3 -fopenmp -msse2 -std=c++17 -fPIC -ffp-contract=off

all: _ref/spherical_filter_test

_ref/spherical_filter_test: ../tests/cpp/spherical_filter_test.cpp ../alicevision_b200/adaptor/GeometricFilter_b200.hpp ../alicevision_b200/adaptor/guidedMatchingFast_b200.hpp ../alicevision_b200/adaptor/RegionsMatcher_b200.hpp ../alicevision_b200/libb200match.so _ref/libref_acransac.so _ref/libref_acransac_s.so _ref/libref_guided_fast.so
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -I shim -I $(REF) -I ../include -I ../alicevision_b200/adaptor $< -o $@ -L ../alicevision_b200 -lb200match -L _ref -lref_acransac -lref_acransac_s -lref_guided_fast -Wl,-rpath,'$$ORIGIN/../../alicevision_b200' -Wl,-rpath,'$$ORIGIN'

clean:
	rm -f _ref/spherical_filter_test
