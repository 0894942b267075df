# Build recipe of the position-only guided-matching oracle and of the GeometricFilterMatrix_H_AC batch adaptor test (TEST
# INFRASTRUCTURE), with the flags of oracle/Makefile.  `make -f homography_filter.mk` builds the oracle; `adaptor REF=<AliceVision>/src`
# compiles tests/cpp/homography_filter_test.cpp against the reference's own headers (through shim/) and links the "ref" a-contrario
# RANSAC (homography) and guided-matching oracles, into _ref/ (git-ignored).
CXX = g++
REF ?= $(ALICEVISION_SRC)
CXXFLAGS = -O3 -fopenmp -msse2 -std=c++17 -fPIC -ffp-contract=off

all: libguided_positions.so
adaptor: _ref/homography_filter_test

libguided_positions.so: guided_positions_oracle.cpp
	$(CXX) $(CXXFLAGS) -shared $< -o $@

_ref/homography_filter_test: ../tests/cpp/homography_filter_test.cpp ../alicevision_b200/adaptor/GeometricFilter_b200.hpp ../alicevision_b200/adaptor/guidedMatchingFast_b200.hpp ../alicevision_b200/adaptor/RegionsMatcher_b200.hpp ../alicevision_b200/libb200match.so _ref/libref_acransac_h.so libguided_positions.so
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -I shim -I $(REF) -I ../include -I ../alicevision_b200/adaptor $< -o $@ -L ../alicevision_b200 -lb200match -L _ref -lref_acransac_h -L . -lguided_positions -Wl,-rpath,'$$ORIGIN/../../alicevision_b200' -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/..'

clean:
	rm -f libguided_positions.so _ref/homography_filter_test
