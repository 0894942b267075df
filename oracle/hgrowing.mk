# Build recipe of the homography-growing oracle (TEST INFRASTRUCTURE): the single-threaded port on the engine's shared math header.
# There is no "ref" build: the reference's fits and refine need Eigen's JacobiSVD and Ceres.  `adaptor REF=<AliceVision>/src` compiles
# tests/cpp/hgrowing_filter_test.cpp against the reference's own headers (through shim/) and links the port, into _ref/ (git-ignored).
CXX = g++
REF ?= $(ALICEVISION_SRC)
CXXFLAGS = -O3 -msse2 -std=c++17 -fPIC -ffp-contract=off

all: libport_hgrowing.so
adaptor: _ref/hgrowing_filter_test

libport_hgrowing.so: hgrowing_oracle.cpp ../alicevision_b200/csrc/hgrowing_math.h ../alicevision_b200/csrc/acransac_math.h
	$(CXX) $(CXXFLAGS) -shared $< -o $@

_ref/hgrowing_filter_test: ../tests/cpp/hgrowing_filter_test.cpp ../alicevision_b200/adaptor/GeometricFilter_b200.hpp ../alicevision_b200/adaptor/RegionsMatcher_b200.hpp ../alicevision_b200/libb200match.so libport_hgrowing.so
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -fopenmp -I shim -I $(REF) -I ../include -I ../alicevision_b200/adaptor $< -o $@ -L ../alicevision_b200 -lb200match -L . -lport_hgrowing -Wl,-rpath,'$$ORIGIN/../../alicevision_b200' -Wl,-rpath,'$$ORIGIN/..'

clean:
	rm -f libport_hgrowing.so _ref/hgrowing_filter_test
