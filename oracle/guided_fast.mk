# Build recipe of the guided-matching-on-double-positions oracle and of the guidedMatchingFundamentalFast adaptor test (TEST
# INFRASTRUCTURE), with the flags of oracle/Makefile.  `make -f guided_fast.mk` builds the port; `ref REF=<AliceVision>/src`
# additionally compiles the reference's own Regions headers into _ref/ (git-ignored); `adaptor REF=...` builds the C++ adaptor test.
CXX = g++
REF ?= $(ALICEVISION_SRC)
CXXFLAGS = -O3 -fopenmp -msse2 -std=c++17 -fPIC -ffp-contract=off

all: libport_guided_fast.so
ref: _ref/libref_guided_fast.so
adaptor: _ref/guided_fast_adaptor_test

libport_guided_fast.so: guided_fast_oracle.cpp
	$(CXX) $(CXXFLAGS) -shared $< -o $@

_ref/libref_guided_fast.so: guided_fast_oracle.cpp $(wildcard shim/*/* shim/*/*/*)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -shared -DGF_USE_REFERENCE -I shim -I $(REF) $< -o $@

_ref/guided_fast_adaptor_test: ../tests/cpp/guided_fast_test.cpp ../alicevision_b200/adaptor/guidedMatchingFast_b200.hpp ../alicevision_b200/adaptor/RegionsMatcher_b200.hpp ../alicevision_b200/libb200match.so _ref/libref_guided_fast.so
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -I shim -I $(REF) -I ../include -I ../alicevision_b200/adaptor $< -o $@ -L ../alicevision_b200 -lb200match -L _ref -lref_guided_fast -Wl,-rpath,'$$ORIGIN/../../alicevision_b200' -Wl,-rpath,'$$ORIGIN'

clean:
	rm -f libport_guided_fast.so _ref/libref_guided_fast.so _ref/guided_fast_adaptor_test
