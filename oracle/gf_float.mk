# ORACLE — test infrastructure only.  liborc_gf_float.so: the gd_float restatement (orc_gf_float.hpp) with its C entry points, on top of
# the headers of liborc.so and with its flags (Makefile): IEEE results independent of the flags.
CXX      := /usr/bin/g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -fopenmp -Wall -Wno-unused-function -Wno-array-bounds

liborc_gf_float.so: orc_gf_float.cpp $(wildcard *.hpp)
	$(CXX) $(CXXFLAGS) -shared -o $@ orc_gf_float.cpp -ldl
