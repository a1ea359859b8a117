# ORACLE — test infrastructure only.  liborc_registered.so: pubPointCloud at a given pose (orc_registered.cpp), on top of the headers of
# liborc.so and with its flags (Makefile): IEEE results independent of the flags.
CXX      := /usr/bin/g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -fopenmp -Wall -Wno-unused-function -Wno-array-bounds

liborc_registered.so: orc_registered.cpp $(wildcard *.hpp)
	$(CXX) $(CXXFLAGS) -shared -o $@ orc_registered.cpp -ldl
