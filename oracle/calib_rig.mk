# ORACLE — test infrastructure only.  liborc_calib_rig.so: the online-calibration step over the whole rig with its priors
# (orc_calib_rig.cpp), on top of the headers of liborc.so and with its flags (Makefile): IEEE results independent of the flags.
CXX      := /usr/bin/g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -fopenmp -Wall -Wno-unused-function -Wno-array-bounds

liborc_calib_rig.so: orc_calib_rig.cpp $(wildcard *.hpp)
	$(CXX) $(CXXFLAGS) -shared -o $@ orc_calib_rig.cpp -ldl
