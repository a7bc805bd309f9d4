# Builds the frame ingest's checker (test infrastructure), next to the oracle of Makefile:
#   liborb_ingest.so    the CPU restatement of cvtColor(*2GRAY), remap(INTER_LINEAR, CV_32FC1 maps) and Tracking's 16-bit
#                       depth conversion (orb_ingest.cpp)
# Every float expression is compiled as written: -ffp-contract=off.
# Used as `make -f ingest.mk liborb_ingest.so`.
CXX ?= g++

liborb_ingest.so: orb_ingest.cpp ingest_oracle.h
	$(CXX) -O2 -march=x86-64-v3 -ffp-contract=off -fno-fast-math -std=c++17 -fPIC -Wall -shared -o $@ orb_ingest.cpp
