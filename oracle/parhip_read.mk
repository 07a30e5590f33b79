# The reference's ParHIP reader as a program (_ref/parhip_read, ref_parhip_read.cc + the unmodified
# $(REF)/kaminpar-io/parhip_parser.cc), timed by scripts/bench_parhip.py. Release flags as the reference's default
# CMake build type (-O3 -DNDEBUG); the rest of the reference comes from _ref/libkaminpar_ref_full.so (Makefile:
# ref_full). The parser's tbb::parallel_for loops run on the serial oneTBB stand-in: one thread, not the reference's
# TBB build on all cores.
#     make -f parhip_read.mk
REF      ?= /root/reference
CXX      := /usr/bin/g++
REF_INC  := -I ref_shim -I $(REF) -I $(REF)/include -I $(REF)/include/kaminpar-shm

_ref/parhip_read: ref_parhip_read.cc $(REF)/kaminpar-io/parhip_parser.cc _ref/libkaminpar_ref_full.so
	$(CXX) -std=c++20 -O3 -DNDEBUG -w -mcx16 $(REF_INC) ref_parhip_read.cc $(REF)/kaminpar-io/parhip_parser.cc \
	  -o $@ -L_ref -lkaminpar_ref_full -Wl,-rpath,'$$ORIGIN'

