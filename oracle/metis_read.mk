# The reference's METIS reader as a program (_ref/metis_read, ref_metis_read.cc + the unmodified
# $(REF)/kaminpar-io/metis_parser.cc), timed by scripts/bench_metis.py. Release flags as the reference's default CMake
# build type (-O3 -DNDEBUG); the rest of the reference comes from _ref/libkaminpar_ref_full.so (Makefile: ref_full).
#     make -f metis_read.mk
REF      ?= /root/reference
CXX      ?= g++
REF_INC  := -I ref_shim -I $(REF) -I $(REF)/include -I $(REF)/include/kaminpar-shm

_ref/metis_read: ref_metis_read.cc $(REF)/kaminpar-io/metis_parser.cc _ref/libkaminpar_ref_full.so
	$(CXX) -std=c++20 -O3 -DNDEBUG -w -mcx16 $(REF_INC) ref_metis_read.cc $(REF)/kaminpar-io/metis_parser.cc \
	  -o $@ -L_ref -lkaminpar_ref_full -Wl,-rpath,'$$ORIGIN'
