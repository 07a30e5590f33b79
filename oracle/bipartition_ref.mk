# The reference's initial bipartitioner as a program (ref_bipartition.cc + _ref/libkaminpar_ref_full.so), timed by
# scripts/bench_bipartition.py: _ref/bipartition_ref at one thread, _ref/bipartition_ref_omp with the blocks on all
# cores (OpenMP, timing only). Release flags as the reference's default CMake build type (-O3 -DNDEBUG).
#     make -f bipartition_ref.mk
REF      ?= /root/reference
CXX      := /usr/bin/g++
REF_INC  := -I ref_shim -I $(REF) -I $(REF)/include -I $(REF)/include/kaminpar-shm

all: _ref/bipartition_ref _ref/bipartition_ref_omp

_ref/bipartition_ref: ref_bipartition.cc _ref/libkaminpar_ref_full.so
	$(CXX) -std=c++20 -O3 -DNDEBUG -w -mcx16 $(REF_INC) ref_bipartition.cc -o $@ -L_ref -lkaminpar_ref_full \
	  -Wl,-rpath,'$$ORIGIN'

_ref/bipartition_ref_omp: ref_bipartition.cc _ref/libkaminpar_ref_full.so
	$(CXX) -std=c++20 -O3 -DNDEBUG -w -mcx16 -fopenmp $(REF_INC) ref_bipartition.cc -o $@ -L_ref \
	  -lkaminpar_ref_full -Wl,-rpath,'$$ORIGIN'
