# oracle/bwa_index.mk -- the checkers of the BwaIndex queries (test infrastructure only):
#   libunc_oracle_bwa_index.so   the C restatement (unc_oracle_bwa_index.c, which compiles unc_oracle.c into itself)
#   _ref/libref_bwa_index.so     the reference's own BwaIndex<k5> and k-mer helpers (ref_build/ref_bwa_index.cpp), over
#                                _ref/libuncalled_ref.so, when the reference tree is present (else a prebuilt one is
#                                kept).  Its own definitions are hidden.
# Same flags as oracle/Makefile and oracle/ref_build/Makefile.  make -C oracle -f bwa_index.mk
CC ?= gcc
CXX ?= g++
REF ?= /root/reference
CFLAGS := -O2 -ffp-contract=off -fPIC -Wall -Wno-unused-function -pthread
CXXFLAGS := -std=c++11 -O3 -fPIC -pthread -w
INCS := -Iref_build/stubs -I$(REF)/src -I$(REF)/submods -I$(REF)/submods/pdqsort

all: libunc_oracle_bwa_index.so ref

libunc_oracle_bwa_index.so: unc_oracle_bwa_index.c unc_oracle.c unc_oracle.h
	$(CC) $(CFLAGS) -shared -o $@ unc_oracle_bwa_index.c -lm

ref:
	@if [ -d $(REF)/src ]; then $(MAKE) -C ref_build REF=$(REF) && $(MAKE) -f bwa_index.mk _ref/libref_bwa_index.so; else echo "no reference tree: keeping prebuilt oracle/_ref"; fi

_ref/libref_bwa_index.so: ref_build/ref_bwa_index.cpp _ref/libuncalled_ref.so
	$(CXX) $(CXXFLAGS) -fvisibility=hidden $(INCS) -shared -o $@ ref_build/ref_bwa_index.cpp -L_ref -luncalled_ref -Wl,-rpath,'$$ORIGIN' -lz -lm

.PHONY: all ref
