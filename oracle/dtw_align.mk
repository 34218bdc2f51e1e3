# oracle/dtw_align.mk -- the checkers of `uncalled_b200 dtw` (test infrastructure only):
#   libunc_oracle_dtw_align.so   the C restatement (unc_oracle_dtw_align.c), over libunc_oracle.so
#   _ref/libref_dtw_align.so     the reference's own code (ref_build/ref_dtw_align.cpp), over _ref/libuncalled_ref.so,
#                                when the reference tree is present (else a prebuilt one is kept).  Its own definitions
#                                are hidden: the driver's dtwcost_r94d (float abs) must not interpose on the library's
#                                (int abs), which has the same name.
# Same flags as oracle/Makefile and oracle/ref_build/Makefile.  make -C oracle -f dtw_align.mk
CC ?= gcc
CXX ?= g++
REF ?= /root/reference
CFLAGS := -O2 -ffp-contract=off -fPIC -Wall -Wno-unused-function -pthread
CXXFLAGS := -std=c++11 -O3 -fPIC -pthread -w
INCS := -Iref_build/stubs -I$(REF)/src -I$(REF)/submods -I$(REF)/submods/pdqsort

all: libunc_oracle_dtw_align.so ref

libunc_oracle.so: unc_oracle.c unc_oracle.h
	$(MAKE) libunc_oracle.so

libunc_oracle_dtw_align.so: unc_oracle_dtw_align.c unc_oracle.h libunc_oracle.so
	$(CC) $(CFLAGS) -shared -o $@ unc_oracle_dtw_align.c -L. -lunc_oracle -Wl,-rpath,'$$ORIGIN' -lm

ref:
	@if [ -d $(REF)/src ]; then $(MAKE) -C ref_build REF=$(REF) && $(MAKE) -f dtw_align.mk _ref/libref_dtw_align.so; else echo "no reference tree: keeping prebuilt oracle/_ref"; fi

_ref/libref_dtw_align.so: ref_build/ref_dtw_align.cpp _ref/libuncalled_ref.so
	$(CXX) $(CXXFLAGS) -fvisibility=hidden $(INCS) -shared -o $@ ref_build/ref_dtw_align.cpp -L_ref -luncalled_ref -Wl,-rpath,'$$ORIGIN' -lz -lm

.PHONY: all ref
