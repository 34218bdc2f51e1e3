# oracle/events.mk -- the checkers of `uncalled_b200 events` (test infrastructure only):
#   libunc_oracle_events.so   the C restatement (unc_oracle_events.c, which compiles unc_oracle.c into itself)
#   _ref/libref_events.so     the reference's own EventDetector / EventProfiler / Normalizer / PoreModel
#                             (ref_build/ref_events.cpp), over _ref/libuncalled_ref.so, when the reference tree is present
#                             (else a prebuilt one is kept)
# Same flags as oracle/Makefile and oracle/ref_build/Makefile.  make -C oracle -f events.mk
CC ?= gcc
CXX ?= g++
REF ?= /root/reference
CFLAGS := -O2 -ffp-contract=off -fPIC -Wall -Wno-unused-function -pthread
CXXFLAGS := -std=c++11 -O3 -fPIC -pthread -w
INCS := -Iref_build/stubs -I$(REF)/src -I$(REF)/submods -I$(REF)/submods/pdqsort

all: libunc_oracle_events.so ref

libunc_oracle_events.so: unc_oracle_events.c unc_oracle_events.h unc_oracle.c unc_oracle.h
	$(CC) $(CFLAGS) -shared -o $@ unc_oracle_events.c -lm

ref:
	@if [ -d $(REF)/src ]; then $(MAKE) -C ref_build REF=$(REF) && $(MAKE) -f events.mk _ref/libref_events.so; else echo "no reference tree: keeping prebuilt oracle/_ref"; fi

_ref/libref_events.so: ref_build/ref_events.cpp _ref/libuncalled_ref.so
	$(CXX) $(CXXFLAGS) -fvisibility=hidden $(INCS) -shared -o $@ ref_build/ref_events.cpp -L_ref -luncalled_ref -Wl,-rpath,'$$ORIGIN' -lz -lm

.PHONY: all ref
