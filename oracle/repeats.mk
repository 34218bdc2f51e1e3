# oracle/repeats.mk -- the checker of `uncalled_b200 find-repeats` (test infrastructure only):
#   libunc_oracle_repeats.so   the C restatement (unc_oracle_repeats.c, which compiles unc_oracle.c into itself)
# The reference's own walk is its self_align, already in _ref/libuncalled_ref.so (oracle/Makefile).
# Same flags as oracle/Makefile.  make -C oracle -f repeats.mk
CC ?= gcc
CFLAGS := -O2 -ffp-contract=off -fPIC -Wall -Wno-unused-function -pthread

all: libunc_oracle_repeats.so

libunc_oracle_repeats.so: unc_oracle_repeats.c unc_oracle_repeats.h unc_oracle.c unc_oracle.h
	$(CC) $(CFLAGS) -shared -o $@ unc_oracle_repeats.c -lm

.PHONY: all
