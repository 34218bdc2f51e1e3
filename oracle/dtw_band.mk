# oracle/dtw_band.mk -- the checker of the banded DTW sweep (test infrastructure only):
#   libunc_oracle_dtw_band.so   the C restatement (unc_oracle_dtw_band.c), over libunc_oracle.so
# Same flags as oracle/Makefile.  make -C oracle -f dtw_band.mk
CC ?= gcc
CFLAGS := -O2 -ffp-contract=off -fPIC -Wall -Wno-unused-function -pthread

all: libunc_oracle_dtw_band.so

libunc_oracle.so: unc_oracle.c unc_oracle.h
	$(MAKE) libunc_oracle.so

libunc_oracle_dtw_band.so: unc_oracle_dtw_band.c unc_oracle.h libunc_oracle.so
	$(CC) $(CFLAGS) -shared -o $@ unc_oracle_dtw_band.c -L. -lunc_oracle -Wl,-rpath,'$$ORIGIN' -lm

.PHONY: all
