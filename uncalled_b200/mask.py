"""Iterative high-frequency k-mer masking of a reference (the reference's masking/mask_internal.sh) over
`unc_mask_internal` (include/unc_b200.h).  There is no CPU path.

    mask_internal("ref.fa", 10, 30, "out/ref_")   # writes out/ref_mask30.fa, returns [(kmer, count), ...]

Each iteration masks every occurrence of the most frequent k-mer (forward strand, bases case-insensitive) with N;
the counts are recomputed after each masking, because masking one k-mer changes the counts of those overlapping it.
Where two k-mers share the highest count the lexicographically smallest is masked (the shell script takes
jellyfish's hash order).  With a unique maximum in every iteration the output is byte-identical to the script's."""
import ctypes as C
import os
import sys

import numpy as np

from . import _native as N


def kmer_str(code, k):
    """the k-mer of a 2-bit code, first base in the top bits"""
    return "".join("ACGT"[(int(code) >> (2 * (k - 1 - i))) & 3] for i in range(k))


def mask_internal(fasta, k, iters, out_prefix, log=True):
    """Masks `iters` iterations of k-mers of `fasta` into `<out_prefix>mask<iters>.fa` and returns the masked k-mers
    with their counts.  The list is shorter than `iters` when no k-mer was left to mask.  `log` gets the script's
    line per iteration: True for sys.stderr, a text stream, or None for none."""
    d = os.path.dirname(out_prefix)
    if d and not os.path.isdir(d):
        raise N.UncError('directory "%s" does not exist' % d)
    iters = int(iters)
    out = "%smask%d.fa" % (out_prefix, iters)
    codes = np.zeros(max(iters, 1), np.uint64)
    counts = np.zeros(max(iters, 1), np.uint64)
    done = C.c_uint32()
    N.check(N.lib().unc_mask_internal(os.fsencode(fasta), os.fsencode(out), int(k), iters, codes.ctypes.data,
                                      counts.ctypes.data, C.byref(done)))
    res = [(kmer_str(codes[i], k), int(counts[i])) for i in range(done.value)]
    if log is True:
        log = sys.stderr
    if log:
        for i, (km, n) in enumerate(res):
            log.write("Iteration %d: masked %d occurences of %s\n" % (i, n, km))
        log.flush()
    return res


def last_kernel_ms():
    """CUDA-event time of the last mask_internal call's device loop"""
    return float(N.lib().unc_mask_last_kernel_ms())
