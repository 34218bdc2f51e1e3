"""Repeat masking of a reference before `index`, the two steps of the reference's masking/README.md.  There is no
CPU path.

Iterative high-frequency k-mer masking (masking/mask_internal.sh) over `unc_mask_internal` (include/unc_b200.h):

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


def mask_external(full_fasta, target_fasta, min_len, min_copy, out_prefix, piece_bases=0):
    """Masks every min_len window of `target_fasta` that occurs more than `min_copy` times in `full_fasta`, counting
    exact matches on both strands (masking/mask_external.sh, over `unc_mask_external`).  Writes
    `<out_prefix>masked<min_copy>.fa` and `<out_prefix>reps_m<min_copy>.bed` and returns (masked_bp, intervals), the
    intervals being the BED lines as (name, start, end).  `piece_bases` bounds the full reference's share of device
    memory (0 = the library's default)."""
    d = os.path.dirname(out_prefix)
    if d and not os.path.isdir(d):
        raise N.UncError('directory "%s" does not exist' % d)
    out_fa = "%smasked%d.fa" % (out_prefix, int(min_copy))
    out_bed = "%sreps_m%d.bed" % (out_prefix, int(min_copy))
    n_sel, n_bp = C.c_uint64(), C.c_uint64()
    N.check(N.lib().unc_mask_external(os.fsencode(full_fasta), os.fsencode(target_fasta), int(min_len), int(min_copy),
                                      os.fsencode(out_fa), os.fsencode(out_bed), int(piece_bases), None,
                                      C.byref(n_sel), C.byref(n_bp)))
    with open(out_bed, "rb") as f:
        intervals = [(nm.decode(), int(a), int(b)) for nm, a, b in (ln.split(b"\t") for ln in f.read().splitlines())]
    return int(n_bp.value), intervals


def external_last_kernel_ms():
    """CUDA-event time of the last mask_external call's kernels"""
    return float(N.lib().unc_mask_external_last_kernel_ms())
