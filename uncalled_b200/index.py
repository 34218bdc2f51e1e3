"""`uncalled index` (reference scripts/uncalled:38-78) on this package's native library: the bwa-compatible FM
index (`BwaIndex.create`, reference src/bwa_index.hpp:92-101 -> unc_index_build_device on a GPU machine,
unc_index_build otherwise), the sampled self-alignments
(`self_align`, reference src/self_align_ref.cpp:34-91, src/pybinder.cpp:59 -> unc_self_align on the GPU) and the
parameter search that turns them into the `.uncl` thresholds (index_params.py).  No CPU fallback: `self_align`
raises UncError without a usable CUDA device."""
import ctypes as C
import os
import sys

import numpy as np

from . import _native as N
from . import index_params as IP

BWA_SUFFS = [".amb", ".ann", ".bwt", ".pac", ".sa"]            # uncalled/index.py:33-40
UNCL_SUFF = ".uncl"


class BwaIndex:
    @staticmethod
    def create(fasta_filename, bwa_prefix):
        """BwaIndex<K>::create (src/bwa_index.hpp:92-101): <prefix>.pac/.ann/.amb/.bwt/.sa as bwa writes them.  Built
        on the GPU (unc_index_build_device) when a CUDA device is visible, by the host builder otherwise: the files are
        the same, byte for byte."""
        L = N.lib()
        build = L.unc_index_build_device if L.unc_device_count() > 0 else L.unc_index_build
        N.check(build(os.fsencode(fasta_filename), os.fsencode(bwa_prefix)))


def self_align_csr(bwa_prefix, sample_dist):
    """unc_self_align: (offsets[n+1], values) -- path i holds values[offsets[i]:offsets[i+1]]."""
    L = N.lib()
    n, po, pv = C.c_uint64(), C.c_void_p(), C.c_void_p()
    N.check(L.unc_self_align(os.fsencode(bwa_prefix), int(sample_dist), C.byref(n), C.byref(po), C.byref(pv)))
    try:
        off = np.ctypeslib.as_array(C.cast(po, C.POINTER(C.c_uint64)), (n.value + 1,)).copy()
        nv = int(off[-1])
        val = np.ctypeslib.as_array(C.cast(pv, C.POINTER(C.c_uint64)), (max(nv, 1),)).copy()[:nv]
    finally:
        L.unc_free(po)
        L.unc_free(pv)
    return off, val


def self_align(bwa_prefix, sample_dist):
    """The reference's `_uncalled.self_align`: a list of lists of FM range lengths."""
    off, val = self_align_csr(bwa_prefix, sample_dist)
    v = val.tolist()
    return [v[int(off[i]):int(off[i + 1])] for i in range(len(off) - 1)]


def write_uncl(bwa_prefix, probs=None, speeds=None, self_align_fn=None, **opts):
    """IndexParameterizer(args) + add_preset(...) + write() (scripts/uncalled:57-76): writes <prefix>.uncl.
    `self_align_fn(prefix, sample_dist) -> (offsets, values)` replaces the GPU call in CPU-only tests."""
    o = dict(IP.DEFAULTS, **opts)
    sd = IP.sample_distance(IP.reference_length(bwa_prefix), o["max_sample_dist"], o["min_samples"], o["max_samples"])
    off, val = (self_align_fn or self_align_csr)(bwa_prefix, sd)
    text = IP.uncl_text(off, val, probs=probs, speeds=speeds, **opts)
    with open(bwa_prefix + UNCL_SUFF, "w") as f:
        f.write(text)
    return text


def index_cmd(fasta_filename, bwa_prefix=None, probs=None, speeds=None, self_align_fn=None, **opts):
    """`uncalled index [-o PREFIX] [--probs a,b] [--speeds c,d] FASTA` (scripts/uncalled:38-78): reuses an existing
    BWA index, builds it otherwise; then the parameter search.  `opts`: the remaining `uncalled index` options
    (max_sample_dist, min_samples, max_samples, kmer_len, matchpr1, matchpr2, pathlen_percentile, max_replen)."""
    if bwa_prefix is None:
        bwa_prefix = fasta_filename
    if all(os.path.exists(bwa_prefix + s) for s in BWA_SUFFS):
        sys.stderr.write("Using previously built BWA index.\nNote: to fully re-build the index delete files with "
                         "the \"%s.*\" prefix.\n" % bwa_prefix)
    else:
        BwaIndex.create(fasta_filename, bwa_prefix)
    sys.stderr.write("Initializing parameter search\n")
    write_uncl(bwa_prefix, probs=probs, speeds=speeds, self_align_fn=self_align_fn, **opts)
    sys.stderr.write("Done\n")
    return bwa_prefix
