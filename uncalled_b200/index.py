"""`uncalled index` (reference scripts/uncalled:38-78) on this package's native library: the bwa-compatible FM
index (`BwaIndex.create`, reference src/bwa_index.hpp:92-101 -> unc_index_build_device on a GPU machine,
unc_index_build otherwise), the sampled self-alignments
(`self_align`, reference src/self_align_ref.cpp:34-91, src/pybinder.cpp:59 -> unc_self_align on the GPU) and the
parameter search that turns them into the `.uncl` thresholds (index_params.py).  No CPU fallback: `self_align`
raises UncError without a usable CUDA device.

`BwaIndex(prefix, pacseq)` also answers the reference's index queries (src/bwa_index.hpp:103-333): the FM-index ones
(`sa`, `get_neighbor`, `range_to_fms`, `get_kmers`, the k-mer ranges) on the GPU through unc_bwa_*, the contig table
and `.pac` lookups on the host.  `Range` (src/range.cpp) and the k = 5 `kmer_*` helpers of src/bp.hpp are host code."""
import ctypes as C
import os
import sys

import numpy as np

from . import _native as N
from . import index_params as IP

BWA_SUFFS = [".amb", ".ann", ".bwt", ".pac", ".sa"]            # uncalled/index.py:33-40
UNCL_SUFF = ".uncl"


K = 5
_BASE_BYTES = {ord("A"): 0, ord("C"): 1, ord("G"): 2, ord("T"): 3, ord("a"): 0, ord("c"): 1, ord("g"): 2, ord("t"): 3}
_U64 = (1 << 64) - 1


def kmer_count():
    return 4 ** K


def str_to_kmer(kmer, offset=0):
    """src/bp.hpp str_to_kmer<5>: u16 arithmetic, a non-ACGT character ORs in 4 as the reference's table does"""
    b = kmer.encode() if isinstance(kmer, str) else bytes(kmer)
    index = _BASE_BYTES.get(b[offset], 4)
    for i in range(1, K):
        index = ((index << 2) | _BASE_BYTES.get(b[offset + i], 4)) & 0xFFFF
    return index


def kmer_comp(kmer):
    return (kmer ^ ((1 << 2 * K) - 1)) & 0xFFFF


def kmer_revcomp(kmer):
    """complement, then reverse the order of the five 2-bit bases (bits above the k-mer are dropped)"""
    x, r = (kmer ^ 0x3FF) & 0x3FF, 0
    for _ in range(K):
        r, x = (r << 2) | (x & 3), x >> 2
    return r


def kmer_head(kmer):
    return (kmer >> (2 * K - 2)) & 3


def kmer_neighbor(kmer, i):
    return (((kmer << 2) & ((1 << 2 * K) - 1)) | (i & 0xFF)) & 0xFFFF


def kmer_base(kmer, i):
    if not 0 <= i < K:
        raise ValueError("base index outside the k-mer")
    return (kmer >> (2 * (K - i - 1))) & 3


def kmer_to_str(kmer):
    return "".join("ACGT"[kmer_base(kmer, i)] for i in range(K))


class Range:
    """src/range.cpp: an FM-index row range [start, end], u64 arithmetic; Range() is the empty range (1, 0)"""
    __slots__ = ("start", "end")

    def __init__(self, start=1, end=0):
        self.start, self.end = int(start) & _U64, int(end) & _U64

    def __repr__(self):
        return "Range(%d, %d)" % (self.start, self.end)

    def length(self):
        return (self.end - self.start + 1) & _U64

    def is_valid(self):
        return self.start <= self.end

    def intersects(self, q):
        return (self.is_valid() and q.is_valid() and not (self.start > q.end or self.end < q.start)
                and not (q.start > self.end or q.end < self.start))

    def intersect(self, r):
        return Range(max(self.start, r.start), min(self.end, r.end)) if self.intersects(r) else Range()

    def merge(self, r):
        return Range(min(self.start, r.start), max(self.end, r.end)) if self.intersects(r) else Range()

    def get_recp_overlap(self, r):
        if not self.intersects(r):
            return 0.0
        f = np.float32
        return float(f(self.intersect(r).length()) / f(self.merge(r).length()))

    def split_range(self, r):
        """Range::split_range: returns the part left of r and keeps the part right of it (or the empty range)"""
        left = Range()
        if self.start < r.start:
            left = Range(self.start, (r.start - 1) & _U64)
        if self.start <= r.end:
            if self.end > r.end:
                self.start = (r.end + 1) & _U64
            else:
                self.start, self.end = 1, 0
        return left

    def same_range(self, q):
        return self.start == q.start and self.end == q.end

    def __eq__(self, q):
        return isinstance(q, Range) and self.same_range(q)

    def __lt__(self, q):
        return self.start < q.start or (self.start == q.start and self.end < q.end)

    def __hash__(self):
        return hash((self.start, self.end))


def _u64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.uint64).reshape(-1))


class BwaIndex:
    """The reference's BwaIndex<5> (src/bwa_index.hpp:88-377) over unc_bwa_*: the files are read on the host, and the
    first FM-index query builds the device image on `device`.  Array forms: `sa(rows)` and
    `get_neighbor(starts, ends, bases)` take and return numpy arrays; a scalar call is a batch of one."""

    def __init__(self, prefix="", pacseq=False, device=0):
        self._h = None
        self._kr = None
        self._device = int(device)
        if prefix:
            self.load_index(prefix)
        if pacseq:
            self.load_pacseq()

    def __del__(self):
        self.destroy()

    def load_index(self, prefix):
        self.destroy()
        h = C.c_void_p()
        N.check(N.lib().unc_bwa_open(os.fsencode(prefix), 0, self._device, C.byref(h)))
        self._h = h
        self._kr = None
        sl, lp, ns, pl = C.c_uint64(), C.c_uint64(), C.c_int32(), C.c_int32()
        L2 = (C.c_uint64 * 5)()
        N.check(N.lib().unc_bwa_info(h, C.byref(sl), C.byref(lp), C.byref(ns), C.byref(pl), L2))
        self._size, self._l_pac, self._L2 = sl.value, lp.value, list(L2)
        self._seqs = []
        for i in range(ns.value):
            nm, off, ln = C.c_char_p(), C.c_uint64(), C.c_uint64()
            N.check(N.lib().unc_bwa_seq(h, i, C.byref(nm), C.byref(off), C.byref(ln)))
            self._seqs.append((nm.value.decode(), off.value, ln.value))

    def is_loaded(self):
        return self._h is not None

    def _handle(self):
        if self._h is None:
            raise N.UncError("no index loaded")
        return self._h

    def load_pacseq(self):
        N.check(N.lib().unc_bwa_load_pac(self._handle()))

    def pacseq_loaded(self):
        if self._h is None:
            return False
        pl = C.c_int32()
        N.check(N.lib().unc_bwa_info(self._h, None, None, None, C.byref(pl), None))
        return bool(pl.value)

    def destroy(self):
        if getattr(self, "_h", None) is not None:
            N.lib().unc_bwa_free(self._h)
            self._h = None

    # ---- host: the contig table and the .pac
    def size(self):
        self._handle()
        return self._size

    def get_seqs(self):
        self._handle()
        return [(nm, ln) for nm, _, ln in self._seqs]

    def get_rid(self, sa_loc):
        return int(N.lib().unc_bwa_pos2rid(self._handle(), int(sa_loc)))

    def _ann(self, rid):
        if not 0 <= rid < len(self._seqs):
            raise IndexError("no contig %d" % rid)
        return self._seqs[rid]

    def get_ref_coord(self, sa_loc):
        rid = self.get_rid(sa_loc)
        return rid, (int(sa_loc) - self._ann(rid)[1]) & 0xFFFFFFFF

    def get_ref_name(self, rid):
        self._handle()
        return self._ann(rid)[0]

    def get_ref_len(self, rid):
        self._handle()
        return self._ann(rid)[2]

    def coord_to_pacseq(self, name, coord):
        out = C.c_uint64()
        N.check(N.lib().unc_bwa_coord_to_pacseq(self._handle(), name.encode(), int(coord) & _U64, C.byref(out)))
        return out.value

    def get_sa_loc(self, name, coord):
        self._handle()
        for nm, off, _ in self._seqs:
            if nm == name:
                return (off + int(coord)) & _U64
        return 0

    def translate_loc(self, sa_loc):
        """(ref_len, ref_name, ref_loc); ref_len 0 (and "", 0) when sa_loc lies in no contig"""
        rid = self.get_rid(sa_loc)
        if rid < 0:
            return 0, "", 0
        nm, off, ln = self._ann(rid)
        return ln, nm, (int(sa_loc) - off) & _U64

    def get_base(self, i):
        out = C.c_uint8()
        N.check(N.lib().unc_bwa_get_base(self._handle(), int(i), C.byref(out)))
        return out.value

    def get_base_range(self, base):
        self._handle()
        if not 0 <= base <= 3:
            raise ValueError("base outside 0..3")
        return Range(self._L2[base], self._L2[base + 1])

    # ---- device
    def _kmer_ranges(self):
        self._handle()
        if self._kr is None:
            st, en = np.zeros(1024, np.uint64), np.zeros(1024, np.uint64)
            N.check(N.lib().unc_bwa_kmer_ranges(self._handle(), st.ctypes.data, en.ctypes.data))
            self._kr = (st, en)
        return self._kr

    def get_kmer_range(self, kmer):
        st, en = self._kmer_ranges()
        return Range(int(st[kmer]), int(en[kmer]))

    def get_kmer_count(self, kmer):
        return self.get_kmer_range(kmer).length()

    def neighbors(self, starts, ends, bases):
        """get_neighbor for arrays: (starts, ends) as uint64 arrays"""
        st, en = _u64(starts), _u64(ends)
        b = np.ascontiguousarray(np.asarray(bases, dtype=np.uint8).reshape(-1))
        if not len(st) == len(en) == len(b):
            raise ValueError("starts, ends and bases differ in length")
        os_, oe = np.empty(len(st), np.uint64), np.empty(len(st), np.uint64)
        N.check(N.lib().unc_bwa_neighbor(self._handle(), len(st), st.ctypes.data, en.ctypes.data, b.ctypes.data,
                                         os_.ctypes.data, oe.ctypes.data))
        return os_, oe

    def get_neighbor(self, r, base, bases=None):
        """get_neighbor(Range, base) -> Range, or get_neighbor(starts, ends, bases) -> (starts, ends) arrays"""
        if bases is not None:
            return self.neighbors(r, base, bases)
        s, e = self.neighbors([r.start], [r.end], [base])
        return Range(int(s[0]), int(e[0]))

    def sa(self, rows):
        scalar = np.ndim(rows) == 0
        r = _u64(rows)
        out = np.empty(len(r), np.uint64)
        N.check(N.lib().unc_bwa_sa(self._handle(), len(r), r.ctypes.data, out.ctypes.data))
        return int(out[0]) if scalar else out

    def range_to_fms(self, ref_name, start, end):
        """(first, second) as the reference returns them: first = reverse-walk rows of positions pac_min .. pac_max,
        second = forward-walk rows of pac_max down to pac_min; uint64 arrays"""
        n = max(int(end) - int(start), 0)
        a, b = np.empty(max(n, 1), np.uint64), np.empty(max(n, 1), np.uint64)
        N.check(N.lib().unc_bwa_range_to_fms(self._handle(), ref_name.encode(), int(start) & _U64, int(end) & _U64,
                                             a.ctypes.data, b.ctypes.data))
        return a[:n], b[:n]

    def get_kmers(self, *args):
        """get_kmers(pac_st, pac_en) or get_kmers(name, st, en): the k-mers of bases [st, en) as a uint16 array"""
        if len(args) == 3:
            st, en = self.coord_to_pacseq(args[0], args[1]), self.coord_to_pacseq(args[0], args[2])
        else:
            st, en = (int(a) for a in args)
        n = max(en - st - 4, 0)
        out = np.empty(max(n, 1), np.uint16)
        N.check(N.lib().unc_bwa_get_kmers(self._handle(), st, en, out.ctypes.data))
        return out[:n]

    def last_kernel_ms(self):
        ms = C.c_float()
        N.check(N.lib().unc_bwa_last_kernel_ms(self._handle(), C.byref(ms)))
        return ms.value

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
