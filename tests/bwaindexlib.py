"""Test support for the BwaIndex queries (uncalled_b200.index.BwaIndex, unc_bwa_*), never imported by the product.

- `FIXTURES` / `build`: the example index, a multi-contig index with N runs, a poly-A/T index, a self-reverse-complement
  record and a repeat-rich genome (tandem copies longer than the slop, so that anchor searches end on ranges of many
  rows), all indexed by the product's host builder (byte-identical to bwa);
- `emu()`: tests/emul/libunc_emul_bwa_index.so, the device code under the warp emulator;
- `orc()`: oracle/libunc_oracle_bwa_index.so, the serial C restatement;
- `spans`: the range_to_fms cases of an index: whole contigs, one-base spans, spans starting at 0 and ending at
  ref_len - 1, and spans across each contig join;
- `Ref`: the reference's own BwaIndex<k5> and k-mer helpers (oracle/_ref/libref_bwa_index.so, where it is built);
- `golden` / `golden_record`: tests/golden/bwa_index_golden.json, what the reference computed on the fixtures, written
  by tools/make_bwa_index_golden.py and read where oracle/_ref is not built."""
import ctypes as C
import os
import subprocess

import numpy as np

import fmsteplib
import orclib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
U64 = C.c_uint64
GOLDEN = os.path.join(ROOT, "tests", "golden", "bwa_index_golden.json")
REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libref_bwa_index.so")
SEGS = (3, 16, 512)


def fx_tandem(seed=45):
    """two records: 40 copies of a 37-base unit inside random flanks, and five copies of a 300-base block"""
    rng = np.random.default_rng(seed)
    r = lambda n: fmsteplib._rand(rng, n)
    unit, block = r(37), r(300)
    a = r(150) + unit * 40 + r(120)
    b = r(80) + b"".join(block + r(int(rng.integers(5, 30))) for _ in range(5)) + r(60)
    return fmsteplib._wrap(b"tandemA", a) + fmsteplib._wrap(b"tandemB", b)


FIXTURES = ("example", "multi_n", "poly", "palindrome", "tandem")


def build(name, d):
    """the index files of fixture `name` under directory d, without a .uncl; returns the prefix"""
    if name == "example":
        prefix = orclib.materialise_example_index(str(d))
    elif name == "tandem":
        from uncalled_b200 import _native as N
        prefix = os.path.join(str(d), name)
        if not os.path.exists(prefix + ".bwt"):
            open(prefix + ".fa", "wb").write(fx_tandem())
            assert N.lib().unc_index_build((prefix + ".fa").encode(), prefix.encode()) == 0
    else:
        prefix = fmsteplib.build(name, d)
    if os.path.exists(prefix + ".uncl"):
        os.remove(prefix + ".uncl")
    return prefix


def contigs(prefix):
    """[(name, offset, length)] from the .ann"""
    with open(prefix + ".ann") as f:
        n = int(f.readline().split()[1])
        out = []
        for _ in range(n):
            name = f.readline().split()[1]
            off, ln = (int(v) for v in f.readline().split()[:2])
            out.append((name, off, ln))
    return out


def spans(prefix):
    """(name, start, end) cases of range_to_fms"""
    cs = contigs(prefix)
    out = []
    for name, off, ln in cs:
        out += [(name, 0, ln), (name, 0, 1), (name, ln - 1, ln), (name, ln // 2, ln // 2 + 1), (name, 0, min(ln, 40)),
                (name, max(ln - 40, 0), ln), (name, ln // 3, ln // 3 + 97), (name, ln // 3, min(ln, ln // 3 + 300))]
    for (a, off, ln), _ in zip(cs, cs[1:]):                             # across the join into the next contig
        out.append((a, max(ln - 30, 0), ln + 30))
    offs, l_pac = {n: o for n, o, _ in cs}, sum(c[2] for c in cs)
    return [s for s in out if s[2] > s[1] and offs[s[0]] + s[2] <= l_pac]


def uncalled_module():
    """the `_uncalled` extension module, imported under that top-level name as the reference's package imports it"""
    import sys
    from uncalled_b200 import _native as N
    N.build_pymodule()
    if N.PKG_DIR not in sys.path:
        sys.path.insert(0, N.PKG_DIR)
    import _uncalled
    return _uncalled


def pac(prefix):
    return np.fromfile(prefix + ".pac", np.uint8)


def pac_bases(prefix, st, en):
    p = pac(prefix)
    i = np.arange(st, en, dtype=np.int64)
    return (p[i >> 2] >> ((3 - (i & 3)) * 2)) & 3


def seq_to_kmers(prefix, st, en):
    """src/bp.hpp seq_to_kmers<5> over the .pac, restated in numpy"""
    if en <= st + 4:
        return np.zeros(0, np.uint16)
    b = pac_bases(prefix, st, en).astype(np.uint16)
    k = np.zeros(len(b) - 4, np.uint16)
    for j in range(5):
        k = (k << 2) | b[j:len(b) - 4 + j]
    return k


_emu = None


def emu():
    global _emu
    if _emu is None:
        src = os.path.join(EMUL_DIR, "emul_bwa_index.cpp")
        out = os.path.join(EMUL_DIR, "libunc_emul_bwa_index.so")
        csrc = os.path.join(ROOT, "uncalled_b200", "csrc")
        deps = [src, os.path.join(EMUL_DIR, "warp_emul.hpp")] + [os.path.join(csrc, f) for f in (
            "unc_bwa.cuh", "unc_selfalign.cuh", "unc_device.cuh", "unc_host_index.hpp")]
        if not (os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(x) for x in deps)):
            subprocess.run(["g++", "-O2", "-g", "-std=c++17", "-ffp-contract=off", "-DUNC_EMUL", "-DK2_MAXSEG=16u", "-fPIC",
                            "-shared", "-I" + EMUL_DIR, "-I" + csrc, "-o", out, src], check=True, capture_output=True)
        L = C.CDLL(out)
        L.emu_bwa_neighbor.argtypes = [C.c_char_p, U64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.emu_bwa_sa.argtypes = [C.c_char_p, U64, C.c_void_p, C.c_void_p]
        L.emu_bwa_range_to_fms.argtypes = [C.c_char_p, U64, U64, C.c_uint32, C.c_void_p, C.c_void_p]
        _emu = L
    return _emu


_orc = None


def orc():
    global _orc
    if _orc is None:
        path = os.path.join(ORACLE_DIR, "libunc_oracle_bwa_index.so")
        if not os.path.exists(path):
            subprocess.run(["make", "-C", ORACLE_DIR, "-f", "bwa_index.mk"], check=True, capture_output=True)
        L = C.CDLL(path)
        L.orc_index_load.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]
        L.orc_index_free.argtypes = [C.c_void_p]
        L.orc_sa.argtypes = [C.c_void_p, U64]
        L.orc_sa.restype = U64
        L.orc_bwa_neighbors.argtypes = [C.c_void_p, U64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_range_to_fms.argtypes = [C.c_void_p, C.c_void_p, U64, U64, C.c_void_p, C.c_void_p]
        _orc = L
    return _orc


class Restated:
    """the C restatement over one index"""

    def __init__(self, prefix):
        self.prefix = prefix
        self.L = orc()
        self.idx = C.c_void_p()
        assert self.L.orc_index_load(prefix.encode(), b"-", C.byref(self.idx)) == 0
        self.pac = pac(prefix)
        self.contigs = {n: o for n, o, _ in contigs(prefix)}
        self.size = int(np.fromfile(prefix + ".bwt", np.uint64, 5)[4])

    def __del__(self):
        self.L.orc_index_free(self.idx)

    def sa(self, rows):
        return np.array([self.L.orc_sa(self.idx, int(r)) for r in rows], np.uint64)

    def neighbors(self, st, en, base):
        st, en = np.ascontiguousarray(st, np.uint64), np.ascontiguousarray(en, np.uint64)
        base = np.ascontiguousarray(base, np.uint8)
        os_, oe = np.empty(len(st), np.uint64), np.empty(len(st), np.uint64)
        self.L.orc_bwa_neighbors(self.idx, len(st), st.ctypes.data, en.ctypes.data, base.ctypes.data, os_.ctypes.data,
                                 oe.ctypes.data)
        return os_, oe

    def range_to_fms(self, name, start, end):
        n = end - start
        a, b = np.empty(n, np.uint64), np.empty(n, np.uint64)
        self.L.orc_range_to_fms(self.idx, self.pac.ctypes.data, self.contigs[name] + start, n, a.ctypes.data, b.ctypes.data)
        return a, b


def emu_sa(prefix, rows):
    rows = np.ascontiguousarray(rows, np.uint64)
    out = np.empty(len(rows), np.uint64)
    assert emu().emu_bwa_sa(prefix.encode(), len(rows), rows.ctypes.data, out.ctypes.data) == 0
    return out


def emu_neighbors(prefix, st, en, base):
    st, en = np.ascontiguousarray(st, np.uint64), np.ascontiguousarray(en, np.uint64)
    base = np.ascontiguousarray(base, np.uint8)
    os_, oe = np.empty(len(st), np.uint64), np.empty(len(st), np.uint64)
    assert emu().emu_bwa_neighbor(prefix.encode(), len(st), st.ctypes.data, en.ctypes.data, base.ctypes.data,
                                  os_.ctypes.data, oe.ctypes.data) == 0
    return os_, oe


def emu_range_to_fms(prefix, pac_min, n, seg):
    a, b = np.empty(n, np.uint64), np.empty(n, np.uint64)
    rc = emu().emu_bwa_range_to_fms(prefix.encode(), pac_min, n, seg, a.ctypes.data, b.ctypes.data)
    assert rc == 0, rc
    return a, b


def neighbor_queries(size, rng):
    """every row as start and as end with the four bases, plus start 0, start size + 1 and inverted ranges"""
    rows = np.arange(size + 1, dtype=np.uint64)
    st = np.concatenate([rows, rows + 1, np.zeros(64, np.uint64), rows[rng.integers(0, size + 1, 4 * size)] + 0])
    en = np.concatenate([np.minimum(rows + rng.integers(0, 200, size + 1).astype(np.uint64), size), rows,
                         rng.integers(0, size + 1, 64).astype(np.uint64), rows[rng.integers(0, size + 1, 4 * size)]])
    st, en = np.repeat(st, 4), np.repeat(en, 4)
    base = np.tile(np.arange(4, dtype=np.uint8), len(st) // 4)
    return st, en, base


def kmer_spans(prefix):
    """(pac_st, pac_en) cases of get_kmers: whole contigs, fewer than five bases, exactly five, across each join"""
    cs = contigs(prefix)
    out = []
    for name, off, ln in cs:
        out += [(off, off + ln), (off, off + min(ln, 4)), (off + 3, off + min(ln, 8)), (off + ln - 5, off + ln)]
    for (_, off, ln), _ in zip(cs, cs[1:]):
        out.append((off + ln - 20, off + ln + 20))
    return out


def edge_locs(prefix):
    """translate_loc cases: both ends of every contig, the middle, and l_pac itself (no contig)"""
    cs = contigs(prefix)
    out = []
    for _, off, ln in cs:
        out += [off, off + ln // 2, off + ln - 1]
    return out + [cs[-1][1] + cs[-1][2]]


class Ref:
    """the reference's own BwaIndex<k5>(prefix, true), through oracle/_ref/libref_bwa_index.so"""
    _lib = None

    @classmethod
    def available(cls):
        return os.path.exists(REF_LIB)

    @classmethod
    def lib(cls):
        if cls._lib is None:
            L = C.CDLL(REF_LIB)
            vp = C.c_void_p
            L.ref_bwa_open.argtypes, L.ref_bwa_open.restype = [C.c_char_p], vp
            L.ref_bwa_free.argtypes = [vp]
            L.ref_bwa_size.argtypes, L.ref_bwa_size.restype = [vp], U64
            L.ref_bwa_sa.argtypes = [vp, U64, vp, vp]
            L.ref_bwa_neighbor.argtypes = [vp, U64, vp, vp, vp, vp, vp]
            L.ref_bwa_kmer_ranges.argtypes = [vp, vp, vp]
            L.ref_bwa_range_to_fms.argtypes = [vp, C.c_char_p, U64, U64, vp, vp]
            L.ref_bwa_get_kmers.argtypes, L.ref_bwa_get_kmers.restype = [vp, U64, U64, vp, vp], U64
            L.ref_bwa_translate_loc.argtypes, L.ref_bwa_translate_loc.restype = [vp, U64, C.c_char_p, U64, C.POINTER(U64)], U64
            L.ref_kmer_helpers.argtypes = [vp] * 7
            L.ref_str_to_kmer.argtypes, L.ref_str_to_kmer.restype = [C.c_char_p, U64], C.c_uint16
            L.ref_kmer_count.restype = C.c_uint16
            cls._lib = L
        return cls._lib

    def __init__(self, prefix):
        self.L = self.lib()
        self.h = self.L.ref_bwa_open(prefix.encode())
        self.size = int(self.L.ref_bwa_size(self.h))

    def __del__(self):
        self.L.ref_bwa_free(self.h)

    def sa(self, rows):
        rows = np.ascontiguousarray(rows, np.uint64)
        out = np.empty(len(rows), np.uint64)
        self.L.ref_bwa_sa(self.h, len(rows), rows.ctypes.data, out.ctypes.data)
        return out

    def neighbors(self, st, en, base):
        st, en = np.ascontiguousarray(st, np.uint64), np.ascontiguousarray(en, np.uint64)
        base = np.ascontiguousarray(base, np.uint8)
        os_, oe = np.empty(len(st), np.uint64), np.empty(len(st), np.uint64)
        self.L.ref_bwa_neighbor(self.h, len(st), st.ctypes.data, en.ctypes.data, base.ctypes.data, os_.ctypes.data,
                                oe.ctypes.data)
        return os_, oe

    def kmer_ranges(self):
        st, en = np.empty(1024, np.uint64), np.empty(1024, np.uint64)
        self.L.ref_bwa_kmer_ranges(self.h, st.ctypes.data, en.ctypes.data)
        return st, en

    def range_to_fms(self, name, start, end):
        a, b = np.empty(end - start, np.uint64), np.empty(end - start, np.uint64)
        self.L.ref_bwa_range_to_fms(self.h, name.encode(), start, end, a.ctypes.data, b.ctypes.data)
        return a, b

    def get_kmers(self, st, en):
        n = max(en - st - 4, 0)
        a, b = np.empty(max(n, 1), np.uint16), np.empty(max(n, 1), np.uint16)
        assert self.L.ref_bwa_get_kmers(self.h, st, en, a.ctypes.data, b.ctypes.data) == n
        return a[:n], b[:n]

    def translate_loc(self, sa_loc):
        name, loc = C.create_string_buffer(8192), U64()
        ln = int(self.L.ref_bwa_translate_loc(self.h, sa_loc, name, 8192, C.byref(loc)))
        return (ln, name.value.decode(), loc.value) if ln else (0, "", 0)

    @classmethod
    def kmer_helpers(cls):
        """{name: array} over the 1024 k-mers"""
        o = dict(comp=np.empty(1024, np.uint16), revcomp=np.empty(1024, np.uint16), head=np.empty(1024, np.uint8),
                 base=np.empty(5 * 1024, np.uint8), neighbor=np.empty(4 * 1024, np.uint16),
                 roundtrip=np.empty(1024, np.uint16), str=np.zeros(6 * 1024, np.uint8))
        cls.lib().ref_kmer_helpers(*(o[k].ctypes.data for k in ("comp", "revcomp", "head", "base", "neighbor", "roundtrip",
                                                                 "str")))
        return o


def golden_record(prefix, X):
    """what golden holds for one fixture, computed by X (Ref, Restated-like or an emulated / GPU wrapper with sa,
    neighbors, range_to_fms; get_kmers and translate_loc when it has them)"""
    from orclib import digest
    size = X.size
    rec = {"size": size, "sa": digest(X.sa(np.arange(size + 1, dtype=np.uint64)))}
    st, en, base = neighbor_queries(size, np.random.default_rng(7))
    rec["neighbor"] = digest(*X.neighbors(st, en, base))
    rec["fms"] = [[n, a, b, digest(*X.range_to_fms(n, a, b))] for n, a, b in spans(prefix)]
    if hasattr(X, "get_kmers"):
        rec["kmers"] = [[a, b, digest(*X.get_kmers(a, b))] for a, b in kmer_spans(prefix)]
    if hasattr(X, "translate_loc"):
        rec["translate_loc"] = [[p] + list(X.translate_loc(p)) for p in edge_locs(prefix)]
    return rec


def golden():
    import json
    return json.load(open(GOLDEN))
