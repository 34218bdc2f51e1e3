"""BwaIndex queries on the CPU: the device code of unc_bwa.cuh under the warp emulator against the serial C
restatement of the reference's loops (oracle/unc_oracle_bwa_index.c); the host half of uncalled_b200.index.BwaIndex
and of `_uncalled.BwaIndex` (contig table, argument checks made before the device is touched); Range and the k-mer
helpers."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import bwaindexlib as B
from uncalled_b200 import _native as N
from uncalled_b200 import index as I

REF_BWA_INDEX = "/root/reference/src/bwa_index.hpp"


@pytest.fixture(scope="module", params=B.FIXTURES)
def fixture(request, tmp_path_factory):
    return B.build(request.param, tmp_path_factory.mktemp(request.param))


def test_sa_every_row(fixture):
    R = B.Restated(fixture)
    rows = np.arange(R.size + 1, dtype=np.uint64)
    got = B.emu_sa(fixture, rows)
    assert got[0] == np.uint64(2**64 - 1)
    assert np.array_equal(got, R.sa(rows))
    assert np.array_equal(np.sort(got[1:]), np.arange(R.size, dtype=np.uint64))     # a permutation of the text


def test_neighbor_every_row_and_inverted_ranges(fixture):
    R = B.Restated(fixture)
    st, en, base = B.neighbor_queries(R.size, np.random.default_rng(7))
    got = B.emu_neighbors(fixture, st, en, base)
    want = R.neighbors(st, en, base)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert (st > en).sum() > 1000                                    # inverted ranges were among the queries


@pytest.mark.parametrize("seg", [3, 16, 512])
def test_range_to_fms_segments_match_the_serial_walk(fixture, seg):
    R = B.Restated(fixture)
    offs = {n: o for n, o, _ in B.contigs(fixture)}
    for name, st, en in B.spans(fixture):
        want = R.range_to_fms(name, st, en)
        got = B.emu_range_to_fms(fixture, offs[name] + st, en - st, seg)
        assert np.array_equal(got[0], want[0]), (name, st, en, seg, "first (reverse walk)")
        assert np.array_equal(got[1], want[1]), (name, st, en, seg, "second (forward walk)")


class Emulated:
    """the device code under the warp emulator, at `seg` positions per range_to_fms segment"""

    def __init__(self, prefix, seg):
        self.prefix, self.seg = prefix, seg
        self.size = int(np.fromfile(prefix + ".bwt", np.uint64, 5)[4])
        self.offs = {n: o for n, o, _ in B.contigs(prefix)}

    def sa(self, rows):
        return B.emu_sa(self.prefix, rows)

    def neighbors(self, st, en, base):
        return B.emu_neighbors(self.prefix, st, en, base)

    def range_to_fms(self, name, start, end):
        return B.emu_range_to_fms(self.prefix, self.offs[name] + start, end - start, self.seg)


def _fixture_name(prefix):
    return [n for n in B.FIXTURES if os.path.basename(prefix) == n or (n == "example" and "example" in prefix)][0]


def _check_against_golden(prefix, X, keys):
    want = B.golden()["fixtures"][_fixture_name(prefix)]
    got = B.golden_record(prefix, X)
    for k in keys:
        assert got[k] == want[k], (prefix, k)


def test_restatement_matches_the_golden(fixture):
    """the C restatement of the reference's loops against what the reference's own BwaIndex computed"""
    _check_against_golden(fixture, B.Restated(fixture), ("size", "sa", "neighbor", "fms"))


@pytest.mark.parametrize("seg", B.SEGS)
def test_emulated_kernels_match_the_golden(fixture, seg):
    """sa of every row, every row's neighbours (start 0, start size() + 1, inverted ranges) and every range_to_fms span,
    from the device code at segment lengths down to 3, against the reference's results"""
    keys = ("size", "sa", "neighbor", "fms") if seg == B.SEGS[0] else ("size", "fms")
    _check_against_golden(fixture, Emulated(fixture, seg), keys)


def test_golden_queries_cover_inverted_ranges_and_the_reverse_anchor_match():
    import tempfile
    d = tempfile.mkdtemp()
    prefix = B.build("poly", d)
    st, en, _ = B.neighbor_queries(B.Restated(prefix).size, np.random.default_rng(7))
    assert (st > en).sum() > 1000
    name, off, ln = B.contigs(prefix)[0]
    bases = B.pac_bases(prefix, off, off + ln)
    assert (bases[200:500] == 0).all()                                    # fmsteplib.fx_poly: 200 random, then 300 A
    assert any(a > 216 and a < 500 and b > 500 for n, a, b in B.spans(prefix))   # starts after > slop + 1 A, leaves the run


@pytest.mark.skipif(not B.Ref.available(), reason="oracle/_ref/libref_bwa_index.so is not built")
def test_reference_live_on_random_rows_and_spans(fixture):
    """the reference's own BwaIndex, live: random rows' sa and neighbours, random spans' range_to_fms, get_kmers,
    translate_loc and the k-mer ranges, against the emulated kernels and the host queries"""
    rng = np.random.default_rng(11)
    Rf = B.Ref(fixture)
    rows = rng.integers(0, Rf.size + 1, 3000).astype(np.uint64)
    assert np.array_equal(B.emu_sa(fixture, rows), Rf.sa(rows))
    st, en = rng.integers(0, Rf.size + 2, 3000).astype(np.uint64), rng.integers(0, Rf.size + 1, 3000).astype(np.uint64)
    base = rng.integers(0, 4, 3000).astype(np.uint8)
    got, want = B.emu_neighbors(fixture, st, en, base), Rf.neighbors(st, en, base)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    cs = B.contigs(fixture)
    l_pac = cs[-1][1] + cs[-1][2]
    for _ in range(25):
        name, off, ln = cs[int(rng.integers(0, len(cs)))]
        a = int(rng.integers(0, ln))
        b = int(min(l_pac - off, a + rng.integers(1, 400)))
        got, want = B.emu_range_to_fms(fixture, off + a, b - a, int(rng.integers(2, 64))), Rf.range_to_fms(name, a, b)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (name, a, b)
        k = Rf.get_kmers(off + a, off + b)
        assert np.array_equal(k[0], B.seq_to_kmers(fixture, off + a, off + b))
        assert np.array_equal(k[1], np.array([I.kmer_revcomp(int(x)) for x in k[0][::-1]], np.uint16))
    X = I.BwaIndex(fixture, True)
    for p in B.edge_locs(fixture) + [int(v) for v in rng.integers(0, l_pac + 2, 50)]:
        assert tuple(X.translate_loc(p)) == Rf.translate_loc(p), p


def test_host_queries_match_the_golden(fixture):
    """translate_loc at contig edges from the host table, and seq_to_kmers restated, against the reference's results"""
    from orclib import digest
    want = B.golden()["fixtures"][_fixture_name(fixture)]
    X = I.BwaIndex(fixture, True)
    assert [[p] + list(X.translate_loc(p)) for p in B.edge_locs(fixture)] == want["translate_loc"]
    got = []
    for a, b in B.kmer_spans(fixture):
        k = B.seq_to_kmers(fixture, a, b)
        got.append([a, b, digest(k, np.array([I.kmer_revcomp(int(x)) for x in k[::-1]], np.uint16))])
    assert got == want["kmers"]


def test_forward_list_is_the_inverse_suffix_array(fixture):
    """range_to_fms's second list over a whole contig: row of position p is the row whose SA value is p"""
    R = B.Restated(fixture)
    sa = B.emu_sa(fixture, np.arange(R.size + 1, dtype=np.uint64))
    isa = np.empty(R.size + 1, np.uint64)
    isa[sa[1:].astype(np.int64)] = np.arange(1, R.size + 1, dtype=np.uint64)
    name, off, ln = B.contigs(fixture)[0]
    _, second = B.emu_range_to_fms(fixture, off, ln, 16)
    assert np.array_equal(second, isa[np.arange(off + ln - 1, off - 1, -1)])


def test_reverse_anchor_the_reference_matches():
    """pac_min at the end of a poly-A run of more than slop + 1 bases: the reference's reverse scan matches the suffix
    one position off, and its walk leaves the exact chain for the rest of the span"""
    import tempfile
    d = tempfile.mkdtemp()
    prefix = B.build("poly", d)
    R = B.Restated(prefix)
    name, off, ln = B.contigs(prefix)[0]
    bases = B.pac_bases(prefix, off, off + ln)
    a_end = 200 + 300                                                   # fmsteplib.fx_poly: 200 random, 300 A
    assert (bases[200:a_end] == 0).all()
    for st in (a_end - 1, a_end - 2, 230):
        want = R.range_to_fms(name, st, st + 120)
        got = B.emu_range_to_fms(prefix, off + st, 120, 8)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def _open(prefix, pac=True):
    h = C.c_void_p()
    assert N.lib().unc_bwa_open(prefix.encode(), int(pac), 0, C.byref(h)) == 0, N.lib().unc_last_error()
    return h


def test_undefined_arguments_fail_before_the_device(fixture):
    """every argument the reference leaves undefined is an error from the host checks, on a machine with no GPU too"""
    L = N.lib()
    cs = B.contigs(fixture)
    name, off, ln = cs[-1]
    l_pac = off + ln
    size = 2 * l_pac
    h = _open(fixture)
    a, b = np.empty(l_pac + 8, np.uint64), np.empty(l_pac + 8, np.uint64)
    try:
        for nm, st, en in [("no-such-contig", 0, 10), (name, 10, 10), (name, 10, 5), (name, ln - 5, ln + 1),
                           (name, ln, ln + 1)]:
            assert L.unc_bwa_range_to_fms(h, nm.encode(), st, en, a.ctypes.data, b.ctypes.data) == -1, (nm, st, en)
        rows = np.array([size + 1], np.uint64)
        assert L.unc_bwa_sa(h, 1, rows.ctypes.data, a.ctypes.data) == -1
        for st, en, base in [(size + 2, 0, 0), (0, size + 1, 0), (1, 1, 4)]:
            s, e, bb = (np.array([v], t) for v, t in ((st, np.uint64), (en, np.uint64), (base, np.uint8)))
            assert L.unc_bwa_neighbor(h, 1, s.ctypes.data, e.ctypes.data, bb.ctypes.data, a.ctypes.data, b.ctypes.data) == -1
        assert L.unc_bwa_get_kmers(h, 0, l_pac + 1, a.ctypes.data) == -1
        u8 = C.c_uint8()
        assert L.unc_bwa_get_base(h, l_pac, C.byref(u8)) == -1
    finally:
        L.unc_bwa_free(h)
    h = _open(fixture, pac=False)                                     # no .pac: range_to_fms, get_kmers, get_base
    try:
        assert L.unc_bwa_range_to_fms(h, name.encode(), 0, 1, a.ctypes.data, b.ctypes.data) == -1
        assert L.unc_bwa_get_kmers(h, 0, 10, a.ctypes.data) == -1
        assert L.unc_bwa_load_pac(h) == 0
    finally:
        L.unc_bwa_free(h)
    if L.unc_device_count() == 0:                                    # a valid query reaches the device step
        h = _open(fixture)
        try:
            assert L.unc_bwa_range_to_fms(h, name.encode(), 0, 1, a.ctypes.data, b.ctypes.data) == -4
        finally:
            L.unc_bwa_free(h)


def test_open_reports_missing_and_inconsistent_files(tmp_path):
    src = B.build("multi_n", tmp_path)
    h = C.c_void_p()
    for suff in (".bwt", ".sa", ".ann", ".amb"):
        p = str(tmp_path / ("miss" + suff.strip(".")))
        for s in (".bwt", ".sa", ".ann", ".amb", ".pac"):
            if s != suff:
                os.link(src + s, p + s)
        assert N.lib().unc_bwa_open(p.encode(), 0, 0, C.byref(h)) == -2, suff
    p = str(tmp_path / "badamb")
    for s in (".bwt", ".sa", ".ann", ".pac"):
        os.link(src + s, p + s)
    open(p + ".amb", "w").write("12 1 0\n")
    assert N.lib().unc_bwa_open(p.encode(), 0, 0, C.byref(h)) == -2
    p = str(tmp_path / "nopac")
    for s in (".bwt", ".sa", ".ann", ".amb"):
        os.link(src + s, p + s)
    assert N.lib().unc_bwa_open(p.encode(), 1, 0, C.byref(h)) == -2
    assert N.lib().unc_bwa_open(p.encode(), 0, 0, C.byref(h)) == 0
    N.lib().unc_bwa_free(h)


def test_host_queries(fixture):
    """contig table, translate_loc at contig edges, coord_to_pacseq, get_base, get_base_range: index.BwaIndex and
    _uncalled.BwaIndex against the .ann / .pac"""
    U = B.uncalled_module()
    cs = B.contigs(fixture)
    l_pac = cs[-1][1] + cs[-1][2]
    bases = B.pac_bases(fixture, 0, l_pac)
    L2 = [0] + [int(v) for v in np.fromfile(fixture + ".bwt", np.uint64, 5)[1:5]]
    for X in (I.BwaIndex(fixture, True), U.BwaIndex(fixture, True)):
        assert X.is_loaded() and X.pacseq_loaded()
        assert X.size() == 2 * l_pac
        assert [tuple(s) for s in X.get_seqs()] == [(n, ln) for n, _, ln in cs]
        for rid, (name, off, ln) in enumerate(cs):
            assert X.get_ref_name(rid) == name and X.get_ref_len(rid) == ln
            assert X.coord_to_pacseq(name, 7) == off + 7 and X.get_sa_loc(name, 7) == off + 7
            for p in (off, off + ln - 1, off + ln // 2):
                assert X.get_rid(p) == rid
                assert tuple(X.translate_loc(p)) == (ln, name, p - off)
                assert tuple(X.get_ref_coord(p)) == (rid, p - off)
        assert X.coord_to_pacseq("no-such-contig", 3) == 2**31 - 1 and X.get_sa_loc("no-such-contig", 3) == 0
        assert X.get_rid(l_pac) == -1 and tuple(X.translate_loc(l_pac))[0] == 0
        for i in list(range(0, l_pac, 97)) + [l_pac - 1]:
            assert X.get_base(i) == bases[i]
        for b in range(4):
            r = X.get_base_range(b)
            assert (r.start, r.end) == (L2[b], L2[b + 1])
        X.destroy()
        assert not X.is_loaded()


def test_python_index_opens_without_pac_and_loads_it(fixture):
    X = I.BwaIndex(fixture)
    assert X.is_loaded() and not X.pacseq_loaded()
    X.load_pacseq()
    assert X.pacseq_loaded()
    empty = I.BwaIndex()
    assert not empty.is_loaded()
    for call in (lambda: empty.get_kmer_range(0), lambda: empty.sa(1), lambda: empty.get_base_range(0)):
        with pytest.raises(N.UncError):
            call()
    for b in (-1, 4):
        with pytest.raises(ValueError):
            X.get_base_range(b)


def _reference_method_names():
    src = open(REF_BWA_INDEX).read()
    body = src[src.index("static void pybind_defs"):src.index("#endif", src.index("static void pybind_defs"))]
    return sorted(set(re.findall(r"PY_BWA_INDEX_METH\((\w+)\)", body)) | set(re.findall(r'c\.def\("(\w+)"', body)))


@pytest.mark.skipif(not os.path.exists(REF_BWA_INDEX), reason="the reference tree is not here")
def test_uncalled_binds_the_reference_method_list():
    U = B.uncalled_module()
    names = _reference_method_names()
    assert len(names) == 23
    ours = sorted(n for n in dir(U.BwaIndex) if not n.startswith("_"))
    assert ours == names
    assert all(hasattr(I.BwaIndex, n) for n in names)


def _kmer_helpers_restated():
    """src/bp.hpp's helpers for k = 5, written out from their definitions"""
    comp = {0: 3, 1: 2, 2: 1, 3: 0}
    out = {}
    for k in range(1024):
        b = [(k >> (2 * (4 - i))) & 3 for i in range(5)]
        rc = 0
        for x in reversed(b):
            rc = (rc << 2) | comp[x]
        out[k] = dict(comp=k ^ 0x3FF, revcomp=rc, head=b[0], bases=b, s="".join("ACGT"[x] for x in b),
                      nb=[((k << 2) & 0x3FF) | i for i in range(4)])
    return out


def _helper_arrays(M):
    """the k-mer helpers of module M over the 1024 k-mers, laid out as oracle/_ref's ref_kmer_helpers writes them"""
    ks = range(1024)
    return dict(comp=np.array([M.kmer_comp(k) for k in ks], np.uint16),
                revcomp=np.array([M.kmer_revcomp(k) for k in ks], np.uint16),
                head=np.array([M.kmer_head(k) for k in ks], np.uint8),
                base=np.array([M.kmer_base(k, i) for k in ks for i in range(5)], np.uint8),
                neighbor=np.array([M.kmer_neighbor(k, b) for k in ks for b in range(4)], np.uint16),
                roundtrip=np.array([M.str_to_kmer(M.kmer_to_str(k)) for k in ks], np.uint16),
                str=np.frombuffer(b"".join(M.kmer_to_str(k).encode() + b"\0" for k in ks), np.uint8))


def test_kmer_helpers_for_every_kmer():
    """index.py's and _uncalled's helpers against the reference's bp.hpp: its digest in the golden, and live where
    oracle/_ref is built; plus restated definitions and strings with non-ACGT characters"""
    from orclib import digest
    U = B.uncalled_module()
    want = _kmer_helpers_restated()
    gold = B.golden()["kmer_helpers"]
    for M in (I, U):
        assert M.kmer_count() == 1024
        h = _helper_arrays(M)
        assert digest(*(h[k] for k in sorted(h))) == gold
        if B.Ref.available():
            r = B.Ref.kmer_helpers()
            for k in r:
                assert np.array_equal(h[k], r[k]), k
        for k, w in want.items():
            assert M.kmer_comp(k) == w["comp"] and M.kmer_revcomp(k) == w["revcomp"] and M.kmer_head(k) == w["head"]
            assert M.str_to_kmer("GG" + w["s"].lower(), 2) == k
    for s in ("ACGTN", "NACGT", "AXCGT", "nnnnn", "TTTTG"):               # a non-ACGT character ORs in 4, in u16
        assert I.str_to_kmer(s) == U.str_to_kmer(s)
        if B.Ref.available():
            assert I.str_to_kmer(s) == B.Ref.lib().ref_str_to_kmer(s.encode(), 0)


def test_range_arithmetic():
    U = B.uncalled_module()
    rng = np.random.default_rng(3)
    for _ in range(3000):
        a, b, c, d = (int(v) for v in rng.integers(0, 12, 4))
        for M in (I, U):
            x, y = M.Range(a, b), M.Range(c, d)
            z = M.Range(a, b)
            left = z.split_range(y)
            row = (x.length(), x.is_valid(), x.intersects(y), (x.intersect(y).start, x.intersect(y).end),
                   (x.merge(y).start, x.merge(y).end), x.same_range(y), x == y, x < y,
                   np.float32(x.get_recp_overlap(y)), (left.start, left.end), (z.start, z.end))
            if M is I:
                first = row
            else:
                assert row == first, (a, b, c, d)
    assert (I.Range().start, I.Range().end) == (1, 0) and I.Range(5, 2).length() == 2**64 - 2
