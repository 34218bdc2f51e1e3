"""`mask-external`: masking the windows of a target reference that occur more than min_copy times in a full reference
(masking/mask_external.sh, with the selection its README documents).

CPU: the numpy oracle (`oracle`, below) against a brute-force search on small inputs; the device source under the warp
emulator against the oracle, with a table small enough that probes collide and wrap, pieces smaller than a tile and
than k, and two CTA sizes; rejected inputs, `UNC_E_NO_DEVICE` and the CLI parser.  GPU: every fixture through the
C-ABI and the CLI, a 200 Mb full reference with a 2 Mb target over several pieces, the counts against FM-index ranges,
and `mask-internal` -> `mask-external` -> `index` -> `map`."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import masklib as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
_COMP = bytes.maketrans(b"ACGT", b"TGCA")
_MIX = np.uint64(0x9E3779B97F4A7C15)


def revcomp(w):
    return w[::-1].translate(_COMP)


# ---------------------------------------------------------------- the semantics, restated in numpy

def _pack(c, L):
    """u64 value of the L (1..32) bases starting at each position of c (2-bit codes as u64, first base in the top
    bits): len(c) - L + 1 values, built by doubling"""
    acc, alen, p, plen = None, 0, c, 1
    while True:
        if L & plen:
            if acc is None:
                acc, alen = p, plen
            else:
                m = len(c) - (alen + plen) + 1
                acc = (acc[:m] << np.uint64(2 * plen)) | p[alen:alen + m]
                alen += plen
        if plen * 2 > L:
            return acc
        m = len(p) - plen
        p = (p[:m] << np.uint64(2 * plen)) | p[plen:plen + m]
        plen *= 2


def _keys(c, k):
    """(hi, lo) of the k-mer at each start of c: lo = its last min(k, 32) bases, hi = the first k - 32"""
    lo = _pack(c[k - min(k, 32):], min(k, 32))
    hi = _pack(c, k - 32)[:len(lo)] if k > 32 else np.zeros(len(lo), np.uint64)
    return hi, lo


def canon(codes, k):
    """per window start of `codes` (0-3 = ACGT, 4 = anything else): canonical key (hi, lo), palindrome, valid"""
    n = len(codes) - k + 1
    if n <= 0:
        e = np.zeros(0, np.uint64)
        return e, e, np.zeros(0, bool), np.zeros(0, bool)
    c = (codes & 3).astype(np.uint64)
    fh, fl = _keys(c, k)
    rh, rl = _keys((np.uint64(3) - c)[::-1].copy(), k)
    rh, rl = rh[::-1], rl[::-1]
    bad = np.concatenate([[0], np.cumsum(codes >= 4)])
    valid = bad[k:k + n] - bad[:n] == 0
    fwd = (fh < rh) | ((fh == rh) & (fl <= rl))
    return np.where(fwd, fh, rh), np.where(fwd, fl, rl), (fh == rh) & (fl == rl), valid


def _flat(data):
    heads, seqs = M.read_fasta(data)
    return heads, seqs, np.frombuffer(b"\n".join(seqs), np.uint8)


def window_counts(full, target, k, chunk=1 << 23):
    """per target position (records joined with one separator), occ(w) + occ(revcomp(w)) over the full reference's
    records of the window w starting there, 0 where no valid window starts; saturated at 2^32 - 1"""
    _, _, tflat = _flat(target)
    th, tl, _, tv = canon(M._CODE[tflat], k)
    out = np.zeros(len(tflat), np.uint64)
    idx = np.flatnonzero(tv)
    if len(idx) == 0:
        return out.astype(np.uint32)
    h = tl[idx] ^ (th[idx] * _MIX)
    uh, first, inv = np.unique(h, return_index=True, return_inverse=True)
    assert len(np.unique(np.stack([th[idx], tl[idx]], 1), axis=0)) == len(uh)    # no two keys share a hash
    uk_h, uk_l = th[idx][first], tl[idx][first]
    acc = np.zeros(len(uh), np.float64)
    gflat = _flat(full)[2]
    for a in range(0, max(len(gflat) - k + 1, 0), chunk):
        gh, gl, gp, gv = canon(M._CODE[gflat[a:a + chunk + k - 1]], k)
        gh, gl, gp = gh[gv], gl[gv], gp[gv]
        hh = gl ^ (gh * _MIX)
        pos = np.minimum(np.searchsorted(uh, hh), len(uh) - 1)
        m = (uh[pos] == hh) & (uk_h[pos] == gh) & (uk_l[pos] == gl)
        acc += np.bincount(pos[m], weights=1.0 + gp[m], minlength=len(uh))
    out[idx] = acc.astype(np.uint64)[inv]
    return np.minimum(out, 2 ** 32 - 1).astype(np.uint32)


def oracle(full, target, k, min_copy):
    """(window counts, masked FASTA bytes, BED bytes, masked bp)"""
    counts = window_counts(full, target, k)
    heads, seqs, flat = _flat(target)
    n = len(flat)
    sel = np.flatnonzero(counts > min_copy)
    d = np.zeros(n + k + 1, np.int64)
    np.add.at(d, sel, 1)
    np.add.at(d, sel + k, -1)
    masked = np.cumsum(d)[:n] > 0
    out = flat.copy()
    out[masked] = ord("N")
    recs, bed, pos = [], [], 0
    for h, s in zip(heads, seqs):
        recs.append(out[pos:pos + len(s)].tobytes())
        mk = np.concatenate([[0], masked[pos:pos + len(s)].astype(np.int8), [0]])
        edges = np.flatnonzero(np.diff(mk))
        name = h[1:].split()[0] if h[1:].split() else b""
        bed += [b"%s\t%d\t%d\n" % (name, a, b) for a, b in zip(edges[::2], edges[1::2])]
        pos += len(s) + 1
    return counts, M.write_fasta(heads, recs), b"".join(bed), int(masked.sum())


def brute_counts(full, target, k):
    """the same counts by overlapping str.find of w and revcomp(w) in every upper-cased record"""
    recs = [s.upper() for s in M.read_fasta(full)[1]]

    def occ(r, w):
        c, i = 0, r.find(w)
        while i >= 0:
            c, i = c + 1, r.find(w, i + 1)
        return c
    out = []
    for s in M.read_fasta(target)[1]:
        u = s.upper()
        for i in range(len(u)):
            w = u[i:i + k]
            ok = len(w) == k and all(ch in b"ACGT" for ch in w)
            out.append(sum(occ(r, w) + occ(r, revcomp(w)) for r in recs) if ok else 0)
        out.append(0)
    return np.array(out[:-1], np.uint64)


# ---------------------------------------------------------------- fixtures: (full reference, target)

def _rand(rng, n):
    return bytearray(b"ACGT"[i] for i in rng.integers(0, 4, n))


def _put(s, p, unit):
    s[p:p + len(unit)] = unit


def fx_planted(seed=21):
    """exact and reverse-complement copies of two elements, tandem repeats; the target holds one copy of each"""
    rng = np.random.default_rng(seed)
    e1, e2 = bytes(_rand(rng, 150)), bytes(_rand(rng, 90))
    full = []
    for r, n in enumerate((4000, 2500, 1800)):
        s = _rand(rng, n)
        for j in range(2 + r):
            _put(s, 100 + 700 * j, e1 if j % 2 == 0 else revcomp(e1))
        _put(s, n - 400, e2 if r else revcomp(e2))
        _put(s, n - 200, b"CAGT" * 25)
        full.append(b">chr%d some text\n" % (r + 1) + M._wrap(s, 60))
    t = _rand(rng, 1500)
    _put(t, 50, e1)
    _put(t, 400, revcomp(e2))
    _put(t, 700, b"CAGT" * 12)
    _put(t, 1000, b"TTAGGG" * 10)
    return b"".join(full), b">tgt1 first\n" + M._wrap(t, 70) + b">tgt2\n" + M._wrap(_rand(rng, 300), 50)


def fx_mixed(seed=22):
    """lowercase, N and IUPAC runs in both files, palindromes (x + revcomp(x)), CRLF line ends, blank lines"""
    rng = np.random.default_rng(seed)
    pal = bytes(_rand(rng, 20))
    pal = pal + revcomp(pal)
    elem = bytes(_rand(rng, 80))
    parts = []
    for r in range(3):
        s = _rand(rng, 2500)
        for j in range(3):
            _put(s, 200 + 600 * j + 40 * r, pal)
        _put(s, 1900, elem.lower() if r == 1 else elem)
        for b in b"NNRYKn-":
            p, L = int(rng.integers(0, len(s) - 40)), int(rng.integers(1, 30))
            _put(s, p, bytes([b]) * L)
        p = int(rng.integers(0, len(s) - 300))
        _put(s, p, bytes(s[p:p + 300]).lower())
        parts.append(b">m%d\r\n" % r + M._wrap(s, 61, b"\r\n") + b"\r\n")
    t = _rand(rng, 1200)
    _put(t, 100, pal)
    _put(t, 300, elem)
    _put(t, 500, revcomp(elem).lower())
    _put(t, 330, b"N")                                                     # one copy broken by an N
    _put(t, 800, b"ACGTRYACGT")
    _put(t, 900, pal[:10] + b"nn" + pal[12:])
    return b"".join(parts), b">t  x\r\n" + M._wrap(t, 55, b"\r\n")


def fx_boundary(seed=23):
    """target windows at the ends of records, and copies in the full reference cut by record boundaries and Ns"""
    rng = np.random.default_rng(seed)
    x = bytes(_rand(rng, 200))
    a, b = _rand(rng, 1000), _rand(rng, 1000)
    a[-100:] = x[:100]                                                     # x spans the record boundary a | b
    b[:100] = x[100:]
    c = _rand(rng, 900)
    _put(c, 100, x[:60] + b"N" + x[61:])                                   # broken by an N
    _put(c, 500, x)                                                        # one whole copy
    full = b">a\n" + M._wrap(a, 60) + b">b\n" + M._wrap(b, 60) + b">c\n" + M._wrap(c, 60)
    target = b">x1\n" + x + b"\n>x2\n" + x[:70] + b"\n>x3 short\n" + x[150:] + b"\n>x4\nAC\n"
    return full, target


def fx_contained(seed=24):
    """the target is a part of the full reference: every window counts at least once"""
    rng = np.random.default_rng(seed)
    recs = [_rand(rng, n) for n in (3000, 2000)]
    for s in recs:
        for j in range(4):
            _put(s, 300 + 400 * j, b"AAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAA")
    full = b"".join(b">c%d\n" % i + M._wrap(s, 80) for i, s in enumerate(recs))
    return full, b">part\n" + M._wrap(recs[1][500:1800], 80)


def fx_exact(seed=25):
    """an element planted exactly four times (twice reversed): its windows count 4, at and one above min_copy 3/4"""
    rng = np.random.default_rng(seed)
    e = bytes(_rand(rng, 100))
    s = _rand(rng, 6000)
    for j, p in enumerate((200, 1500, 3000, 4700)):
        _put(s, p, e if j % 2 else revcomp(e))
    t = _rand(rng, 500)
    _put(t, 200, e)
    return b">g\n" + M._wrap(s, 60), b">t\n" + M._wrap(t, 60)


FIXTURES = {"planted": fx_planted, "mixed": fx_mixed, "boundary": fx_boundary, "contained": fx_contained,
            "exact": fx_exact}
# (fixture, min_len, min_copy)
CASES = [("planted", 50, 5), ("planted", 2, 100), ("planted", 31, 2), ("planted", 32, 2), ("planted", 33, 3),
         ("mixed", 40, 2), ("mixed", 20, 1), ("mixed", 32, 1), ("boundary", 31, 1), ("boundary", 64, 1),
         ("boundary", 63, 1), ("contained", 50, 1), ("contained", 33, 3), ("exact", 50, 3), ("exact", 50, 4),
         ("exact", 64, 3), ("exact", 2, 800)]
BRUTE = [("planted", 2), ("planted", 33), ("mixed", 20), ("mixed", 32), ("boundary", 31), ("boundary", 64),
         ("boundary", 63), ("contained", 50), ("exact", 50), ("exact", 2)]


def _write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


def _files(tmp_path, fx):
    full, target = FIXTURES[fx]()
    return full, target, _write(tmp_path, "full.fa", full), _write(tmp_path, "target.fa", target)


# ---------------------------------------------------------------- the emulator

_lib = None


def emu_lib():
    global _lib
    if _lib is None:
        src = os.path.join(EMUL_DIR, "emul_mask_external.cpp")
        out = os.path.join(EMUL_DIR, "libunc_emul_mask_external.so")
        csrc = os.path.join(ROOT, "uncalled_b200", "csrc")
        deps = [src, os.path.join(EMUL_DIR, "warp_emul.hpp")] + \
            [os.path.join(csrc, f) for f in ("unc_mask_ext.cuh", "unc_mask_ext_host.hpp", "unc_mask.cuh",
                                             "unc_mask_host.hpp", "unc_device.cuh", "unc_warp.cuh")]
        if not (os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps)):
            subprocess.run(["g++", "-O2", "-g", "-std=c++17", "-ffp-contract=off", "-DUNC_EMUL", "-DK2_MAXSEG=16u", "-fPIC",
                            "-shared", "-I" + EMUL_DIR, "-I" + csrc, "-o", out, src], check=True, capture_output=True)
        L = C.CDLL(out)
        u32, u64 = C.c_uint32, C.c_uint64
        L.emu_mask_external.argtypes = [C.c_char_p, C.c_char_p, u32, u32, C.c_char_p, C.c_char_p, u64, C.c_int, u64,
                                        u64, C.c_void_p, C.POINTER(u64), C.POINTER(u64)]
        _lib = L
    return _lib


def _out(tmp_path, min_copy):
    return str(tmp_path / ("o_masked%d.fa" % min_copy)), str(tmp_path / ("o_reps_m%d.bed" % min_copy))


def emu_mask_external(full, target, k, min_copy, out_fa, out_bed, piece=0, n_threads=32, cap=0, filter_bits=0):
    """(status, window counts, n_selected, masked bp) of the device source on the CPU"""
    counts = np.zeros(os.path.getsize(target) + 1, np.uint32)            # at least one per target position
    sel, bp = C.c_uint64(), C.c_uint64()
    rc = emu_lib().emu_mask_external(full.encode(), target.encode(), k, min_copy, out_fa.encode(), out_bed.encode(),
                                     piece, n_threads, cap, filter_bits, counts.ctypes.data, C.byref(sel), C.byref(bp))
    n = len(_flat(open(target, "rb").read())[2]) if rc == 0 else 0
    return rc, counts[:n], sel.value, bp.value


def native_call(full, target, k, min_copy, out_fa, out_bed, piece=0, counts=None):
    import uncalled_b200._native as N
    sel, bp = C.c_uint64(), C.c_uint64()
    rc = N.lib().unc_mask_external(full.encode(), target.encode(), k, min_copy, out_fa.encode(), out_bed.encode(),
                                   piece, None if counts is None else counts.ctypes.data, C.byref(sel), C.byref(bp))
    return rc, N.lib().unc_last_error().decode(), sel.value, bp.value


def _distinct_keys(target, k):
    th, tl, _, tv = canon(M._CODE[_flat(target)[2]], k)
    return len(np.unique(np.stack([th[tv], tl[tv]], 1), axis=0))


# ---------------------------------------------------------------- CPU

@pytest.mark.parametrize("fx,k", BRUTE)
def test_oracle_matches_brute_force(fx, k):
    full, target = FIXTURES[fx]()
    want = brute_counts(full, target, k)
    assert np.array_equal(window_counts(full, target, k, chunk=997), want)
    assert want.max() > 1


def test_fixtures_cover_the_cases():
    full, target = fx_mixed()
    c = window_counts(full, target, 40)
    assert c[100] >= 2 and c[100] % 2 == 0                                 # a palindrome: 2 per locus
    assert c[300] == 0 and c[500] >= 1                                     # an N in the window / a lowercase revcomp copy
    assert c[800 - 39 + 5] == 0                                            # an IUPAC code in the window
    full, target = fx_boundary()
    c = window_counts(full, target, 31)
    # x: a whole copy, a copy cut at 100 by a record boundary, a copy with an N at 60
    assert (c[0], c[30], c[69], c[70]) == (3, 2, 3, 2)
    full, target = fx_exact()
    c = window_counts(full, target, 50)
    assert set(c[200:251].tolist()) == {4} and c[199] == 0 and c[251] == 0
    assert window_counts(b">a\nACGT\n", b">b\nACGT\n", 4)[0] == 2          # ACGT is its own reverse complement
    assert window_counts(b">a\nACGT\n>b\nACGT\n", b">b\nACGT\n", 2).tolist() == [4, 4, 4, 0]


@pytest.mark.parametrize("fx,k,min_copy", CASES)
def test_emulated_device_source_matches_oracle(fx, k, min_copy, tmp_path):
    full, target, ffa, tfa = _files(tmp_path, fx)
    counts, fa, bed, bp = oracle(full, target, k, min_copy)
    out_fa, out_bed = _out(tmp_path, min_copy)
    rc, got, sel, gbp = emu_mask_external(ffa, tfa, k, min_copy, out_fa, out_bed)
    assert rc == 0
    assert np.array_equal(got, counts)
    assert open(out_fa, "rb").read() == fa and open(out_bed, "rb").read() == bed
    assert gbp == bp and sel == int((counts > min_copy).sum())


@pytest.mark.parametrize("n_threads", [32, 64])
@pytest.mark.parametrize("fx,k,min_copy,piece", [("planted", 50, 2, 7), ("planted", 33, 1, 3000), ("mixed", 64, 1, 5),
                                                 ("boundary", 31, 1, 1), ("contained", 2, 50, 61),
                                                 ("exact", 63, 3, 2047)])
def test_emulated_pieces_tiny_table_and_cta_sizes(fx, k, min_copy, piece, n_threads, tmp_path):
    """pieces smaller than k and than a tile (windows straddle pieces), a table with one free slot more than the
    distinct keys rounded up to a power of two (probes collide and wrap), a 64-bit filter (every probe passes it)"""
    full, target, ffa, tfa = _files(tmp_path, fx)
    counts, fa, bed, bp = oracle(full, target, k, min_copy)
    cap = 1 << int(_distinct_keys(target, k)).bit_length()
    out_fa, out_bed = _out(tmp_path, min_copy)
    rc, got, sel, gbp = emu_mask_external(ffa, tfa, k, min_copy, out_fa, out_bed, piece=piece, n_threads=n_threads,
                                          cap=cap, filter_bits=64)
    assert rc == 0 and np.array_equal(got, counts)
    assert open(out_fa, "rb").read() == fa and open(out_bed, "rb").read() == bed and gbp == bp


def test_exactly_min_copy_is_not_masked(tmp_path):
    full, target, ffa, tfa = _files(tmp_path, "exact")
    for min_copy, want_bp, want_bed in ((4, 0, b""), (3, 100, b"t\t200\t300\n")):  # the element's 51 windows count 4
        out_fa, out_bed = _out(tmp_path, min_copy)
        rc, _, sel, bp = emu_mask_external(ffa, tfa, 50, min_copy, out_fa, out_bed)
        assert rc == 0 and bp == want_bp and sel == (51 if want_bp else 0)
        assert open(out_bed, "rb").read() == want_bed


_NO_COPY_FA = b">a\nACGTACGTTT\n"


@pytest.mark.parametrize("what,full,target,k,min_copy,sub", [
    ("k1", _NO_COPY_FA, _NO_COPY_FA, 1, 1, ""),
    ("k65", _NO_COPY_FA, _NO_COPY_FA, 65, 1, ""),
    ("min_copy0", _NO_COPY_FA, _NO_COPY_FA, 10, 0, ""),
    ("missing_dir", _NO_COPY_FA, _NO_COPY_FA, 4, 1, "nope/"),
    ("empty_full", b"", _NO_COPY_FA, 4, 1, ""),
    ("empty_target", _NO_COPY_FA, b"", 4, 1, ""),
    ("no_header_full", b"ACGT\n>a\nACGT\n", _NO_COPY_FA, 4, 1, ""),
    ("no_header_target", _NO_COPY_FA, b"\n>a\nACGT\n", 4, 1, ""),
    ("record_without_sequence_full", b">a\n>b\nACGT\n", _NO_COPY_FA, 4, 1, ""),
    ("record_without_sequence_target", _NO_COPY_FA, b">a\nACGT\n>b\n  \n", 4, 1, ""),
])
def test_rejected_inputs(what, full, target, k, min_copy, sub, tmp_path):
    import uncalled_b200 as U
    import uncalled_b200._native as N
    ffa, tfa = _write(tmp_path, "full.fa", full), _write(tmp_path, "target.fa", target)
    out_fa, out_bed = str(tmp_path / (sub + "o.fa")), str(tmp_path / (sub + "o.bed"))
    rc, msg, _, _ = native_call(ffa, tfa, k, min_copy, out_fa, out_bed)
    assert rc == -1 and msg, (what, rc, msg)                               # UNC_E_ARG
    assert emu_mask_external(ffa, tfa, k, min_copy, out_fa, out_bed)[0] == -1
    with pytest.raises(N.UncError, match="bad argument|does not exist"):
        U.mask_external(ffa, tfa, k, min_copy, str(tmp_path / (sub + "x_")))
    assert sorted(os.listdir(tmp_path)) == ["full.fa", "target.fa"]


def test_missing_file_is_an_io_error(tmp_path):
    fa = _write(tmp_path, "t.fa", _NO_COPY_FA)
    rc, msg, _, _ = native_call(str(tmp_path / "nope.fa"), fa, 4, 1, str(tmp_path / "o.fa"), str(tmp_path / "o.bed"))
    assert rc == -2 and "nope.fa" in msg


def test_fails_loudly_without_a_gpu(tmp_path):
    """No CPU path: a valid call without a CUDA device reports UNC_E_NO_DEVICE and writes nothing."""
    import uncalled_b200._native as N
    if N.lib().unc_device_count() > 0:
        pytest.skip("a CUDA device is present")
    _, _, ffa, tfa = _files(tmp_path, "planted")
    rc, _, _, _ = native_call(ffa, tfa, 50, 5, str(tmp_path / "o.fa"), str(tmp_path / "o.bed"))
    assert rc == -4
    assert not os.path.exists(str(tmp_path / "o.fa")) and not os.path.exists(str(tmp_path / "o.bed"))


def test_cli_parser():
    from uncalled_b200 import cli
    _, _, a = cli.load_conf(["mask-external", "full.fa", "t.fa", "50", "5", "out/t_", "--device", "1"])
    assert (a.subcmd, a.full_reference, a.target, a.min_len, a.min_copy, a.out_prefix, a.device) == \
        ("mask-external", "full.fa", "t.fa", 50, 5, "out/t_", 1)
    with pytest.raises(SystemExit):
        cli.load_conf(["mask-external", "full.fa", "t.fa", "50"])


# ---------------------------------------------------------------- GPU

@pytest.mark.gpu
@pytest.mark.parametrize("fx,k,min_copy", CASES)
def test_gpu_matches_oracle(fx, k, min_copy, tmp_path, capsys):
    from uncalled_b200 import cli
    full, target, ffa, tfa = _files(tmp_path, fx)
    counts, fa, bed, bp = oracle(full, target, k, min_copy)
    for piece in (0, 5, 4096):
        got = np.zeros(len(counts), np.uint32)
        out_fa, out_bed = _out(tmp_path, min_copy)
        rc, msg, sel, gbp = native_call(ffa, tfa, k, min_copy, out_fa, out_bed, piece=piece, counts=got)
        assert rc == 0, msg
        assert np.array_equal(got, counts) and gbp == bp and sel == int((counts > min_copy).sum())
        assert open(out_fa, "rb").read() == fa and open(out_bed, "rb").read() == bed
    capsys.readouterr()
    prefix = str(tmp_path / "cli_")
    assert cli.main(["mask-external", ffa, tfa, str(k), str(min_copy), prefix]) == 0
    assert capsys.readouterr().out == "Masked %d basepairs\n" % bp
    assert open(prefix + "masked%d.fa" % min_copy, "rb").read() == fa
    assert open(prefix + "reps_m%d.bed" % min_copy, "rb").read() == bed


def big_pair(n_full, n_target, seed=5):
    """a seeded full reference (masklib.big_genome) and a target: two thirds copied from it, one third random"""
    full = M.big_genome(n_full, seed=seed)
    flat = _flat(full)[2]
    rng = np.random.default_rng(seed + 1)
    parts = []
    for i in range(4):
        L = n_target // 6
        p = int(rng.integers(0, len(flat) - L))
        parts.append(b">from%d\n" % i + M._wrap(flat[p:p + L].tobytes(), 60))
    rnd = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n_target // 3)].tobytes()
    parts.append(b">random\n" + M._wrap(rnd, 60))
    return full, b"".join(parts)


@pytest.mark.gpu
def test_gpu_200mb_full_reference(tmp_path):
    import uncalled_b200 as U
    full, target = big_pair(200_000_000, 2_000_000)
    ffa, tfa = _write(tmp_path, "full.fa", full), _write(tmp_path, "target.fa", target)
    counts, fa, bed, bp = oracle(full, target, 50, 5)
    got = np.zeros(len(counts), np.uint32)
    out_fa, out_bed = _out(tmp_path, 5)
    rc, msg, _, gbp = native_call(ffa, tfa, 50, 5, out_fa, out_bed, piece=48_000_000, counts=got)
    assert rc == 0, msg
    assert np.array_equal(got, counts) and gbp == bp and bp > 0
    assert open(out_fa, "rb").read() == fa and open(out_bed, "rb").read() == bed
    masked, intervals = U.mask_external(ffa, tfa, 50, 5, str(tmp_path / "api_"))
    assert masked == bp and b"".join(b"%s\t%d\t%d\n" % (n.encode(), a, b) for n, a, b in intervals) == bed


@pytest.mark.gpu
def test_gpu_counts_equal_fm_index_ranges(tmp_path):
    """On an N-free single-record full reference, each window's count is the length of its FM range found by backward
    search in the bwa index of the reference (which holds both strands), except for the windows that also match
    across the junction of the forward and reverse-complement texts: those are found and left out explicitly."""
    import uncalled_b200 as U
    rng = np.random.default_rng(31)
    g = _rand(rng, 60000)
    e = bytes(_rand(rng, 120))
    for j in range(8):
        _put(g, 2000 + 7000 * j, e if j % 3 else revcomp(e))
    _put(g, 30000, b"TTAGGG" * 30)
    gs = bytes(g)
    full = b">g\n" + M._wrap(gs, 60)
    t = bytes(_rand(rng, 300)) + e + gs[100:400] + b"TTAGGG" * 15 + gs[-200:] + revcomp(gs[:150])
    target = b">t\n" + t + b"\n"
    ffa, tfa = _write(tmp_path, "g.fa", full), _write(tmp_path, "t.fa", target)
    from uncalled_b200 import cli
    assert cli.main(["index", ffa]) == 0
    with open(ffa + ".bwt", "rb") as f:
        head = np.frombuffer(f.read(40), np.uint64)                       # primary, then L2[1..4]
    L2 = np.concatenate([[0], head[1:5]]).astype(np.uint64)
    idx = U.Index(ffa)
    k = 24
    got = np.zeros(len(t), np.uint32)
    rc, msg, _, _ = native_call(ffa, tfa, k, 1, str(tmp_path / "o.fa"), str(tmp_path / "o.bed"), counts=got)
    assert rc == 0, msg
    code = {ord(c): i for i, c in enumerate("ACGT")}
    n_win = len(t) - k + 1
    st = np.array([L2[code[t[i + k - 1]]] + 1 for i in range(n_win)], np.uint64)
    en = np.array([L2[code[t[i + k - 1]] + 1] for i in range(n_win)], np.uint64)
    for j in range(k - 2, -1, -1):                                         # backward search, last base first
        st, en = idx.neighbors(st, en, np.array([code[t[i + j]] for i in range(n_win)], np.uint8))
    fm = np.where(en >= st, en - st + 1, 0).astype(np.int64)
    rc_text = revcomp(gs)
    junction = gs[-(k - 1):] + rc_text[:k - 1]                            # forward text followed by its reverse complement
    skipped = 0
    for i in range(n_win):
        w = t[i:i + k]
        if w in junction or revcomp(w) in junction:
            skipped += 1
            continue
        assert got[i] == fm[i], (i, got[i], fm[i])
    assert skipped < n_win // 10 and got[:n_win].max() >= 8
    idx.close()


@pytest.mark.gpu
def test_gpu_mask_internal_then_external_then_index_then_map(tmp_path, capsys):
    """the reference's recipe on the example reference: `mask-internal`, `mask-external` of its output against the
    reference, `index` of the result, `map` of the example read"""
    import orclib
    from uncalled_b200 import cli
    os.makedirs(tmp_path / "src")
    src = orclib.materialise_example_index(str(tmp_path / "src"))
    fa = _write(tmp_path, "ref.fa", open(src + ".fa", "rb").read())
    assert cli.main(["mask-internal", fa, "10", "5", str(tmp_path / "ref_")]) == 0
    m5 = str(tmp_path / "ref_mask5.fa")
    capsys.readouterr()
    assert cli.main(["mask-external", fa, m5, "24", "1", str(tmp_path / "ref_mask5_")]) == 0
    out = capsys.readouterr().out
    masked = str(tmp_path / "ref_mask5_masked1.fa")
    _, want_fa, _, want_bp = oracle(open(fa, "rb").read(), open(m5, "rb").read(), 24, 1)
    assert out == "Masked %d basepairs\n" % want_bp and open(masked, "rb").read() == want_fa
    assert cli.main(["index", masked]) == 0
    capsys.readouterr()
    assert cli.main(["map", masked, os.path.join(ROOT, "tests", "golden", "fast5", "example_single.fast5")]) == 0
    lines = capsys.readouterr().out.strip().split("\n")
    assert len(lines) == 1
    f = lines[0].split("\t")
    assert len(f) >= 12 and f[4] in "+-*"
