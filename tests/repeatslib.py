"""Test support for `find-repeats` (uncalled_b200.repeats, unc_repeats_*), never imported by the product:

- `oracle_lengths`: the oracle's orc_repeat_lengths (oracle/unc_oracle_repeats.c);
- `from_self_align`: L per position derived from self_align's paths at sample_dist 1 (the oracle's or the
  reference's own), by the relation `test_self_align_relation` checks;
- `brute_lengths`: L counted in numpy from the sorted suffixes of the forward text plus its reverse complement;
- `genome_fasta`: seeded N-free genomes with planted repeats, palindromes and repeats across contig ends;
- `expected_lines` / `expected_bed`: the CLI's output restated from an array of L;
- `repeat_lengths`: the device function under the emulator (tests/emul/emul_repeats.cpp);
- `expect_reference`: a result against the stored digest of what the reference's own code computed
  (tests/golden/repeats_digests.json);
- `EmuLib`: the unc_repeats_* entry points over the emulator, to stand in for the C-ABI under the Python layer."""
import bisect
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
DIGESTS = os.path.join(ROOT, "tests", "golden", "repeats_digests.json")

_emu = None


def emu():
    """tests/emul/libunc_emul_repeats.so, compiled on first use (and when a source is newer)"""
    global _emu
    if _emu is None:
        src = os.path.join(EMUL_DIR, "emul_repeats.cpp")
        out = os.path.join(EMUL_DIR, "libunc_emul_repeats.so")
        csrc = os.path.join(ROOT, "uncalled_b200", "csrc")
        deps = [src, os.path.join(EMUL_DIR, "warp_emul.hpp")] + [os.path.join(csrc, f) for f in (
            "unc_selfalign.cuh", "unc_selfalign_host.hpp", "unc_device.cuh", "unc_host_index.hpp")]
        if not (os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(x) for x in deps)):
            subprocess.run(["g++", "-O2", "-g", "-std=c++17", "-ffp-contract=off", "-DUNC_EMUL", "-DK2_MAXSEG=16u", "-fPIC",
                            "-shared", "-I" + EMUL_DIR, "-I" + csrc, "-o", out, src], check=True, capture_output=True)
        _emu = C.CDLL(out)
        _emu.emu_repeat_lengths.argtypes = [C.c_char_p, C.c_uint64, C.c_uint32, C.c_void_p]
    return _emu


def repeat_lengths(prefix, pac_st, n):
    """unc_repeat_length on the CPU: the repeat lengths of .pac positions [pac_st, pac_st + n) as uint32"""
    out = np.zeros(max(n, 1), np.uint32)
    rc = emu().emu_repeat_lengths(prefix.encode(), pac_st, n, out.ctypes.data)
    if rc != 0:
        raise RuntimeError("emu_repeat_lengths failed (%d)" % rc)
    return out[:n]


def expect_reference(key, got, live=False):
    """orclib.expect_reference over this feature's own digest file: `got` (a tuple of arrays) against the digest of what
    the reference's own code computed for the same inputs.  live=True: the caller has just compared `got` with
    oracle/_ref itself; with UNC_RECORD_REF_DIGESTS=1 its digest is then (re)written instead."""
    import json
    import orclib
    gold = json.load(open(DIGESTS)) if os.path.exists(DIGESTS) else {}
    d = orclib.digest(*got)
    if live and os.environ.get("UNC_RECORD_REF_DIGESTS") == "1":
        gold[key] = d
        with open(DIGESTS, "w") as f:
            json.dump(gold, f, indent=0, sort_keys=True)
            f.write("\n")
        return
    assert key in gold, "no stored reference result for %s" % key
    assert d == gold[key], "%s differs from the reference's result" % key

_orc = None


def orc():
    global _orc
    if _orc is None:
        path = os.path.join(ORACLE_DIR, "libunc_oracle_repeats.so")
        if not os.path.exists(path):
            subprocess.run(["make", "-C", ORACLE_DIR, "-f", "repeats.mk"], check=True, capture_output=True)
        lib = C.CDLL(path)
        lib.orc_index_load.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]
        lib.orc_index_free.argtypes = [C.c_void_p]
        lib.orc_repeat_lengths.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint64, C.c_void_p]
        _orc = lib
    return _orc


def layout(prefix):
    """(l_pac, [(name, offset, length)], holes [(offset, length)]) from the .ann and .amb"""
    with open(prefix + ".ann") as f:
        l_pac, n = (int(v) for v in f.readline().split()[:2])
        contigs = []
        for _ in range(n):
            name = f.readline().split()[1]
            off, ln = (int(v) for v in f.readline().split()[:2])
            contigs.append((name, off, ln))
    with open(prefix + ".amb") as f:
        nh = int(f.readline().split()[2])
        holes = [tuple(int(v) for v in f.readline().split()[:2]) for _ in range(nh)]
    return l_pac, contigs, holes


def pac_codes(prefix):
    l_pac = layout(prefix)[0]
    pac = np.fromfile(prefix + ".pac", np.uint8)[:(l_pac + 3) // 4]
    codes = np.empty(pac.size * 4, np.uint8)
    for k in range(4):
        codes[k::4] = (pac >> (6 - 2 * k)) & 3
    return codes[:l_pac]


def oracle_lengths(prefix, pac_st=0, n=None):
    lib = orc()
    n = layout(prefix)[0] - pac_st if n is None else n
    idx = C.c_void_p()
    if lib.orc_index_load(prefix.encode(), b"-", C.byref(idx)) != 0:
        raise RuntimeError("oracle index load failed: " + prefix)
    try:
        out = np.zeros(max(n, 1), np.uint32)
        rc = lib.orc_repeat_lengths(idx, prefix.encode(), pac_st, n, out.ctypes.data)
        if rc != 0:
            raise RuntimeError("orc_repeat_lengths: %d" % rc)
        return out[:n]
    finally:
        lib.orc_index_free(idx)


def remaining(prefix):
    """lim - p for every .pac position: the bases from p to the end of its contig"""
    return np.concatenate([np.arange(ln, 0, -1, dtype=np.int64) for _, _, ln in layout(prefix)[1]])


def from_self_align(off, val, rem):
    """L per position from self_align's paths at sample_dist 1 (one path per position, .pac order): a path has L + 1
    range lengths, except one whose walk ended on an empty range (its last length > 1 and fewer than lim - p lengths),
    which has L"""
    off = np.asarray(off, np.int64)
    cnt = np.diff(off)
    assert len(cnt) == len(rem) and cnt.min() >= 1
    last = np.asarray(val, np.int64)[off[1:] - 1]
    empty_end = (last > 1) & (cnt < rem)
    return (cnt - 1 + empty_end).astype(np.uint32)


def brute_lengths(prefix, quirk=True):
    """L for every position from its definition: the least t >= 1 at which the t + 1 bases from p occur at most once in
    T = forward + revcomp(forward) (the concatenated .pac), capped by the end of p's contig.  quirk: the walk's first range
    [L2[c], L2[c + 1]] also holds row L2[c] (src/bwa_index.hpp:172-174), the last suffix below base c, which stays in the
    range while the text before it matches; its count is added.  N-free references only (holes have other bases in the
    .pac than in the BWT)."""
    f = pac_codes(prefix)
    T = bytes(np.concatenate([f, 3 - f[::-1]]).tolist())
    n = len(T)
    sa = sorted(range(n), key=lambda i: T[i:])
    keys = [T[i:] for i in sa]
    L2 = np.concatenate([[0], np.cumsum(np.bincount(np.frombuffer(T, np.uint8), minlength=4))])
    # text position of row L2[c] (row 0 is the `$` suffix, at the end of the text)
    z = [n if L2[c] == 0 else sa[L2[c] - 1] for c in range(4)]
    out = np.zeros(len(f), np.uint32)
    st = 0
    for _, _, ln in layout(prefix)[1]:
        for i in range(ln):
            p = st + i
            c0 = 3 - f[p]
            t = 0
            while p + t + 1 < st + ln:
                t += 1
                s = T[p:p + t + 1]
                cnt = bisect.bisect_right(keys, s + b"\xff") - bisect.bisect_left(keys, s)
                if quirk:
                    # the extra row after t steps: T[z - t:] with T[z - t:z] = revcomp(f[p + 1 .. p + t])
                    zz = z[c0]
                    want = bytes((3 - f[p + 1:p + t + 1][::-1]).tolist())
                    cnt += int(zz - t >= 0 and T[zz - t:zz] == want)
                if cnt <= 1:
                    break
            out[p] = t
        st += ln
    return out


def _rand(rng, n):
    return rng.integers(0, 4, n).astype(np.uint8)


def _rc(a):
    return (3 - a[::-1]).astype(np.uint8)


def genome_fasta(path, seed, n_contigs=3, size=900):
    """seeded N-free contigs with planted repeats: copies of a 60-base unit within and across contigs, a 40-base
    palindrome (its own reverse complement), a reverse-complement copy, a copy of a contig's end inside the next contig,
    a copy of the text across the end of the first contig, and a tandem run; returns the contigs' codes"""
    rng = np.random.default_rng(seed)
    unit, half, tail = _rand(rng, 60), _rand(rng, 20), _rand(rng, 35)
    pal = np.concatenate([half, _rc(half)])
    cs = [_rand(rng, size + 37 * k) for k in range(n_contigs)]
    cs[0][100:160] = unit
    cs[0][400:440] = pal
    cs[0][-35:] = tail                                  # the end of contig 0 ...
    cs[1][50:110] = unit
    cs[1][300:360] = _rc(unit)
    cs[1][500:535] = tail                               # ... inside contig 1
    cs[-1][200:320] = np.tile(_rand(rng, 8), 15)        # tandem
    cs[-1][600:660] = unit
    cs[-1][750:810] = np.concatenate([cs[0][-30:], cs[1][:30]])   # occurs only across the end of contig 0
    with open(path, "w") as fa:
        for k, c in enumerate(cs):
            fa.write(">ctg%d\n" % k)
            s = "".join("ACGT"[v] for v in c)
            for i in range(0, len(s), 70):
                fa.write(s[i:i + 70] + "\n")
    return cs


def build(fa, prefix):
    from uncalled_b200 import _native as N
    assert N.lib().unc_index_build(fa.encode(), prefix.encode()) == 0
    return prefix


def _reported(prefix, L, min_k):
    l_pac, contigs, holes = layout(prefix)
    hole = np.zeros(l_pac, bool)
    for o, ln in holes:
        hole[o:o + ln] = True
    for name, off, ln in contigs:
        for i in range(ln):
            if L[off + i] >= min_k and not hole[off + i]:
                yield name, off, i, int(L[off + i])


def expected_lines(prefix, L, min_k):
    """find_repeats.cpp's lines for the repeat lengths L of every .pac position: hole positions skipped, hole bases N"""
    l_pac, contigs, holes = layout(prefix)
    s = np.frombuffer(b"ACGT", np.uint8)[pac_codes(prefix)].copy()
    for o, ln in holes:
        s[o:o + ln] = ord("N")
    s = s.tobytes().decode()
    return "".join("%d\t%s\t%d\t%d\t%s\n" % (li, name, i, i + li, s[off + i:off + i + li])
                   for name, off, i, li in _reported(prefix, L, min_k))


def expected_bed(prefix, L, min_k):
    """the union of [p, p + L) of the reported positions, per contig, as BED (restated base by base)"""
    out = []
    l_pac, contigs, _ = layout(prefix)
    cover = {name: np.zeros(ln + 1, bool) for name, _, ln in contigs}
    for name, off, i, li in _reported(prefix, L, min_k):
        cover[name][i:i + li] = True
    for name, _, _ in contigs:
        c = cover[name].astype(np.int8)
        d = np.diff(np.concatenate([[0], c]))
        for a, b in zip(np.flatnonzero(d == 1), np.flatnonzero(d == -1)):
            out.append("%s\t%d\t%d\n" % (name, a, b))
    return "".join(out)


class EmuLib:
    """unc_init and unc_repeats_* over emu_repeat_lengths (the device function on the CPU), with the C-ABI's
    argument checks; `calls` records every entry point used"""
    UNC_E_ARG = -1

    def __init__(self):
        self.calls, self.handles = [], {}

    def unc_init(self, device):
        self.calls.append("unc_init")
        return 0

    def unc_repeats_create(self, prefix, ph):
        self.calls.append("unc_repeats_create")
        h = len(self.handles) + 1
        self.handles[h] = prefix.decode()
        ph._obj.value = h
        return 0

    def unc_repeats_lengths(self, h, pac_st, n, ptr):
        self.calls.append("unc_repeats_lengths")
        rc = emu().emu_repeat_lengths(self.handles[h.value].encode(), pac_st, n, ptr)
        return 0 if rc == 0 else self.UNC_E_ARG

    def unc_repeats_destroy(self, h):
        self.calls.append("unc_repeats_destroy")
        self.handles.pop(h.value)

    def unc_strerror(self, rc):
        return b"bad argument"

    def unc_last_error(self):
        return b"emulated"


def family_genome(n, seed, families=((300, 600), (2000, 20)), dup=5000, tandem=40):
    """n seeded bases (ACGT codes) with planted repeat families: per (length, copies) that many copies of one element (a
    tenth of them with one substitution per 500 bases), a segmental duplication of `dup` bases, a tandem array of
    `tandem` copies of a 171-base unit and a 2 kb reverse-complement copy"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 4, n, dtype=np.uint8)
    for ln, copies in families:
        unit = g[rng.integers(0, n - ln):][:ln].copy()
        for p in rng.integers(0, n - ln, copies):
            u = unit.copy()
            if rng.random() < 0.1:
                u[::500] = (u[::500] + 1) % 4
            g[p:p + ln] = u
    a, b = rng.integers(0, n - dup, 2)
    g[b:b + dup] = g[a:a + dup]
    t = int(rng.integers(0, n - 171 * tandem))
    g[t:t + 171 * tandem] = np.tile(rng.integers(0, 4, 171, dtype=np.uint8), tandem)
    c = int(rng.integers(0, n - 2000))
    g[c:c + 2000] = 3 - g[a:a + 2000][::-1]
    return g


def write_fasta(path, codes, names):
    """codes (0-3 = ACGT, 4 = N) split evenly into len(names) records of 60-column lines"""
    cuts = np.linspace(0, len(codes), len(names) + 1).astype(np.int64)
    lut = np.frombuffer(b"ACGTN", np.uint8)
    with open(path, "wb") as f:
        for name, a, b in zip(names, cuts[:-1], cuts[1:]):
            s = lut[codes[a:b]]
            full = len(s) // 60 * 60
            body = np.full((full // 60, 61), ord("\n"), np.uint8)
            body[:, :60] = s[:full].reshape(-1, 60)
            f.write(b">" + name.encode() + b"\n" + body.tobytes() + (s[full:].tobytes() + b"\n" if full < len(s) else b""))
