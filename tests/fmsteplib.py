"""Test support for the mapper's FM-index step (unc_occ2_neighbors through unc_fm_step / emu_fm_step), never imported
by the product.

- `FIXTURES`: small seeded references indexed by the product's host builder (unc_index_build, byte-identical to bwa),
  chosen so that seq_len mod 128 takes the values where the last, partial bwa block changes shape, so that the `$` row
  (primary) falls at the start and end of a 64-row occ2 block and into the last one, and so that most 5-mers of the
  tiny ones are absent (empty k-mer ranges);
- `PlainFM`: Occ(k, c) for every row, from the .bwt file unpacked in numpy with the `$` put back at primary;
- `occ_at_rows` / `step_at_rows`: bwt_occ at given rows only, for indexes too large to unpack (the 1.1 Gbp test);
- `check_*`: the checks, run against any step function with the signature of uncalled_b200.Index.fm_step."""
import ctypes as C
import json
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDTHS = (0, 1, 31, 32, 63, 64, 127, 128, 129)
SEQ_LEN_MOD_128 = (0, 2, 16, 30, 32, 62, 64, 66, 126)


def _rand(rng, n):
    return np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)].tobytes()


def _revcomp(s):
    return s[::-1].translate(bytes.maketrans(b"ACGT", b"TGCA"))


def _wrap(name, seq, width=60):
    return b">" + name + b"\n" + b"".join(seq[i:i + width] + b"\n" for i in range(0, len(seq), width))


def fx_mod(r, seed):
    """one record of 2 * (576 + r/2) FM rows: seq_len mod 128 == r"""
    return _wrap(b"mod%d" % r, _rand(np.random.default_rng(seed), 576 + r // 2))


def fx_primary(seed, head=b""):
    """a record whose text starts with `head`: a run of T puts the `$` row near the end of the BWT"""
    return _wrap(b"p%d" % seed, head + _rand(np.random.default_rng(seed), 700))


def fx_multi_n(seed=41):
    """three records with N runs (bwa replaces them with seeded random bases, and cuts the .amb holes)"""
    rng = np.random.default_rng(seed)
    out = b""
    for r in range(3):
        s = bytearray(_rand(rng, 300 + 170 * r))
        for _ in range(2):
            p, L = int(rng.integers(0, len(s) - 40)), int(rng.integers(1, 40))
            s[p:p + L] = b"N" * L
        out += _wrap(b"rec%d" % r, bytes(s))
    return out


def fx_poly(seed=42):
    rng = np.random.default_rng(seed)
    return _wrap(b"poly", _rand(rng, 200) + b"A" * 300 + _rand(rng, 100) + b"T" * 250 + _rand(rng, 90))


def fx_palindrome(seed=43):
    """a record that is its own reverse complement"""
    h = _rand(np.random.default_rng(seed), 400)
    return _wrap(b"pal", h + _revcomp(h))


def fx_tiny(n, seed=44):
    return _wrap(b"tiny%d" % n, _rand(np.random.default_rng(seed + n), n))


# seeds found by drawing until primary mod 64 is 0 and 63 and primary lies in the last 64-row block;
# test_fixture_coverage asserts that they still do
FIXTURES = {"mod%d" % r: (lambda r=r: fx_mod(r, 100 + r)) for r in SEQ_LEN_MOD_128}
FIXTURES.update({"primary_mod0": lambda: fx_primary(PRIMARY_SEEDS[0]), "primary_mod63": lambda: fx_primary(PRIMARY_SEEDS[1]),
                 "primary_last": lambda: fx_primary(PRIMARY_SEEDS[2], b"T" * 12),
                 "multi_n": fx_multi_n, "poly": fx_poly, "palindrome": fx_palindrome})
TINY = (1, 2, 3, 5, 8, 13, 21, 32, 40)
FIXTURES.update({"tiny%d" % n: (lambda n=n: fx_tiny(n)) for n in TINY})
PRIMARY_SEEDS = (28, 54, 1)


def uncl_line():
    return json.load(open(os.path.join(ROOT, "tests", "golden", "synth_uncl.json")))["g200k"]["uncl"]


def build(name, d):
    """bwa index files (and the .uncl threshold line) of fixture `name` under directory d; returns the prefix"""
    from uncalled_b200 import _native as N
    prefix = os.path.join(str(d), name)
    if not os.path.exists(prefix + ".uncl"):
        open(prefix + ".fa", "wb").write(FIXTURES[name]())
        rc = N.lib().unc_index_build((prefix + ".fa").encode(), prefix.encode())
        assert rc == 0, (name, rc)
        open(prefix + ".uncl", "w").write(uncl_line())
    return prefix


class PlainFM:
    """bwt_occ restated from the .bwt file: Occ(k, c) = count of c in BWT rows 0..k (the `$` at primary counts for none)"""

    def __init__(self, prefix):
        raw = np.fromfile(prefix + ".bwt", np.uint8)
        head = raw[:40].view(np.uint64)
        self.primary = int(head[0])
        self.L2 = np.concatenate([[0], head[1:5]]).astype(np.int64)
        self.n = int(self.L2[4])                                           # seq_len: rows 0..n
        words = raw[40:].view(np.uint32)
        i = np.arange(self.n, dtype=np.int64)                              # stored symbols: the BWT without the `$`
        w = words[(i >> 7) * 16 + 8 + ((i & 127) >> 4)]
        stored = ((w >> ((15 - (i & 15)) * 2).astype(np.uint32)) & 3).astype(np.int8)
        self.bwt = np.insert(stored, self.primary, 4)                     # rows 0..n, 4 = `$`
        occ = np.zeros((self.n + 2, 4), np.int64)                         # occ[k + 1] = Occ(k, .), occ[0] = Occ(-1, .)
        for c in range(4):
            occ[1:, c] = np.cumsum(self.bwt == c)
        self.occ = occ
        assert (occ[-1] == np.diff(self.L2)).all()

    def step(self, st, en):
        """(ns, ne) of shape (n, 4): L2[c] + Occ(st-1, c) + 1, L2[c] + Occ(en, c)"""
        st, en = np.asarray(st, np.int64), np.asarray(en, np.int64)
        return self.L2[:4] + self.occ[st] + 1, self.L2[:4] + self.occ[en + 1]

    def lf_walk_hits_primary(self, rows):
        """for each row, whether bwt_sa's LF walk from it (until a multiple of 32) passes through primary"""
        k = np.asarray(rows, np.int64).copy()
        hit = np.zeros(len(k), bool)
        for _ in range(32):
            act = (k & 31) != 0
            if not act.any():
                break
            hit |= act & (k == self.primary)
            c = self.bwt[k].astype(np.int64)
            nxt = np.where(c < 4, self.L2[np.minimum(c, 3)] + self.occ[k + 1, np.minimum(c, 3)], 0)
            k = np.where(act, nxt, k)
        return hit


def occ_at_rows(prefix, rows):
    """bwt_occ (reference submods/bwa/bwt.c:107-129) at the given rows only, read from the .bwt file without unpacking the
    whole text: the row's 128-row block's four u64 counts plus the symbols of the block up to the row.  (len(rows), 4)"""
    head = np.fromfile(prefix + ".bwt", np.uint64, 5)
    primary, L2 = int(head[0]), np.concatenate([[0], head[1:5]]).astype(np.int64)
    n = int(L2[4])
    words = np.memmap(prefix + ".bwt", np.uint32, "r", offset=40)
    k = np.asarray(rows, np.int64)
    out = np.empty((len(k), 4), np.int64)
    end = k == n
    out[end] = np.diff(L2)
    kk = k[~end] - (k[~end] >= primary)
    base = (kk >> 7) * 16
    cnt = words[np.minimum(base[:, None] + np.arange(8), len(words) - 1)].astype(np.int64)
    cnt = cnt[:, 0::2] | (cnt[:, 1::2] << 32)
    j = np.arange(128)
    w = words[np.minimum(base[:, None] + 8 + (j >> 4), len(words) - 1)].astype(np.int64)
    sym = (w >> ((15 - (j & 15)) * 2)) & 3
    upto = j[None, :] <= (kk & 127)[:, None]
    out[~end] = cnt + np.stack([((sym == c) & upto).sum(1) for c in range(4)], 1)
    return out


def step_at_rows(prefix, st, en):
    """(ns, ne) as PlainFM.step, from occ_at_rows"""
    L2 = np.concatenate([[0], np.fromfile(prefix + ".bwt", np.uint64, 5)[1:5]]).astype(np.int64)
    st, en = np.asarray(st, np.int64), np.asarray(en, np.int64)
    return L2[:4] + occ_at_rows(prefix, st - 1) + 1, L2[:4] + occ_at_rows(prefix, en)


def pairs_at_rows(rows, n, rng):
    """each row as start - 1 and as end, widths 0, 1, 63, 64, 128 and one random width; rows in [0, n]"""
    r = np.asarray(rows, np.int64)
    ds = [np.full(len(r), d, np.int64) for d in (0, 1, 63, 64, 128)] + [rng.integers(0, 5000, len(r))]
    st, en = [], []
    for d in ds:
        m = r < n                                           # as start - 1: (r + 1, min(r + d, n))
        st.append(r[m] + 1); en.append(np.minimum(r[m] + d[m], n))
        m = r >= 1                                          # as end: (max(r - d, 0) + 1, r)
        st.append(np.maximum(r[m] - d[m], 0) + 1); en.append(r[m])
    return np.concatenate(st), np.concatenate(en)


def edge_rows(fm):
    """primary - 1, primary, primary + 1, n - 1, n, and every 64- and 128-row boundary +-1 within 300 rows of those"""
    base = [fm.primary - 1, fm.primary, fm.primary + 1, fm.n - 1, fm.n]
    rows = set(base)
    for b in base:
        for m in range((b - 300) // 64 * 64, b + 301, 64):
            if abs(m - b) <= 300:
                rows.update((m - 1, m, m + 1))
    return np.array(sorted(r for r in rows if 0 <= r <= fm.n), np.int64)


def _check(step, fm, st, en, want):
    ns, ne, valid = step(st, en, want)
    xs, xe = fm.step(st, en)
    bad = np.nonzero((ns.astype(np.int64) != xs).any(1) | (ne.astype(np.int64) != xe).any(1))[0]
    assert not len(bad), [(int(st[i]), int(en[i]), ns[i].tolist(), xs[i].tolist(), ne[i].tolist(), xe[i].tolist())
                          for i in bad[:4]]
    bits = (np.asarray(want, np.int64)[:, None] >> np.arange(4)) & 1
    xv = ((bits == 1) & (xs <= xe)) @ (1 << np.arange(4))
    bad = np.nonzero(valid.astype(np.int64) != xv)[0]
    assert not len(bad), [(int(st[i]), int(en[i]), int(want[i]), int(valid[i]), int(xv[i])) for i in bad[:4]]
    return ns, ne


def every_row_queries(n, rng, widths=WIDTHS, rows=None):
    """(start, end) = (r, min(r + d, n)) for every r (or the given rows) and every width d, plus one random width each"""
    r = np.arange(1, n + 1, dtype=np.int64) if rows is None else np.asarray(rows, np.int64)
    ds = [np.full(len(r), d, np.int64) for d in widths] + [rng.integers(0, max(n, 1) + 1, len(r))]
    st = np.concatenate([r] * len(ds))
    en = np.minimum(st + np.concatenate(ds), n)
    return st, en


def check_every_row(step, fm, rng, chunk=1 << 22, **kw):
    st, en = every_row_queries(fm.n, rng, **kw)
    st, en = np.append(st, fm.n + 1), np.append(en, fm.n)    # start - 1 == n: what an empty range's next step asks
    k0, l0 = st - 1, en
    for o in range(0, len(st), chunk):
        s, e = st[o:o + chunk], en[o:o + chunk]
        _check(step, fm, s, e, rng.integers(0, 16, len(s)))
    return k0, l0


def check_edges(step, fm, rng):
    """every pair (st - 1, en) of edge rows with st - 1 <= en, and all 16 want masks on a sample of them"""
    rows = edge_rows(fm)
    k0, l0 = np.meshgrid(rows, rows, indexing="ij")
    keep = k0 <= l0
    st, en = k0[keep] + 1, l0[keep]
    _check(step, fm, st, en, np.full(len(st), 15))
    pick = rng.choice(len(st), min(len(st), 300), replace=False)
    s16, e16 = np.repeat(st[pick], 16), np.repeat(en[pick], 16)
    _check(step, fm, s16, e16, np.tile(np.arange(16), len(pick)))
    return rows


def oracle_neighbors(O, st, en):
    """orc_get_neighbor (the reference's BwaIndex::get_neighbor) for all four bases: (ns, ne) of shape (n, 4)"""
    a, b = C.c_uint64(), C.c_uint64()
    ns, ne = np.zeros((len(st), 4), np.int64), np.zeros((len(st), 4), np.int64)
    for i in range(len(st)):
        for c in range(4):
            O.lib.orc_get_neighbor(O.idx, int(st[i]), int(en[i]), c, C.byref(a), C.byref(b))
            ns[i, c], ne[i, c] = a.value, b.value
    return ns, ne


def oracle_sa(O, rows):
    return np.array([O.lib.orc_sa(O.idx, int(r)) for r in rows], np.uint64)
