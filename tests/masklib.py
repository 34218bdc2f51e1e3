"""Test support for `mask-internal` (never imported by the product).

- `fixtures()`: the seeded FASTA inputs of tests/golden/mask_golden.json (made by tools/make_mask_golden.py);
- `read_fasta` / `oracle`: a numpy restatement of masking/mask_internal.sh + masking/mask_kmers.py with the
  smallest-code tie rule (np.bincount over the valid k-mer codes, masking as the union of the occurrence ranges);
- `emu_mask_internal`: the device source run on the CPU under the warp emulator (tests/emul/emul_mask.cpp)."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
GOLDEN = os.path.join(ROOT, "tests", "golden", "mask_golden.json")

_CODE = np.full(256, 4, np.uint8)
for _i, _b in enumerate(b"ACGT"):
    _CODE[_b] = _CODE[_b | 0x20] = _i
_WS = b" \t\n\r\x0b\x0c\x1c\x1d\x1e\x1f"          # what Python's str.strip() removes from ASCII text


def kmer_str(code, k):
    return "".join("ACGT"[(int(code) >> (2 * (k - 1 - i))) & 3] for i in range(k))


def sha256(data):
    return hashlib.sha256(data).hexdigest()


# ---------------------------------------------------------------- fixtures

def _rand(rng, n):
    return bytearray(b"ACGT"[i] for i in rng.integers(0, 4, n))


def _wrap(seq, width, eol=b"\n"):
    return b"".join(bytes(seq[i:i + width]) + eol for i in range(0, len(seq), width))


def _plant(rng, seq, unit, copies):
    for _ in range(copies):
        p = int(rng.integers(0, len(seq) - len(unit)))
        seq[p:p + len(unit)] = unit


def fasta_repeats(seed=11):
    """three records with tandem repeats and interspersed copies of a few 300-base elements"""
    rng = np.random.default_rng(seed)
    elems = [_rand(rng, 300) for _ in range(3)]
    out = b""
    for r, n in enumerate((9000, 5000, 2600)):
        s = _rand(rng, n)
        for e in elems:
            _plant(rng, s, e, 2 + r)
        _plant(rng, s, bytearray(b"CAGT" * 25), 1)
        _plant(rng, s, bytearray(b"TTAGGG" * 20), 2)
        out += b">chr%d\n" % (r + 1) + _wrap(s, 60)
    return out


def fasta_mixed(seed=12):
    """lowercase stretches, N runs, IUPAC codes and spaces inside lines, lines of uneven length"""
    rng = np.random.default_rng(seed)
    out = b""
    for r in range(3):
        s = _rand(rng, 3000 + 700 * r)
        _plant(rng, s, bytearray(b"GATTACA" * 12), 3)
        for _ in range(6):
            p, L = int(rng.integers(0, len(s) - 200)), int(rng.integers(5, 200))
            s[p:p + L] = bytes(s[p:p + L]).lower()
        for b in b"NNNNRYKMSWBDHVn-. ":
            p, L = int(rng.integers(0, len(s) - 40)), int(rng.integers(1, 40))
            s[p:p + L] = bytes([b]) * L
        lines, i = [], 0
        while i < len(s):
            w = int(rng.integers(1, 90))
            lines.append(bytes(s[i:i + w]))
            i += w
        out += b">rec%d\n" % r + b"".join(l + b"\n" for l in lines)
    return out


def fasta_crlf(seed=13):
    """CRLF line ends, headers with comments and trailing blanks, a record shorter than k, blank lines, no final EOL"""
    rng = np.random.default_rng(seed)
    a = _rand(rng, 4000)
    _plant(rng, a, bytearray(b"ACGTTGCA" * 10), 4)
    b = _rand(rng, 2500)
    b[100:160] = a[1000:1060]
    return (b">first sequence one  \r\n" + _wrap(a, 70, b"\r\n") + b"\r\n" + b">tiny  comment\r\nAC\r\n" +
            b">second\tsome comment\r\n  " + _wrap(b, 61, b"  \r\n")[:-2])


def fasta_polya(seed=14):
    """poly-A and poly-T runs of various lengths between random sequence"""
    rng = np.random.default_rng(seed)
    out = b""
    for r in range(2):
        parts = []
        for _ in range(25):
            parts.append(_rand(rng, int(rng.integers(50, 400))))
            parts.append(bytearray(bytes([b"AT"[int(rng.integers(0, 2))]]) * int(rng.integers(5, 60))))
        out += b">polya%d\n" % r + _wrap(b"".join(parts), 80)
    return out


def fasta_tiny(seed=15):
    """few distinct short k-mers: more iterations than k-mers, so the loop stops early"""
    return b">t1\nACGTTTAC\n>t2\nGGGAAC\n"


def big_genome(n, seed=1, n_records=4):
    """an n-base multi-record FASTA (60-column lines) with planted interspersed elements, tandem repeats, poly-A runs,
    lowercase stretches and N runs: the bench and large-test workload, generated in numpy"""
    rng = np.random.default_rng(seed)
    s = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n, dtype=np.uint8)].copy()
    for L, copies in ((300, n // 30000), (6000, n // 2000000 + 1)):       # interspersed elements (Alu- / L1-like)
        for e in range(4):
            unit = s[rng.integers(0, n - L):][:L].copy()
            pos = rng.integers(0, n - L, copies)
            keep = rng.random(copies) < 0.9                                # a few diverged copies
            for p in pos[keep]:
                s[p:p + L] = unit
    for _ in range(n // 20000):                                            # tandem repeats
        unit = s[rng.integers(0, n - 10):][:int(rng.integers(1, 10))].copy()
        reps = int(rng.integers(5, 60))
        p = int(rng.integers(0, n - len(unit) * reps))
        s[p:p + len(unit) * reps] = np.tile(unit, reps)
    for _ in range(n // 50000):                                            # poly-A, lowercase, N runs
        p = int(rng.integers(0, n - 2000))
        s[p:p + int(rng.integers(10, 80))] = ord("A")
        q = int(rng.integers(0, n - 2000))
        s[q:q + int(rng.integers(10, 2000))] |= 0x20
    for _ in range(n // 1000000 + 1):
        p = int(rng.integers(0, n - 50000))
        s[p:p + int(rng.integers(100, 50000))] = ord("N")
    cuts = np.sort(rng.choice(np.arange(1, n), n_records - 1, replace=False)) if n_records > 1 else np.array([], int)
    out = []
    for r, (a, b) in enumerate(zip(np.r_[0, cuts], np.r_[cuts, n])):
        rec = s[a:b]
        full = len(rec) // 60
        body = np.full((full, 61), ord("\n"), np.uint8)
        body[:, :60] = rec[:full * 60].reshape(full, 60)
        tail = rec[full * 60:].tobytes()
        out.append(b">chr%d synthetic\n" % (r + 1) + body.tobytes() + (tail + b"\n" if tail else b""))
    return b"".join(out)


FIXTURES = {"repeats": fasta_repeats, "mixed": fasta_mixed, "crlf": fasta_crlf, "polya": fasta_polya, "tiny": fasta_tiny}
# (fixture, k, iters)
CASES = [("repeats", 10, 30), ("repeats", 5, 1), ("mixed", 5, 5), ("mixed", 13, 5), ("crlf", 3, 5), ("crlf", 13, 1),
         ("polya", 13, 5), ("polya", 1, 1), ("tiny", 1, 30), ("tiny", 3, 30)]


def fixture(name):
    return FIXTURES[name]()


# ---------------------------------------------------------------- the reference's semantics, restated

def read_fasta(data):
    """(headers, sequences) as mask_kmers.py reads a file: universal newlines, lines stripped, '>' lines are headers"""
    lines = data.replace(b"\r\n", b"\n").replace(b"\r", b"\n").split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    heads, seqs = [], []
    for ln in lines:
        if ln[:1] == b">":
            heads.append(ln.strip(_WS))
            seqs.append([])
        else:
            seqs[-1].append(ln.strip(_WS))
    return heads, [b"".join(s) for s in seqs]


def write_fasta(heads, seqs):
    return b"".join(h + b"\n" + s + b"\n" for h, s in zip(heads, seqs))


def oracle(data, k, iters):
    """(output bytes, [(kmer, count), ...]) of `mask-internal`: each iteration the k-mer of the highest count, ties
    to the smallest code; every position of every occurrence becomes N.  The counts are kept up to date by
    subtracting the k-mers each masking breaks (a full recount gives the same histogram)."""
    heads, seqs = read_fasta(data)
    flat = np.frombuffer(b"\n".join(seqs), np.uint8)
    n = flat.size
    codes = np.concatenate([_CODE[flat], np.full(k, 4, np.uint8)])
    valid = np.ones(n, bool)
    kc = np.zeros(n, np.uint32)
    for j in range(k):
        valid &= codes[j:j + n] < 4
        np.left_shift(kc, 2, out=kc)
        np.bitwise_or(kc, codes[j:j + n] & 3, out=kc)
    hist = np.bincount(kc[valid], minlength=4 ** k)
    masked = np.zeros(n, bool)
    log = []
    off = np.arange(k)
    for _ in range(iters):
        best = int(np.argmax(hist))                           # the first maximum: the smallest code
        cnt = int(hist[best])
        if cnt == 0:
            break
        log.append((kmer_str(best, k), cnt))
        occ = np.flatnonzero(valid & (kc == best))
        cov = np.unique((occ[:, None] + off).ravel())
        masked[cov] = True
        hit = np.unique((cov[:, None] - off).ravel())
        hit = hit[(hit >= 0) & valid[np.maximum(hit, 0)]]
        hist -= np.bincount(kc[hit], minlength=4 ** k)
        valid[hit] = False
    out = flat.copy()
    out[masked] = ord("N")
    pos, res = 0, []
    for s in seqs:
        res.append(out[pos:pos + len(s)].tobytes())
        pos += len(s) + 1
    return write_fasta(heads, res), log


def brute_force_choice(data, k):
    """(kmer, count) of the most frequent k-mer with the smallest-code tie rule, counted with a dict, or None"""
    from collections import Counter
    cnt = Counter()
    for s in read_fasta(data)[1]:
        u = s.upper()
        for i in range(len(u) - k + 1):
            w = u[i:i + k]
            if all(c in b"ACGT" for c in w):
                cnt[w] += 1
    if not cnt:
        return None
    top = max(cnt.values())
    return min(w for w, c in cnt.items() if c == top).decode(), top


# ---------------------------------------------------------------- the emulator

_lib = None


def emu_lib():
    global _lib
    if _lib is None:
        src = os.path.join(EMUL_DIR, "emul_mask.cpp")
        out = os.path.join(EMUL_DIR, "libunc_emul_mask.so")
        csrc = os.path.join(ROOT, "uncalled_b200", "csrc")
        deps = [src, os.path.join(EMUL_DIR, "warp_emul.hpp")] + \
            [os.path.join(csrc, f) for f in ("unc_mask.cuh", "unc_mask_host.hpp", "unc_device.cuh", "unc_warp.cuh")]
        if not (os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps)):
            subprocess.run(["g++", "-O2", "-g", "-std=c++17", "-ffp-contract=off", "-DUNC_EMUL", "-DK2_MAXSEG=16u", "-fPIC",
                            "-shared", "-I" + EMUL_DIR, "-I" + csrc, "-o", out, src], check=True, capture_output=True)
        L = C.CDLL(out)
        L.emu_mask_internal.argtypes = [C.c_char_p, C.c_char_p, C.c_uint32, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p,
                                        C.POINTER(C.c_uint32)]
        _lib = L
    return _lib


def emu_mask_internal(fasta, out, k, iters, n_threads):
    """(status, [(kmer, count), ...]) of the device source on the CPU, with CTAs of n_threads"""
    codes, counts, done = np.zeros(iters, np.uint64), np.zeros(iters, np.uint64), C.c_uint32()
    rc = emu_lib().emu_mask_internal(fasta.encode(), out.encode(), k, iters, n_threads, codes.ctypes.data,
                                     counts.ctypes.data, C.byref(done))
    return rc, [(kmer_str(codes[i], k), int(counts[i])) for i in range(done.value)]
