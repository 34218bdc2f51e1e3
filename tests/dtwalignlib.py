"""Inputs and checkers of the signal-to-span aligner (`uncalled_b200 dtw`, the reference's dtw_test driver): a .pac/.ann
writer for synthetic genomes, seeded reads of reference spans, and the oracle's and the reference's own dtw_test loop
body on one query (oracle/unc_oracle_dtw_align.c orc_dtw_align, oracle/_ref/libref_dtw_align.so ref_dtw_align)."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np

import orclib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "dtw_align_golden.json")
MODEL_TABLE = os.path.join(ROOT, "uncalled_b200", "data", "r94_5mer_template.f32")
CONTIGS = (("chrA", 60000, 11), ("chrB", 90000, 12), ("chrC", 50000, 13))
MAX_MEANS = 50000


def write_genome(prefix, contigs):
    """<prefix>.pac/.ann/.amb of contigs [(name, base codes 0..3)] as bwa writes them (bns_dump, 2 bits per base, first
    base in the high bits, then the count byte)."""
    seq = np.concatenate([c for _, c in contigs]).astype(np.uint8)
    n = len(seq)
    pad = np.zeros((-n) % 4, np.uint8)
    q = np.concatenate([seq, pad]).reshape(-1, 4)
    pac = (q[:, 0] << 6) | (q[:, 1] << 4) | (q[:, 2] << 2) | q[:, 3]
    tail = np.array([0, n % 4] if n % 4 == 0 else [n % 4], np.uint8)
    np.concatenate([pac.astype(np.uint8), tail]).tofile(prefix + ".pac")
    with open(prefix + ".ann", "w") as f:
        f.write("%d %d 11\n" % (n, len(contigs)))
        off = 0
        for name, c in contigs:
            f.write("0 %s (null)\n%d %d 0\n" % (name, off, len(c)))
            off += len(c)
    with open(prefix + ".amb", "w") as f:
        f.write("%d %d 0\n" % (n, len(contigs)))
    return prefix


def multi_contig_genome(dirname):
    """The three-contig test genome (seeded)."""
    gens = [(name, np.random.default_rng(seed).integers(0, 4, n, dtype=np.uint8)) for name, n, seed in CONTIGS]
    return write_genome(os.path.join(dirname, "multi"), gens), dict(gens)


def read_genome(prefix):
    """(pac bytes, {name: (offset, length)}) of a .pac/.ann pair"""
    pac = np.fromfile(prefix + ".pac", dtype=np.uint8)
    contigs = {}
    with open(prefix + ".ann") as f:
        _, n_seqs, _ = f.readline().split()
        for _ in range(int(n_seqs)):
            name = f.readline().split()[1]
            off, ln, _ = f.readline().split()
            contigs[name] = (int(off), int(ln))
    return pac, contigs


def span_signal(codes, fwd, rng, flat=()):
    """A seeded r9.4-like signal of the bases `codes` read on strand fwd (dwell 1 + Geometric(1/7.9) samples per k-mer,
    noise of the k-mer's stdv).  flat: (start, length) k-mer index ranges replaced by a pore-stall level that only
    alternates by 2 pA, so the event windows there have a stdv below 5 pA."""
    tab = np.fromfile(MODEL_TABLE, dtype=np.float32).reshape(1024, 2).astype(np.float64)
    s = codes if fwd else (3 - codes[::-1])
    n = len(s) - 4
    k = np.zeros(n, np.int64)
    for i in range(5):
        k = (k << 2) | s[i:i + n]
    lv, sd = tab[k, 0].copy(), tab[k, 1].copy()
    for st, ln in flat:
        lv[st:st + ln] = 70.0 + 2.0 * (np.arange(ln) % 2)
        sd[st:st + ln] = 0.3
    dwell = 1 + rng.geometric(1.0 / 7.9, size=n)
    idx = np.repeat(np.arange(n), dwell)
    return (lv[idx] + rng.standard_normal(len(idx)) * sd[idx]).astype(np.float32)


def digest_path(path):
    """SHA-256 of a path's (event index, k-mer index) columns as little-endian u64 pairs, end cell first"""
    return hashlib.sha256(np.ascontiguousarray(path, dtype="<u8").tobytes()).hexdigest()


def f32_bits(x):
    return int(np.float32(x).view(np.uint32))


ORACLE_DIR = os.path.join(ROOT, "oracle")
REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libref_dtw_align.so")
_orc = None
_ref = None


def ref_available():
    """oracle/_ref holds the reference's own dtw_test loop body (built by oracle/dtw_align.mk)"""
    return os.path.exists(REF_LIB)


def orc():
    """the C restatement (oracle/unc_oracle_dtw_align.c), its parameters and the template model"""
    global _orc
    if _orc is None:
        base = orclib.orc()
        path = os.path.join(ORACLE_DIR, "libunc_oracle_dtw_align.so")
        if not os.path.exists(path):
            subprocess.run(["make", "-C", ORACLE_DIR, "-f", "dtw_align.mk", "libunc_oracle_dtw_align.so"], check=True,
                           capture_output=True)
        L = C.CDLL(path)
        L.orc_dtw_align.argtypes = [C.POINTER(orclib.OrcParams), C.POINTER(orclib.OrcModel), C.c_void_p, C.c_uint32, C.c_void_p,
                                    C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_span_kmers.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_int, C.c_void_p]
        L.orc_full_mask.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.orc_full_mask.restype = C.c_uint32
        L.orc_span_target.argtypes = [C.POINTER(orclib.OrcModel), C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        L.orc_normalize_to.argtypes = [C.c_float, C.c_float, C.c_void_p, C.c_uint32, C.c_void_p]
        P = orclib.OrcParams()
        base.orc_params_default(C.byref(P))
        M = orclib.OrcModel()
        tab = np.fromfile(MODEL_TABLE, dtype=np.float32)
        base.orc_model_init(C.byref(M), tab.ctypes.data_as(orclib.f32p), 0)
        _orc = (L, P, M)
    return _orc


def span_kmers(genome, contig, rf_st, rf_en, fwd):
    """oracle: the span's k-mers from the .pac"""
    L, _, _ = orc()
    pac, contigs = genome
    out = np.zeros(max(rf_en - rf_st - 4, 1), np.uint16)
    L.orc_span_kmers(pac.ctypes.data, contigs[contig][0] + rf_st, rf_en - rf_st, int(fwd), out.ctypes.data)
    return out[:rf_en - rf_st - 4]


def oracle_align(genome, sig, contig, rf_st, rf_en, fwd):
    """orc_dtw_align on one query: dict of the golden's fields (plus the means, k-mers and path)"""
    L, P, M = orc()
    sig = np.ascontiguousarray(sig, dtype=np.float32)
    km = span_kmers(genome, contig, rf_st, rf_en, fwd)
    n = len(sig)
    ne, nk, tgt = C.c_uint32(), C.c_uint32(), np.zeros(2, np.float32)
    means = np.zeros(n + 1, np.float32)
    path = np.zeros((n + len(km) + 1, 2), np.uint64)
    plen, score = C.c_uint64(), C.c_float()
    rc = L.orc_dtw_align(C.byref(P), C.byref(M), sig.ctypes.data, n, km.ctypes.data, len(km), C.byref(ne), C.byref(nk),
                         tgt.ctypes.data, means.ctypes.data, path.ctypes.data, C.byref(plen), C.byref(score))
    return _record(rc, ne.value, nk.value, tgt, means[:nk.value], km, path[:plen.value], score.value)


def ref_align(prefix, sig, contig, rf_st, rf_en, fwd):
    """oracle/_ref: the reference's own code (oracle/ref_build/ref_dtw_align.cpp) on one query"""
    global _ref
    if _ref is None:
        _ref = C.CDLL(REF_LIB)
    R = _ref
    R.ref_dtw_align.argtypes = [C.c_char_p, C.c_void_p, C.c_uint32, C.c_char_p, C.c_uint64, C.c_uint64, C.c_int, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    sig = np.ascontiguousarray(sig, dtype=np.float32)
    n, nkm = len(sig), rf_en - rf_st - 4
    ne, nk, tgt = C.c_uint32(), C.c_uint32(), np.zeros(2, np.float32)
    means = np.zeros(n + 1, np.float32)
    km = np.zeros(max(nkm, 1), np.uint16)
    path = np.zeros((n + nkm + 1, 2), np.uint64)
    plen, score, ms = C.c_uint64(), C.c_float(), C.c_float()
    rc = R.ref_dtw_align(prefix.encode(), sig.ctypes.data, n, contig.encode(), rf_st, rf_en, int(fwd), C.byref(ne), C.byref(nk),
                         tgt.ctypes.data, means.ctypes.data, km.ctypes.data, C.byref(score), C.byref(ms), path.ctypes.data,
                         C.byref(plen))
    rec = _record(rc, ne.value, nk.value, tgt, means[:nk.value], km[:nkm], path[:plen.value], score.value)
    if rc == 0:
        assert rec["mean_score_bits"] == f32_bits(ms.value)
    return rec


def _record(rc, ne, nk, tgt, means, km, path, score):
    rec = {"status": int(rc), "n_events": int(ne), "n_kept": int(nk), "tgt_bits": [f32_bits(tgt[0]), f32_bits(tgt[1])],
           "means_sha": hashlib.sha256(np.ascontiguousarray(means, "<f4").tobytes()).hexdigest(),
           "kmers_sha": hashlib.sha256(np.ascontiguousarray(km, "<u2").tobytes()).hexdigest()}
    if rc == 0:
        ms = np.float32(score) / np.float32(len(path))
        rec.update(score_bits=f32_bits(score), mean_score_bits=f32_bits(ms), mean_score="%g" % float(ms),
                   path_len=int(len(path)), path_sha=digest_path(path))
    rec["_means"], rec["_kmers"], rec["_path"] = means, km, path
    return rec


def public(rec):
    """the fields a golden entry stores"""
    return {k: v for k, v in rec.items() if not k.startswith("_")}


# ---------------------------------------------------------------- the golden's inputs

def example_queries(n_raw, contig_len):
    """(name, rd_st, rd_en, rf_st, rf_en, fwd) of the example read against the example index: the whole read, sample
    sub-ranges, both strands, spans at the contig's start and end.  The read maps to [6938, 6976) of the events' bases
    on the - strand (tests/golden/example_paf.json), about [6000, 9500) in bases."""
    L = contig_len
    return [("whole_minus", 0, 0, 6000, 9500, False),
            ("whole_plus", 0, 0, 6000, 9500, True),
            ("head_minus", 0, 8000, 8600, 9500, False),
            ("mid_minus", 8000, 16000, 7700, 8800, False),
            ("tail_to_end", 24000, 0, 6000, 7000, False),
            ("contig_start", 0, 6000, 0, 700, True),
            ("contig_end", 0, 6000, L - 700, L, False),
            ("five_bases", 100, 900, 5000, 5005, True)]


def synthetic_cases(genome_codes, seed=5, n=24):
    """seeded reads of spans of the multi-contig genome: both strands, flat (pore-stall) stretches at and around the
    mask's 25-event windows, a span at each contig's ends.  (name, signal, contig, rf_st, rf_en, fwd)"""
    rng = np.random.default_rng(seed)
    names = sorted(genome_codes)
    out = []
    for i in range(n):
        contig = names[i % len(names)]
        codes = genome_codes[contig]
        ln = int(rng.integers(300, 1500))
        st = 0 if i % 8 == 3 else (len(codes) - ln if i % 8 == 5 else int(rng.integers(0, len(codes) - ln)))
        fwd = bool(i % 2)
        flat = []
        if i % 3 == 0:
            for _ in range(int(rng.integers(1, 4))):
                flat.append((int(rng.integers(0, ln - 80)), int(rng.choice([3, 12, 24, 25, 26, 40]))))
        sig = span_signal(codes[st:st + ln], fwd, rng, flat)
        out.append(("syn%02d" % i, sig, contig, st, st + ln, fwd))
    return out
