"""The signal-to-span aligner (`uncalled_b200 dtw`, the reference's dtw_test driver) without a GPU: the C oracle against
the golden taken from the reference's own code (and against oracle/_ref live where it is built), the device stages
(a)-(e) under the warp emulator against the oracle, and the checks that reject a query file or skip a query before the
device is touched."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import dtwalignlib as D
import orclib

ROOT = D.ROOT
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
FAST5 = os.path.join(ROOT, "tests", "golden", "fast5", "example_single.fast5")
READ_ID = "f41a60f7-de4a-4b17-9f54-387e52d60b65"


@pytest.fixture(scope="module")
def golden():
    with open(D.GOLDEN) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def example(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("ex"))
    prefix = orclib.materialise_example_index(d)
    raw = np.load(os.path.join(ROOT, "tests", "golden", "example_read.npz"))["raw"]
    g = D.read_genome(prefix)
    contig, (_, clen) = next(iter(g[1].items()))
    cases = [(name, raw[st:(en or len(raw))], contig, rs, re, fwd) for name, st, en, rs, re, fwd in D.example_queries(len(raw), clen)]
    return prefix, g, cases


@pytest.fixture(scope="module")
def synthetic(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("syn"))
    prefix, codes = D.multi_contig_genome(d)
    return prefix, D.read_genome(prefix), D.synthetic_cases(codes)


def test_oracle_reproduces_golden(golden, example, synthetic):
    for key, (prefix, g, cases) in (("example", example), ("synthetic", synthetic)):
        assert len(cases) == len(golden[key])
        for name, sig, contig, rs, re, fwd in cases:
            assert D.public(D.oracle_align(g, sig, contig, rs, re, fwd)) == golden[key][name], name


@pytest.mark.skipif(not D.ref_available(), reason="oracle/_ref/libref_dtw_align.so is not built")
def test_reference_reproduces_golden_live(golden, example, synthetic):
    for key, (prefix, g, cases) in (("example", example), ("synthetic", synthetic)):
        for name, sig, contig, rs, re, fwd in cases:
            assert D.public(D.ref_align(prefix, sig, contig, rs, re, fwd)) == golden[key][name], name


# ---------------------------------------------------------------- the device stages under the emulator

_emu = None


def emu():
    global _emu
    if _emu is None:
        src = os.path.join(EMUL_DIR, "emul_dtw_align.cpp")
        out = os.path.join(EMUL_DIR, "libunc_emul_dtw_align.so")
        csrc = os.path.join(ROOT, "uncalled_b200", "csrc")
        deps = [src, os.path.join(EMUL_DIR, "warp_emul.hpp")] + [os.path.join(csrc, f) for f in (
            "unc_dtw_align.cuh", "unc_k1.cuh", "unc_stream.cuh", "unc_device.cuh", "unc_warp.cuh", "unc_host_index.hpp")]
        if not (os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(x) for x in deps)):
            subprocess.run(["g++", "-O2", "-g", "-std=c++17", "-ffp-contract=off", "-DUNC_EMUL", "-DK2_MAXSEG=16u", "-fPIC",
                            "-shared", "-I" + EMUL_DIR, "-I" + csrc, "-o", out, src], check=True, capture_output=True)
        _emu = C.CDLL(out)
        _emu.emu_dtw_align_stages.argtypes = [C.c_uint32] + [C.c_void_p] * 15 + [C.c_int]
    return _emu


def emu_stages(g, cases, events=False, k1_warps=2):
    """cases: (name, signal or event means, contig, rf_st, rf_en, fwd).  Returns per case the oracle-record fields of
    stages (a)-(e) and the verdict."""
    import uncalled_b200._native as N   # noqa: F401  (MODEL_TABLE only)
    pac, contigs = g
    n = len(cases)
    lens = [len(c[1]) for c in cases]
    descs = (N.ReadDesc * n)()
    off = 0
    for i, L in enumerate(lens):
        descs[i].offset, descs[i].n_samples = off, L
        off += L
    flat = np.ascontiguousarray(np.concatenate([c[1] for c in cases]), dtype=np.float32)
    pac_st = np.array([contigs[c[2]][0] + c[3] for c in cases], np.uint64)
    nkm = np.array([c[4] - c[3] - 4 for c in cases], np.uint32)
    fwd = np.array([int(c[5]) for c in cases], np.uint32)
    stride = max(max(lens), 4)
    ne, nk, tgt = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(2 * n, np.float32)
    means = np.zeros((n, stride), np.float32)
    kmers = np.zeros(int(nkm.sum()) + 1, np.uint16)
    verdict = np.zeros(n, np.int32)
    tab = np.fromfile(D.MODEL_TABLE, dtype=np.float32)
    emu().emu_dtw_align_stages(n, descs, None if events else flat.ctypes.data, flat.ctypes.data if events else None,
                               pac.ctypes.data, pac_st.ctypes.data, nkm.ctypes.data, fwd.ctypes.data, tab.ctypes.data, stride,
                               ne.ctypes.data, nk.ctypes.data, tgt.ctypes.data, means.ctypes.data, kmers.ctypes.data,
                               verdict.ctypes.data, k1_warps)
    out, ko = [], 0
    for i in range(n):
        km = kmers[ko:ko + nkm[i]]
        ko += int(nkm[i])
        out.append({"n_events": int(ne[i]), "n_kept": int(nk[i]), "tgt_bits": [D.f32_bits(tgt[2 * i]), D.f32_bits(tgt[2 * i + 1])],
                    "means_sha": hashlib.sha256(np.ascontiguousarray(means[i, :nk[i]], "<f4").tobytes()).hexdigest(),
                    "kmers_sha": hashlib.sha256(np.ascontiguousarray(km, "<u2").tobytes()).hexdigest(),
                    "verdict": int(verdict[i])})
    return out


STAGE_KEYS = ("n_events", "n_kept", "tgt_bits", "means_sha", "kmers_sha")


@pytest.mark.parametrize("which", ["example", "synthetic"])
def test_emulated_stages_match_oracle(which, example, synthetic, golden):
    prefix, g, cases = example if which == "example" else synthetic
    got = emu_stages(g, cases)
    for c, r in zip(cases, got):
        want = golden[which][c[0]]
        assert {k: r[k] for k in STAGE_KEYS} == {k: want[k] for k in STAGE_KEYS}, c[0]
        assert r["verdict"] == want["status"], c[0]


def test_emulated_mask_around_window_boundaries(synthetic):
    """flat stretches of every length around the profiler's 25-event window, at the start, middle and end of a read"""
    prefix, g, _ = synthetic
    rng = np.random.default_rng(9)
    codes = np.random.default_rng(13).integers(0, 4, 50000, dtype=np.uint8)    # chrC
    cases = []
    for i, (st, ln) in enumerate([(0, 24), (0, 25), (0, 26), (40, 12), (40, 13), (40, 49), (40, 50), (150, 24), (150, 25),
                                  (176, 24), (175, 26), (100, 100)]):
        rs = 1000 + 300 * i
        span = codes[rs:rs + 205]
        cases.append(("b%02d" % i, D.span_signal(span, bool(i % 2), rng, [(st, ln)]), "chrC", rs, rs + 205, bool(i % 2)))
    got = emu_stages(g, cases)
    n_masked = 0
    for c, r in zip(cases, got):
        want = D.oracle_align(g, c[1], c[2], c[3], c[4], c[5])
        assert {k: r[k] for k in STAGE_KEYS} == {k: want[k] for k in STAGE_KEYS}, c[0]
        n_masked += r["n_kept"] < r["n_events"]
    assert n_masked >= 6


@pytest.mark.parametrize("n_means,verdict", [(50000, 0), (50001, 1)])
def test_skip_decision_at_the_limit(n_means, verdict, synthetic):
    """stages (b)-(e) on synthetic event means: 50 000 kept means are aligned, 50 001 are not (dtw_test.cpp:156)"""
    prefix, g, _ = synthetic
    ev = np.random.default_rng(n_means).normal(90, 15, n_means).astype(np.float32)   # window stdv far above 5: nothing masked
    r, = emu_stages(g, [("lim", ev, "chrA", 100, 1100, True)], events=True)
    L, _, M = D.orc()
    kept = np.zeros(n_means, np.float32)
    assert L.orc_full_mask(ev.ctypes.data, n_means, kept.ctypes.data) == n_means == r["n_kept"]
    km = D.span_kmers(g, "chrA", 100, 1100, True)
    mt, st = C.c_float(), C.c_float()
    L.orc_span_target(C.byref(M), km.ctypes.data, len(km), C.byref(mt), C.byref(st))
    out = np.zeros(n_means, np.float32)
    L.orc_normalize_to(mt, st, kept.ctypes.data, n_means, out.ctypes.data)
    assert r["means_sha"] == hashlib.sha256(out.astype("<f4").tobytes()).hexdigest()
    assert r["verdict"] == verdict


# ---------------------------------------------------------------- input checks, before the device

def run_cli(tmp_path, prefix, lines, extra=()):
    qf = tmp_path / "queries.txt"
    qf.write_text("".join(l + "\n" for l in lines))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")          # nothing below may need a device
    return subprocess.run([sys.executable, "-m", "uncalled_b200", "dtw", prefix, FAST5, "--queries", str(qf)] + list(extra),
                          capture_output=True, text=True, cwd=ROOT, env=env, timeout=300)


@pytest.mark.parametrize("line,msg", [
    (READ_ID + " 0 0 no_such_contig 0 100 +", "unknown contig"),
    (READ_ID + " 0 0 Escherichia_coli_chromosome:2400000-2410000 0 100", "expected 7 fields"),
    (READ_ID + " 0 x Escherichia_coli_chromosome:2400000-2410000 0 100 +", "non-negative integers"),
    (READ_ID + " 0 -5 Escherichia_coli_chromosome:2400000-2410000 0 100 +", "non-negative integers"),
    (READ_ID + " 0 0 Escherichia_coli_chromosome:2400000-2410000 0 100 *", "strand must be + or -"),
])
def test_rejected_query_files(tmp_path, example, line, msg):
    prefix = example[0]
    r = run_cli(tmp_path, prefix, [READ_ID + " 0 0 Escherichia_coli_chromosome:2400000-2410000 0 100 +", line])
    assert r.returncode == 1, r.stderr
    assert r.stdout == ""
    assert "Error:" in r.stderr and msg in r.stderr and ":2:" in r.stderr


@pytest.mark.parametrize("query,reason", [
    ("5000 5000 Escherichia_coli_chromosome:2400000-2410000 0 100 +", "empty sample range"),
    ("9000 100 Escherichia_coli_chromosome:2400000-2410000 0 100 +", "empty sample range"),
    ("0 40000 Escherichia_coli_chromosome:2400000-2410000 0 100 +", "rd_en past the end of the signal"),
    ("0 0 Escherichia_coli_chromosome:2400000-2410000 9000 10001 -", "rf_en past the end of the contig"),
    ("0 0 Escherichia_coli_chromosome:2400000-2410000 500 504 +", "reference span shorter than 5 bases"),
])
def test_skipped_queries_never_reach_the_device(tmp_path, example, query, reason):
    r = run_cli(tmp_path, example[0], [READ_ID + " " + query])
    assert r.returncode == 0, r.stderr
    assert r.stdout == ""
    assert "Skipping %s: %s\n" % (READ_ID, reason) in r.stderr


def test_later_query_line_replaces_earlier(tmp_path, example):
    r = run_cli(tmp_path, example[0], [READ_ID + " 0 0 Escherichia_coli_chromosome:2400000-2410000 6000 9500 -",
                 READ_ID + " 0 40000 Escherichia_coli_chromosome:2400000-2410000 0 100 +"])
    assert r.returncode == 0 and r.stdout == ""
    assert "rd_en past the end" in r.stderr
