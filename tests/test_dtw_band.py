"""The banded DTW sweep without a GPU: the C restatement (oracle/unc_oracle_dtw_band.c) against the reference's DTW classes
and the `dtw` golden when the band is the whole matrix, the two facts that follow from the band's definition, the kernel
source (unc_dtw_band.cuh) under the warp emulator against the restatement, and the argument checks."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import dtwalignlib as DA
import dtwbandlib as B
import orclib

u64p = C.POINTER(C.c_uint64)
u16p = C.POINTER(C.c_uint16)
f32p = C.POINTER(C.c_float)


def full(means, km, kind, w):
    """the full sweep: orc_dtw (pinned to the reference's classes by tests/test_dtw.py), subseq NONE"""
    L = orclib.orc()
    L.orc_dtw.argtypes = [C.POINTER(orclib.OrcModel), C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, f32p, C.c_uint32, u16p,
                          C.c_uint32, u64p, u64p, f32p]
    p = np.zeros(2 * (len(means) + len(km)), np.uint64)
    n, s = C.c_uint64(), C.c_float()
    _, M = B.orc()
    assert L.orc_dtw(C.byref(M), kind, 0, w[0], w[1], w[2], means.ctypes.data_as(f32p), len(means), km.ctypes.data_as(u16p),
                     len(km), p.ctypes.data_as(u64p), C.byref(n), C.byref(s)) == 0
    return p[:2 * n.value].reshape(-1, 2).copy(), s.value


def in_band(path, R, C_, W):
    lo, hi = B.band_rows(R, C_, W)
    j, i = path[:, 0].astype(np.int64), path[:, 1].astype(np.int64)
    return bool(np.all((lo[j] <= i) & (i <= hi[j])))


def seeded_problems(seed, n=60):
    """shapes of dtwbandlib.SHAPES plus random ones: narrow bands on long diagonals, noisy and uniform events"""
    rng = np.random.default_rng(seed)
    out = list(B.shape_problems(seed))
    for _ in range(n):
        r, c = int(rng.integers(1, 300)), int(rng.integers(1, 300))
        w = int(rng.choice([1, 2, 3, 5, 8, 16, 40, 400]))
        out.append((B.problem(rng, r, c, rng.random() < 0.75, noise=float(rng.choice([1.0, 2.5, 6.0]))), w))
    return out


# ---------------------------------------------------------------- the restatement with the band = the whole matrix

def test_full_band_restatement_equals_reference_classes():
    """We >= R - 1: path and score equal the reference's DTWr94p / DTWr94d (live from oracle/_ref where it is built, else
    the full restatement pinned to them)"""
    live = orclib.ref_available()
    if live:
        R = orclib.ref()
        R.ref_dtw.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, f32p, C.c_uint32, u16p, C.c_uint32, u64p, u64p,
                              f32p, f32p]
    rng = np.random.default_rng(7)
    for t in range(150):
        nr, nc = int(rng.integers(1, 90)), int(rng.integers(1, 90))
        kind, w = int(rng.integers(0, 2)), B.WEIGHTS[t % 3]
        means, km = B.problem(rng, nr, nc, rng.random() < 0.7)
        band = nr - 1 + int(rng.integers(0, 3)) if nr > 1 else 1
        path, score, _ = B.restated(means, km, band, kind, w)
        if live:
            want = np.zeros(2 * (nr + nc), np.uint64)
            n, s, ms = C.c_uint64(), C.c_float(), C.c_float()
            R.ref_dtw(kind, 0, w[0], w[1], w[2], means.ctypes.data_as(f32p), nc, km.ctypes.data_as(u16p), nr,
                      want.ctypes.data_as(u64p), C.byref(n), C.byref(s), C.byref(ms))
            wp, ws = want[:2 * n.value].reshape(-1, 2), s.value
        else:
            wp, ws = full(means, km, kind, w)
        assert score == ws and np.array_equal(path, wp), (t, nr, nc, kind)


def test_full_band_restatement_equals_dtw_golden(tmp_path):
    """every entry of tests/golden/dtw_align_golden.json (DTWr94d with float abs, {NONE, 1, 1, 1}), bit for bit"""
    golden = json.load(open(DA.GOLDEN))
    prefix = orclib.materialise_example_index(str(tmp_path))
    raw = np.load(os.path.join(DA.ROOT, "tests", "golden", "example_read.npz"))["raw"]
    g = DA.read_genome(prefix)
    contig, (_, clen) = next(iter(g[1].items()))
    sets = {"example": (g, [(n, raw[st:(en or len(raw))], contig, rs, re, f) for n, st, en, rs, re, f in DA.example_queries(len(raw), clen)])}
    sprefix, codes = DA.multi_contig_genome(str(tmp_path))
    sets["synthetic"] = (DA.read_genome(sprefix), DA.synthetic_cases(codes))
    n = 0
    for key, (gen, cases) in sets.items():
        for name, sig, ctg, rs, re, fwd in cases:
            want = golden[key][name]
            if want["status"]:
                continue
            rec = DA.oracle_align(gen, sig, ctg, rs, re, fwd)
            path, score, _ = B.restated(rec["_means"], rec["_kmers"], len(rec["_kmers"]), 2, (1.0, 1.0, 1.0))
            assert DA.f32_bits(score) == want["score_bits"], name
            assert len(path) == want["path_len"] and DA.digest_path(path) == want["path_sha"], name
            n += 1
    assert n >= 30


# ---------------------------------------------------------------- facts (a) and (b)

@pytest.mark.parametrize("kind", [0, 1, 2])
def test_facts_of_the_definition(kind):
    """(a) We >= R - 1: the banded sweep is the full one, breadcrumbs included (against k_dtw's routine under the emulator);
    (b) otherwise the banded score is never below the full one, and equals it, path and all, when the full path is in band"""
    n_full = n_inside = n_worse = 0
    for seed in range(4):
        for (means, km), W in seeded_problems(100 * kind + seed):
            R, C_ = len(km), len(means)
            w = B.WEIGHTS[seed % 2]                     # the two weight sets of the DTW_* presets
            path, score, bc = B.restated(means, km, W, kind, w, want_bc=True)
            if kind < 2:
                fp, fs = full(means, km, kind, w)
            else:
                fp, fs, _ = B.restated(means, km, max(R, 1), 2, w)
            if B.effective_width(R, C_, W) >= R - 1:
                (ep, es, ebc), = B.emulated([(means, km)], 0, kind, w, n_threads=64, want_bc=True)
                assert score == fs == es and np.array_equal(path, fp) and np.array_equal(path, ep)
                assert np.array_equal(bc, ebc.reshape(R, C_).T.ravel())          # column-major band = transposed matrix
                n_full += 1
            else:
                assert np.float32(score) >= np.float32(fs), (R, C_, W)
                if in_band(fp, R, C_, W):
                    assert DA.f32_bits(score) == DA.f32_bits(fs) and np.array_equal(path, fp), (R, C_, W)
                    n_inside += 1
                else:
                    n_worse += score > fs
    assert n_full >= 20 and n_inside >= 20 and n_worse >= 5, (n_full, n_inside, n_worse)


def test_band_geometry():
    """the effective width covers the diagonal's slope, each column's rows meet the previous column's, both corners are in"""
    for R, C_, W in B.SHAPES + [(5000, 3, 1), (3, 5000, 1), (1000, 999, 1), (999, 1000, 1)]:
        lo, hi = B.band_rows(R, C_, W)
        assert lo[0] == 0 and hi[-1] == R - 1
        assert np.all(lo[1:] <= hi[:-1] + 1) and np.all(lo[1:] >= lo[:-1]) and np.all(hi[1:] >= hi[:-1])
        assert int(B.emu().emu_dtw_band_cells(R, C_, W)) == int((hi - lo + 1).sum())


# ---------------------------------------------------------------- the kernel source under the emulator

@pytest.mark.parametrize("n_threads", [32, 64, 96, 256])
def test_emulated_kernel_equals_restatement(n_threads):
    """every problem of the CPU set, at this CTA size, with both weight sets and the three cost kinds: path, score and
    in-band breadcrumbs"""
    probs = seeded_problems(n_threads, n=30)
    for kind in (0, 1, 2):
        w = B.WEIGHTS[kind % 2]
        for W in sorted({w_ for _, w_ in probs}):
            group = [p for p, w_ in probs if w_ == W]
            got = B.emulated(group, W, kind, w, n_threads=n_threads, want_bc=True)
            for (means, km), (path, score, bc) in zip(group, got):
                wp, ws, wbc = B.restated(means, km, W, kind, w, want_bc=True)
                assert score == ws and np.array_equal(path, wp) and np.array_equal(bc, wbc), (len(km), len(means), W, kind)


def test_emulated_kernel_on_tile_edges():
    """R and C at 0, 1 and 7 mod 8 (plus tile multiples of 8) with bands narrower than a tile and as wide as several"""
    rng = np.random.default_rng(77)
    sizes = [8 * t + e for t in (1, 4, 9) for e in (0, 1, 7)]
    probs = [B.problem(rng, r, c) for r in sizes for c in sizes]
    for W in (1, 4, 9, 20):
        got = B.emulated(probs, W, 0, B.WEIGHTS[0], n_threads=64)
        for (means, km), (path, score, _) in zip(probs, got):
            wp, ws, _ = B.restated(means, km, W, 0, B.WEIGHTS[0])
            assert score == ws and np.array_equal(path, wp), (len(km), len(means), W)


def test_emulated_kernel_on_long_reads():
    """three reads over 50 000 kept means, through the aligner's stages (event detection, mask, k-mers, normalisation:
    the restatement pinned to the device stages by tests/test_dtw_align.py), then the banded sweep at W = 64"""
    import tempfile
    d = tempfile.mkdtemp()
    prefix, codes = DA.multi_contig_genome(d)
    g = DA.read_genome(prefix)
    rng = np.random.default_rng(31)
    for contig, st, ln, fwd in (("chrB", 1000, 36000, True), ("chrA", 5000, 34000, False), ("chrC", 2000, 40000, True)):
        sig = DA.span_signal(codes[contig][st:st + ln], fwd, rng)
        rec = DA.oracle_align(g, sig, contig, st, st + ln, fwd)
        assert rec["status"] == 1 and rec["n_kept"] > DA.MAX_MEANS               # skipped by the full sweep
        means, km = rec["_means"], rec["_kmers"]
        (path, score, _), = B.emulated([(means, km)], 64, 2, (1.0, 1.0, 1.0), n_threads=32)
        wp, ws, _ = B.restated(means, km, 64, 2, (1.0, 1.0, 1.0))
        assert score == ws and np.array_equal(path, wp), contig
        assert path[0, 0] == len(means) - 1 and path[0, 1] == len(km) - 1 and not path[-1].any()


# ---------------------------------------------------------------- the workspace plan (unc_dtw_plan.hpp)

def test_workspace_plan_bytes_and_packing():
    """the plan's byte count equals the restatement (dtwbandlib.sweep_bytes) over shapes at 1 x 1, R = 1, C = 1, tile edges
    and W >= R - 1, for both sweeps; the aligner's packing keeps query order, closes a launch only when the next query
    would pass the budget, keeps every launch within it, skips exactly the queries over it on their own and puts every
    other query in one launch"""
    sizes = [1, 2, 7, 8, 9, 15, 16, 17, 63, 64, 65, 200]
    shapes = [(r, c) for r in sizes for c in sizes] + [(r, c) for r, c, _ in B.SHAPES]
    for W in (0, 1, 3, 8, 64, 250):
        for R, C_ in shapes:
            assert int(B.emu().emu_dtw_plan_bytes(R, C_, W)) == B.sweep_bytes([(R, C_)], W), (R, C_, W)

    def check(shapes, W, budget):
        launch, n = B.pack(shapes, W, budget)
        alone = [B.sweep_bytes([s], W) for s in shapes]
        assert [k for k in range(len(shapes)) if launch[k] == B.SKIP] == [k for k in range(len(shapes)) if alone[k] > budget]
        kept = [(k, l) for k, l in enumerate(launch) if l != B.SKIP]
        assert [l for _, l in kept] == sorted(l for _, l in kept) and {l for _, l in kept} == set(range(n))
        for l in range(n):
            ks = [k for k, x in kept if x == l]
            assert B.sweep_bytes([shapes[k] for k in ks], W) <= budget, (l, ks)
            if l + 1 < n:                              # closed because the next query (maybe one skipped) did not fit
                assert B.sweep_bytes([shapes[k] for k in ks + [ks[-1] + 1]], W) > budget, (l, ks)
        return launch, n

    rng = np.random.default_rng(12)
    for trial in range(40):
        shapes = [(int(rng.integers(1, 3000)), int(rng.integers(1, 3000))) for _ in range(int(rng.integers(1, 30)))]
        W = int(rng.choice([0, 1, 8, 64]))
        alone = sorted(B.sweep_bytes([s], W) for s in shapes)
        budget = int(rng.choice([alone[0] - 1, alone[len(alone) // 2], alone[-1], 3 * alone[-1], 100 * alone[-1]]))
        check(shapes, W, budget)
    launch, n = check(B.LONG_READ_SHAPES, 64, B.small_budget(B.LONG_READ_SHAPES, 64))
    assert launch.count(B.SKIP) == 1 and n >= 2


# ---------------------------------------------------------------- argument checks

def test_restatement_rejects_what_the_band_does_not_define():
    rng = np.random.default_rng(5)
    means, km = B.problem(rng, 20, 30)
    for sub in (1, 2):
        with pytest.raises(ValueError, match="rc=-3"):
            B.restated(means, km, 4, 0, subseq=sub)
    with pytest.raises(ValueError, match="rc=-3"):
        B.restated(means, km, 0, 0)


def test_banded_entry_point_argument_errors():
    """unc_dtw_batch_banded: band 0 and subseq ROW / COL are argument errors, reported before any device is needed"""
    import uncalled_b200._native as N
    from uncalled_b200 import dtw as D
    rng = np.random.default_rng(6)
    probs = [B.problem(rng, 20, 30)]
    L = N.lib()
    L.unc_dtw_batch_banded.argtypes = [C.c_void_p, C.c_int, C.POINTER(D.DTWParams), C.c_uint32] + [C.c_void_p] * 8 + [C.c_uint32]
    means, km = probs[0]
    moff, koff, poff = (np.array([0, n], np.uint64) for n in (30, 20, 50))
    path, plen, score = np.zeros(100, np.uint64), np.zeros(1, np.uint64), np.zeros(1, np.float32)
    for prm, band, msg in ((D.DTW_EVENT_GLOB, 0, "band must be at least 1"), (D.DTW_EVENT_QSUB, 8, "subseq must be 0"),
                           (D.DTW_EVENT_RSUB, 8, "subseq must be 0")):
        rc = L.unc_dtw_batch_banded(D.model_table().ctypes.data, 0, C.byref(prm), 1, means.ctypes.data, moff.ctypes.data,
                                    km.ctypes.data, koff.ctypes.data, path.ctypes.data, poff.ctypes.data, plen.ctypes.data,
                                    score.ctypes.data, band)
        assert rc != 0
        assert msg in L.unc_last_error().decode()
    with pytest.raises(ValueError):
        D.dtw_batch(probs, D.DTW_EVENT_GLOB, band=-1)


# ---------------------------------------------------------------- the CLI's host side

FAST5 = os.path.join(DA.ROOT, "tests", "golden", "fast5", "example_single.fast5")
READ_ID = "f41a60f7-de4a-4b17-9f54-387e52d60b65"


def run_cli(tmp_path, prefix, line, extra=()):
    qf = tmp_path / "queries.txt"
    qf.write_text(line + "\n")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    return subprocess.run([sys.executable, "-m", "uncalled_b200", "dtw", prefix, FAST5, "--queries", str(qf)] + list(extra),
                          capture_output=True, text=True, cwd=DA.ROOT, env=env, timeout=300)


def test_cli_band_keeps_host_side_output(tmp_path):
    """the host-side skips print the same with and without --band; a negative band ends the command with status 1"""
    prefix = orclib.materialise_example_index(str(tmp_path))
    line = READ_ID + " 0 40000 Escherichia_coli_chromosome:2400000-2410000 0 100 +"
    plain = run_cli(tmp_path, prefix, line)
    banded = run_cli(tmp_path, prefix, line, ["--band", "64"])
    assert plain.returncode == banded.returncode == 0
    assert (plain.stdout, plain.stderr) == (banded.stdout, banded.stderr)
    assert "rd_en past the end" in plain.stderr
    bad = run_cli(tmp_path, prefix, line, ["--band", "-3"])
    assert bad.returncode == 1 and bad.stdout == "" and "--band" in bad.stderr
