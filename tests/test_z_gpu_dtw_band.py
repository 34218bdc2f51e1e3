"""The banded DTW sweep on the GPU: unc_dtw_batch_banded against the C restatement (oracle/unc_oracle_dtw_band.c, pinned
to the reference and to the kernel source under the emulator by tests/test_dtw_band.py), against unc_dtw_batch when the
band is the whole matrix, and DtwAligner(band=...) on reads the full sweep skips."""
import os
import subprocess
import sys

import numpy as np
import pytest

import dtwalignlib as DA
import dtwbandlib as B
import orclib

pytestmark = pytest.mark.gpu


def _held():
    import ctypes as C
    import uncalled_b200._native as N
    d, p, h = C.c_uint64(), C.c_uint64(), C.c_uint32()
    N.check(N.lib().unc_debug_held(C.byref(d), C.byref(p), C.byref(h)))
    return d.value, p.value, h.value


@pytest.fixture(scope="module", autouse=True)
def device():
    import uncalled_b200._native as N
    N.check(N.lib().unc_init(0))
    N.lib().unc_dtw_release()
    start = _held()
    yield
    N.lib().unc_dtw_release()
    assert _held() == start


def larger_problems(seed, n=220):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        r = int(np.exp(rng.uniform(np.log(50), np.log(6000))))
        c = max(1, int(r * rng.uniform(0.4, 2.5)))
        out.append(B.problem(rng, r, c, rng.random() < 0.85, noise=float(rng.choice([1.0, 2.5, 6.0]))))
    return out


@pytest.mark.parametrize("cost,kind", [("r94p", 0), ("r94d", 1)])
def test_banded_batch_equals_restatement(cost, kind):
    from uncalled_b200 import dtw as D
    from test_dtw_band import seeded_problems
    small = seeded_problems(500 + kind, n=60)
    big = larger_problems(600 + kind)
    cases = [(p, w) for p, w in small] + [(p, w) for p, w in zip(big, [1, 3, 8, 16, 64, 200, 1000] * 40)]
    for prm, w in ((D.DTW_EVENT_GLOB, B.WEIGHTS[0]), (D.DTW_RAW_GLOB, B.WEIGHTS[1])):
        for W in sorted({w_ for _, w_ in cases}):
            group = [p for p, w_ in cases if w_ == W]
            got = D.dtw_batch(group, prm, cost, band=W)
            for (means, km), (path, score) in zip(group, got):
                wp, ws, _ = B.restated(means, km, W, kind, w)
                assert score == ws and np.array_equal(path, wp), (cost, len(km), len(means), W)


def test_band_over_the_rows_equals_full_sweep():
    from uncalled_b200 import dtw as D
    probs = larger_problems(700, n=60)
    W = max(len(k) for _, k in probs)
    for cost in ("r94p", "r94d"):
        for prm in (D.DTW_EVENT_GLOB, D.DTW_RAW_GLOB):
            full = D.dtw_batch(probs, prm, cost)
            band = D.dtw_batch(probs, prm, cost, band=W)
            for (fp, fs), (bp, bs) in zip(full, band):
                assert fs == bs and np.array_equal(fp, bp)


@pytest.fixture(scope="module")
def long_reads(tmp_path_factory):
    """reads of 100 000 - 400 000 samples (over 50 000 kept means from about 270 000) and shorter ones, with the
    restatement's stages"""
    d = str(tmp_path_factory.mktemp("long"))
    prefix, codes = DA.multi_contig_genome(d)
    g = DA.read_genome(prefix)
    rng = np.random.default_rng(4242)
    cases = []
    for i, n_samp in enumerate([100000, 150000, 230000, 280000, 330000, 400000, 20000, 60000]):
        contig = ("chrA", "chrB", "chrC")[i % 3]
        ln = min(n_samp // 8 + 50, len(codes[contig]) - 1)
        st = int(rng.integers(0, len(codes[contig]) - ln))
        fwd = bool(i % 2)
        sig = DA.span_signal(codes[contig][st:st + ln], fwd, rng)[:n_samp]
        cases.append(("r%d" % i, sig, contig, st, st + ln, fwd))
    recs = [DA.oracle_align(g, *c[1:]) for c in cases]
    assert sum(r["status"] == 1 for r in recs) >= 3
    return prefix, cases, recs


def _align(prefix, cases, band, budget=0):
    from uncalled_b200.dtw import DtwAligner
    A = DtwAligner(prefix, budget=budget, band=band)
    got = A.align([(c[0], c[1], None, 0, 0, c[2], c[3], c[4], c[5]) for c in cases], paths=True)
    times = A.last_times()
    A.close()
    return got, times


@pytest.mark.parametrize("W", [64, 256])
def test_aligner_band_aligns_long_reads(long_reads, W):
    prefix, cases, recs = long_reads
    plain, _ = _align(prefix, cases, 0)
    got, (_, launches, cells) = _align(prefix, cases, W)
    want_cells = 0
    for g, p, r, c in zip(got, plain, recs, cases):
        assert (g.n_events, g.n_kept) == (r["n_events"], r["n_kept"]), c[0]
        assert p.skip == ("too many means" if r["status"] == 1 else None), c[0]
        assert g.skip is None, (c[0], g.skip)
        wp, ws, _ = B.restated(r["_means"], r["_kmers"], W, 2, (1.0, 1.0, 1.0))
        assert DA.f32_bits(g.score) == DA.f32_bits(ws) and np.array_equal(g.path[::-1], wp), c[0]
        assert DA.f32_bits(g.mean_score) == DA.f32_bits(np.float32(ws) / np.float32(len(wp)))
        assert np.array_equal(g.means, r["_means"]) and np.array_equal(g.kmers, r["_kmers"])
        lo, hi = B.band_rows(len(r["_kmers"]), len(r["_means"]), W)
        want_cells += int((hi - lo + 1).sum())
    assert cells == want_cells and launches >= 1


def _sweep_bytes(R, C_, W):
    """the aligner's workspace for one banded problem (SweepNeed::bytes in unc_dtw_align_host.inl): problem record,
    in-band breadcrumbs, hrow / vcol / corners, column offsets, path room, path length, score, queue; 256-byte aligned"""
    a = lambda x: (x + 255) // 256 * 256
    lo, hi = B.band_rows(R, C_, W)
    return a(56) + a(int((hi - lo + 1).sum())) + a(4 * (C_ + R + 3 * ((R + 7) // 8) + 8)) + a(8 * (C_ + 1)) + a(16 * (R + C_)) + \
        a(8) + a(4) + a(4)


def test_small_budget_skips_only_the_query_over_it(long_reads):
    prefix, cases, recs = long_reads
    W = 64
    need = [_sweep_bytes(len(r["_kmers"]), len(r["_means"]), W) for r in recs]
    big = int(np.argmax(need))
    budget = (sorted(need)[-2] + need[big]) // 2                    # room for every band but the largest
    got, (_, launches, _) = _align(prefix, cases, W, budget=budget)
    full, _ = _align(prefix, cases, W)
    for i, (g, f) in enumerate(zip(got, full)):
        if i == big:
            assert g.skip == "the DTW matrix exceeds the workspace budget"
            continue
        assert g.skip is None and g.score == f.score and np.array_equal(g.path, f.path), cases[i][0]
    assert launches >= 2


def test_cli_band_on_the_golden_example(tmp_path):
    """--band prints the restatement's numbers; without it the output is the full sweep's (the golden's)"""
    import json
    golden = json.load(open(DA.GOLDEN))["example"]
    prefix = orclib.materialise_example_index(str(tmp_path))
    raw = np.load(os.path.join(DA.ROOT, "tests", "golden", "example_read.npz"))["raw"]
    g = DA.read_genome(prefix)
    contig, (_, clen) = next(iter(g[1].items()))
    fast5 = os.path.join(DA.ROOT, "tests", "golden", "fast5", "example_single.fast5")
    read_id = "f41a60f7-de4a-4b17-9f54-387e52d60b65"
    for name, st, en, rs, re, fwd in DA.example_queries(len(raw), clen)[:4]:
        qf = tmp_path / (name + ".q")
        qf.write_text("%s %d %d %s %d %d %s\n" % (read_id, st, en, contig, rs, re, "+" if fwd else "-"))
        rec = DA.oracle_align(g, raw[st:(en or len(raw))], contig, rs, re, fwd)
        outs = {}
        for W in (0, 16):
            pp = str(tmp_path / ("%s_%d_" % (name, W)))
            r = subprocess.run([sys.executable, "-m", "uncalled_b200", "dtw", prefix, fast5, "--queries", str(qf), "--path-prefix", pp]
                               + (["--band", str(W)] if W else []), capture_output=True, text=True, cwd=DA.ROOT, timeout=600)
            assert r.returncode == 0, r.stderr
            outs[W] = (r.stdout.split("\t")[:2], open(pp + read_id + ".txt").read())
        assert outs[0][0] == [read_id, golden[name]["mean_score"]], name
        wp, ws, _ = B.restated(rec["_means"], rec["_kmers"], 16, 2, (1.0, 1.0, 1.0))
        assert outs[16][0] == [read_id, "%g" % float(np.float32(ws) / np.float32(len(wp)))], name
        lines = outs[16][1].split("\n")[:-1]
        assert [tuple(int(x) for x in l.split("\t")[:2]) for l in lines] == [tuple(int(x) for x in p) for p in wp[::-1]], name
