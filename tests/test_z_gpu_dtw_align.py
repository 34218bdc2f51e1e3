"""The signal-to-span aligner on the GPU (`uncalled_b200 dtw`, unc_dtw_align_batch): the CLI on the example against the
golden taken from the reference's own code, a seeded batch of a few hundred reads against the C oracle (pinned to that
golden by tests/test_dtw_align.py), and the same batch with the sweep's workspace budget forced small."""
import json
import os
import subprocess
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

import dtwalignlib as D
import orclib

pytestmark = pytest.mark.gpu
ROOT = D.ROOT
FAST5 = os.path.join(ROOT, "tests", "golden", "fast5", "example_single.fast5")
READ_ID = "f41a60f7-de4a-4b17-9f54-387e52d60b65"


def test_cli_example_matches_golden(tmp_path):
    golden = json.load(open(D.GOLDEN))["example"]
    prefix = orclib.materialise_example_index(str(tmp_path))
    raw = np.load(os.path.join(ROOT, "tests", "golden", "example_read.npz"))["raw"]
    g = D.read_genome(prefix)
    contig, (_, clen) = next(iter(g[1].items()))
    for name, st, en, rs, re, fwd in D.example_queries(len(raw), clen):
        qf = tmp_path / (name + ".q")
        qf.write_text("%s %d %d %s %d %d %s\n" % (READ_ID, st, en, contig, rs, re, "+" if fwd else "-"))
        pp = str(tmp_path / (name + "_"))
        r = subprocess.run([sys.executable, "-m", "uncalled_b200", "dtw", prefix, FAST5, "--queries", str(qf), "--path-prefix", pp],
                           capture_output=True, text=True, cwd=ROOT, timeout=600)
        assert r.returncode == 0, r.stderr
        f = r.stdout.split("\n")[0].split("\t")
        assert f[:2] == [READ_ID, golden[name]["mean_score"]], name
        lines = open(pp + READ_ID + ".txt").read().split("\n")
        assert lines[-1] == ""
        cols = [l.split("\t") for l in lines[:-1]]
        assert all(len(c) == 6 and c[5] == "" for c in cols)
        path = np.array([[int(c[0]), int(c[1])] for c in cols], np.uint64)
        assert len(path) == golden[name]["path_len"]
        assert D.digest_path(path[::-1]) == golden[name]["path_sha"], name
        want = D.oracle_align(g, raw[st:(en or len(raw))], contig, rs, re, fwd)      # the golden's inputs
        assert D.public(want) == golden[name]
        km, mn = want["_kmers"][path[:, 1].astype(np.int64)], want["_means"][path[:, 0].astype(np.int64)]
        from uncalled_b200.dtw import r94d_cost
        cost = r94d_cost(km, mn)
        assert [c[2:5] for c in cols] == [["%d" % k, "%g" % float(m), "%g" % float(x)] for k, m, x in zip(km, mn, cost)]


def _oracle_job(args):
    prefix, sig, contig, rs, re, fwd = args
    return D.public(D.oracle_align(D.read_genome(prefix), sig, contig, rs, re, fwd))


@pytest.fixture(scope="module")
def batch(tmp_path_factory):
    """~200 seeded reads of 4 000 - 200 000 samples on both strands of the three contigs, and one of about 500 000
    samples (over the 50 000-means limit)"""
    d = str(tmp_path_factory.mktemp("batch"))
    prefix, codes = D.multi_contig_genome(d)
    rng = np.random.default_rng(2024)
    names = sorted(codes)
    cases = []
    for i in range(200):
        contig = names[i % 3]
        n_samp = int(np.exp(rng.uniform(np.log(4000), np.log(200000))))
        ln = min(n_samp // 8 + 10, len(codes[contig]) - 1)
        st = int(rng.integers(0, len(codes[contig]) - ln))
        fwd = bool(rng.integers(0, 2))
        flat = [(int(rng.integers(0, ln - 100)), 30)] if i % 5 == 0 else []
        sig = D.span_signal(codes[contig][st:st + ln], fwd, rng, flat)
        cases.append(("b%03d" % i, sig, contig, st, st + ln, fwd))
    big = D.span_signal(codes["chrB"][0:60000], True, rng)[:500000]
    cases.append(("big", big, "chrB", 0, 60000, True))
    assert len(big) > 450000
    with ProcessPoolExecutor(min(os.cpu_count() or 1, 16)) as ex:
        want = list(ex.map(_oracle_job, [(prefix,) + c[1:] for c in cases], chunksize=1))
    assert want[-1]["status"] == 1
    return prefix, cases, want


def _run(prefix, cases, budget=0):
    import uncalled_b200._native as N
    from uncalled_b200.dtw import DtwAligner
    N.check(N.lib().unc_init(0))
    A = DtwAligner(prefix, budget=budget)
    got, launches = [], 0
    for i in range(0, len(cases), 64):
        part = cases[i:i + 64]
        got += A.align([(c[0], c[1], None, 0, 0, c[2], c[3], c[4], c[5]) for c in part], paths=True)
        launches += A.last_times()[1]
    return got, launches


def _compare(got, want, cases):
    for g, w, c in zip(got, want, cases):
        assert g.read_id == c[0]
        assert (g.n_events, g.n_kept) == (w["n_events"], w["n_kept"]), c[0]
        if w["status"]:
            assert g.skip == {1: "too many means", 2: "no event left after the mask"}[w["status"]], c[0]
            continue
        assert g.skip is None, (c[0], g.skip)
        assert (D.f32_bits(g.score), D.f32_bits(g.mean_score), len(g.path)) == (w["score_bits"], w["mean_score_bits"], w["path_len"]), c[0]
        assert D.digest_path(g.path[::-1]) == w["path_sha"], c[0]


def test_batch_matches_oracle(batch):
    prefix, cases, want = batch
    got, launches = _run(prefix, cases)
    _compare(got, want, cases)
    assert got[-1].skip_message() == "Skipping big"


def test_forced_splits_give_identical_output(batch):
    prefix, cases, want = batch
    got_all, _ = _run(prefix, cases)
    budget = 160 << 20
    got, launches = _run(prefix, cases, budget=budget)
    assert launches >= 8
    too_large = [g for g in got if g.skip == "the DTW matrix exceeds the workspace budget"]
    assert too_large, "the batch holds reads whose matrix alone is over the budget"
    for g, a, w, c in zip(got, got_all, want, cases):
        if g.skip == "the DTW matrix exceeds the workspace budget":
            assert a.skip is None and w["status"] == 0
            assert g.skip_message() == "Skipping %s: the DTW matrix exceeds the workspace budget" % c[0]
            continue
        assert (g.skip, g.n_events, g.n_kept, g.score, g.mean_score) == (a.skip, a.n_events, a.n_kept, a.score, a.mean_score), c[0]
        if g.skip is None:
            assert np.array_equal(g.path, a.path) and np.array_equal(g.means, a.means) and np.array_equal(g.kmers, a.kmers)
