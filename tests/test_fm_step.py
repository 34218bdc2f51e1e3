"""CPU tier: the mapper's FM-index step (unc_occ2_neighbors of unc_k2v2.cuh, over the occ2 blocks k_occ2_build makes)
run by the emulator (emu_fm_step) against bwt_occ restated in numpy from the .bwt file and against the oracle's
get_neighbor, at every row of small indexes whose `$` row and last bwa block sit where the step's special cases are;
the k-mer ranges and the LF walk of bwt_sa against the oracle; mapping on a reference whose k-mer ranges are mostly
empty.  tests/test_z_gpu_fm_step.py runs the same checks through unc_fm_step on the GPU."""
import numpy as np
import pytest

import emulib
import fmsteplib as F
import orclib


@pytest.fixture(scope="module")
def fx_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("fm_step")


@pytest.fixture(scope="module")
def built(fx_dir):
    return {name: F.build(name, fx_dir) for name in F.FIXTURES}


def test_fixture_coverage(built):
    """the fixtures put seq_len mod 128, primary mod 64 and the `$` row where the step's edge cases are"""
    fms = {name: F.PlainFM(p) for name, p in built.items()}
    assert {fm.n % 128 for fm in fms.values()} >= set(F.SEQ_LEN_MOD_128)
    assert {0, 63} <= {fm.primary % 64 for fm in fms.values()}
    assert any(fm.primary // 64 == (fm.n - 1) // 64 for fm in fms.values())
    assert any(fm.primary == fm.n for fm in fms.values())
    assert min(fm.n for fm in fms.values()) == 2 and any(1 <= fm.n // 2 <= 40 for fm in fms.values())
    for name in ("multi_n", "poly", "palindrome"):
        assert name in fms


@pytest.mark.parametrize("name", sorted(F.FIXTURES))
def test_step_every_row_and_edges(built, name):
    fm = F.PlainFM(built[name])
    E = emulib.Emu(built[name])
    try:
        rng = np.random.default_rng(7)
        k0, l0 = F.check_every_row(E.fm_step, fm, rng)
        assert set(k0.tolist()) >= set(range(fm.n)) and set(l0.tolist()) >= set(range(1, fm.n + 1))
        F.check_edges(E.fm_step, fm, rng)
        # the 1.1 Gbp test's queries and per-row reference, at every row
        st, en = F.pairs_at_rows(np.arange(fm.n + 1), fm.n, rng)
        ns, ne = F._check(E.fm_step, fm, st, en, np.full(len(st), 15))
        ys, ye = F.step_at_rows(built[name], st, en)
        assert np.array_equal(ns.astype(np.int64), ys) and np.array_equal(ne.astype(np.int64), ye)
    finally:
        E.L.emu_index_free(E.idx)


@pytest.mark.parametrize("name", sorted(F.FIXTURES))
def test_plain_reference_is_the_oracles_get_neighbor(built, name):
    """the numpy restatement the step is held to agrees with the oracle (pinned to the reference) on every query"""
    fm = F.PlainFM(built[name])
    O = orclib.Oracle(built[name])
    rng = np.random.default_rng(8)
    st, en = F.every_row_queries(fm.n, rng)
    rows = F.edge_rows(fm)
    k0, l0 = np.meshgrid(rows, rows, indexing="ij")
    keep = k0 <= l0
    st, en = np.append(st, k0[keep] + 1), np.append(en, l0[keep])
    ns, ne = F.oracle_neighbors(O, st, en)
    xs, xe = fm.step(st, en)
    assert np.array_equal(ns, xs) and np.array_equal(ne, xe)
    # the per-row restatement the 1.1 Gbp test uses, at every row
    every = np.arange(fm.n + 1)
    assert np.array_equal(F.occ_at_rows(built[name], every), fm.occ[every + 1])


@pytest.mark.parametrize("name", sorted(F.FIXTURES))
def test_kmer_ranges_and_sa_walk(built, name):
    """all 1024 k-mer ranges (starts included) equal the oracle's, the index loads whatever the share of empty ranges,
    and the LF walk of bwt_sa gives the oracle's SA at every row"""
    fm = F.PlainFM(built[name])
    O = orclib.Oracle(built[name])
    E = emulib.Emu(built[name])
    try:
        st, en = E.kmer_ranges()
        ost, oen = O.kmer_ranges()
        assert np.array_equal(st, ost) and np.array_equal(en, oen)
        rows = np.arange(1, fm.n + 1)
        assert np.array_equal(E.sa(rows), F.oracle_sa(O, rows))
    finally:
        E.L.emu_index_free(E.idx)


def test_sa_walks_through_primary(built):
    """a few hundred rows whose walk passes the `$` row, where bwt_sa jumps to row 0"""
    hits = 0
    for name, p in built.items():
        fm = F.PlainFM(p)
        hits += int(fm.lf_walk_hits_primary(np.arange(1, fm.n + 1)).sum())
    assert hits >= 300, hits


def test_tiny_references_have_mostly_empty_kmer_ranges(built):
    O = orclib.Oracle(built["tiny40"])
    st, en = O.kmer_ranges()
    assert (st > en).sum() > 900


def test_plain_reference_on_the_example_index(example_prefix):
    """the numpy restatements against the oracle's get_neighbor on a sample of the example index's queries"""
    fm = F.PlainFM(example_prefix)
    O = orclib.Oracle(example_prefix)
    rng = np.random.default_rng(10)
    rows = rng.choice(np.arange(1, fm.n + 1), 1000, replace=False)
    st, en = F.every_row_queries(fm.n, rng, rows=rows)
    edges = F.edge_rows(fm)
    st, en = np.append(st, edges[:-1] + 1), np.append(en, np.full(len(edges) - 1, fm.n))
    ns, ne = F.oracle_neighbors(O, st, en)
    xs, xe = fm.step(st, en)
    assert np.array_equal(ns, xs) and np.array_equal(ne, xe)
    ys, ye = F.step_at_rows(example_prefix, st, en)
    assert np.array_equal(ys, xs) and np.array_equal(ye, xe)


def test_step_on_the_example_index(example_prefix):
    """1 % of the rows of the shipped example index (9.4 M rows), every width, and its edge rows"""
    fm = F.PlainFM(example_prefix)
    E = emulib.Emu(example_prefix)
    try:
        rng = np.random.default_rng(9)
        rows = np.sort(rng.choice(np.arange(1, fm.n + 1), fm.n // 100, replace=False))
        F.check_every_row(E.fm_step, fm, rng, rows=rows)
        F.check_edges(E.fm_step, fm, rng)
    finally:
        E.L.emu_index_free(E.idx)


def test_map_on_a_reference_with_empty_kmer_ranges(built):
    """seeded reads from a 639-base reference (1 278 FM rows, most 5-mers absent) map as the oracle maps them"""
    import synth
    prefix = built["mod126"]
    O = orclib.Oracle(prefix)
    st, en = O.kmer_ranges()
    assert (st > en).sum() > 100
    seq = open(prefix + ".fa", "rb").read().split(b"\n", 1)[1].replace(b"\n", b"")
    g = np.frombuffer(seq, np.uint8)
    g = np.searchsorted(np.frombuffer(b"ACGT", np.uint8), g).astype(np.uint8)
    sig, _ = synth.reads(g, 8, 1600, seed=3)
    E = emulib.Emu(prefix)
    try:
        recs, _, _, _ = E.map_batch([sig[i] for i in range(8)])
        for i in range(8):
            w = O.map_read(sig[i])
            assert orclib.paf_tuple(w) == emulib.paf_tuple(recs[i]), i
            assert (w.n_children, w.n_sources, w.n_seeds) == (recs[i].n_children, recs[i].n_sources, recs[i].n_seeds), i
    finally:
        E.L.emu_index_free(E.idx)
