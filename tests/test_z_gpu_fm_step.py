"""GPU tier: the mapper's FM-index step through unc_fm_step (UNC_OCC2_STEP, the body the worker warps expand), over the
occ2 blocks k_occ2_build makes on the device, against bwt_occ restated in numpy: every row of the small fixtures of
tests/fmsteplib.py and of the shipped example index.  The k-mer ranges against the oracle; unc_fm_sa with the expanded
suffix array and with the LF walk (UNC_NO_SA_EXPAND=1) against the oracle; and the existing mapping parity sets rerun
on the walk, which is the path an index takes when device memory is short."""
import contextlib
import os

import numpy as np
import pytest

import emulib
import fmsteplib as F
import orclib
import synth
import synthdata
import test_gpu_parity as P
import test_k2_event_trace_emul as T
import test_z_gpu_k2_edges as K

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def U():
    import uncalled_b200
    uncalled_b200._native.lib()
    return uncalled_b200


@contextlib.contextmanager
def sa_walk():
    """index loads inside build no expanded suffix array, so the mapper and unc_fm_sa walk LF"""
    old = os.environ.get("UNC_NO_SA_EXPAND")
    os.environ["UNC_NO_SA_EXPAND"] = "1"
    try:
        yield
    finally:
        if old is None:
            del os.environ["UNC_NO_SA_EXPAND"]
        else:
            os.environ["UNC_NO_SA_EXPAND"] = old


def load_both(U, prefix):
    """(index with the expanded suffix array, index that walks); which path each took, from its device bytes"""
    a = U.Index(prefix, device=0)
    with sa_walk():
        b = U.Index(prefix, device=0)
    assert a.device_bytes - b.device_bytes == 4 * (a.n_rows + 1), (a.device_bytes, b.device_bytes, a.n_rows)
    print("%s: first load expanded the suffix array (%d bytes more), the UNC_NO_SA_EXPAND load walks" %
          (os.path.basename(prefix), 4 * (a.n_rows + 1)))
    return a, b


@pytest.fixture(scope="module")
def built(tmp_path_factory):
    d = tmp_path_factory.mktemp("fm_step_gpu")
    return {name: F.build(name, d) for name in F.FIXTURES}


@pytest.mark.parametrize("name", sorted(F.FIXTURES))
def test_step_kmer_ranges_and_sa_on_small_indexes(U, built, name):
    fm = F.PlainFM(built[name])
    O = orclib.Oracle(built[name])
    a, b = load_both(U, built[name])
    try:
        rng = np.random.default_rng(7)
        k0, l0 = F.check_every_row(a.fm_step, fm, rng)
        assert set(k0.tolist()) >= set(range(fm.n)) and set(l0.tolist()) >= set(range(1, fm.n + 1))
        F.check_edges(a.fm_step, fm, rng)
        st, en = a.kmer_ranges()
        ost, oen = O.kmer_ranges()
        assert np.array_equal(st, ost) and np.array_equal(en, oen)
        rows = np.arange(1, fm.n + 1, dtype=np.uint64)
        want = F.oracle_sa(O, rows)
        assert np.array_equal(a.sa(rows), want)
        assert np.array_equal(b.sa(rows), want)
    finally:
        a.close()
        b.close()


def test_sa_walk_through_primary_on_the_gpu(U, built):
    """the walk's jump at the `$` row, on the rows whose walk passes it"""
    hits = 0
    for name, prefix in built.items():
        fm = F.PlainFM(prefix)
        rows = np.arange(1, fm.n + 1)[fm.lf_walk_hits_primary(np.arange(1, fm.n + 1))]
        if not len(rows):
            continue
        hits += len(rows)
        a, b = load_both(U, prefix)
        try:
            assert np.array_equal(b.sa(rows), F.oracle_sa(orclib.Oracle(prefix), rows)), name
        finally:
            a.close()
            b.close()
    assert hits >= 300


def test_step_on_every_row_of_the_example_index(U, example_prefix):
    """9.4 M rows: widths 0 and one random width at every row, all widths on 1 % of them, the edge rows; the
    neighbour probe against the oracle on a sample; both SA paths against the oracle on a sample"""
    fm = F.PlainFM(example_prefix)
    a, b = load_both(U, example_prefix)
    try:
        rng = np.random.default_rng(9)
        k0, l0 = F.check_every_row(a.fm_step, fm, rng, widths=(0,))
        assert len(np.unique(k0)) == fm.n + 1 and len(np.unique(l0)) == fm.n
        rows = np.sort(rng.choice(np.arange(1, fm.n + 1), fm.n // 100, replace=False))
        F.check_every_row(a.fm_step, fm, rng, rows=rows)
        F.check_edges(a.fm_step, fm, rng)
        O = orclib.Oracle(example_prefix)
        st = rng.integers(1, fm.n + 1, 3000)
        en = np.minimum(st + rng.integers(0, 300, 3000), fm.n)
        base = rng.integers(0, 4, 3000).astype(np.uint8)
        ons, one = F.oracle_neighbors(O, st, en)
        gs, ge = a.neighbors(st, en, base)
        assert np.array_equal(gs.astype(np.int64), ons[np.arange(3000), base])
        assert np.array_equal(ge.astype(np.int64), one[np.arange(3000), base])
        rows = np.concatenate([rng.integers(1, fm.n + 1, 20000), np.arange(fm.primary - 40, fm.primary + 40),
                               np.arange(fm.n - 40, fm.n + 1)]).astype(np.uint64)
        want = F.oracle_sa(O, rows)
        assert np.array_equal(a.sa(rows), want) and np.array_equal(b.sa(rows), want)
    finally:
        a.close()
        b.close()


def _records(out):
    keys = [k for k in out.dtype.names if k not in ("n_sa_steps", "n_occ_blocks")]
    return [tuple(int(r[k]) for k in keys) for r in out]


def test_map_example_read_with_the_sa_walk(U, example_prefix, golden_read):
    a, idx = load_both(U, example_prefix)
    a.close()
    bm = U.BatchMapper(idx, max_reads=64, max_samples=64 * 32000)
    try:
        P.test_map_example_read_matches_reference_paf(U, (idx, bm), golden_read)
        out = bm.map(golden_read["raw"], U.make_descs([len(golden_read["raw"])]))
        assert out[0]["mapped"] and out[0]["n_sa_steps"] > 0
    finally:
        bm.close()
        idx.close()


@pytest.mark.parametrize("name,n_reads,n_samples,seed,max_paths", [("g200k", 256, 4000, 7, None),
                                                                    ("g4m7", 48, 4000, 21, None),
                                                                    ("g200k", 64, 3000, 13, 300)])
def test_map_with_the_sa_walk_matches_oracle_and_expanded_run(U, name, n_reads, n_samples, seed, max_paths):
    """records equal the expanded run's but for n_sa_steps and n_occ_blocks, which count the walk's steps and the Occ
    blocks they read as the emulator (which walks too) counts them"""
    mod = None
    if max_paths:
        def mod(p):
            p.max_paths = max_paths
    expanded, _ = P._compare_with_oracle(U, name, n_reads, n_samples, seed, params_mod=mod)
    with sa_walk():
        walked, _ = P._compare_with_oracle(U, name, n_reads, n_samples, seed, params_mod=mod)
    assert _records(walked) == _records(expanded)
    assert (expanded["n_sa_steps"] == 0).all()
    mapped = walked["mapped"] != 0
    assert mapped.any() and (walked["n_sa_steps"][mapped] > 0).all()
    assert (walked["n_occ_blocks"] >= expanded["n_occ_blocks"]).all()
    prefix, g = synthdata.get_index(name)
    sig, _ = synth.reads(g, n_reads, n_samples, seed=seed)
    E = emulib.Emu(prefix)
    try:
        if mod:
            mod(E.params)
        k = 24
        recs, _, _, _ = E.map_batch([sig[i] for i in range(k)], n_warps=14)
        assert [(int(r.n_sa_steps), int(r.n_occ_blocks)) for r in recs] == \
               [(int(x), int(y)) for x, y in zip(walked["n_sa_steps"][:k], walked["n_occ_blocks"][:k])]
    finally:
        E.L.emu_index_free(E.idx)


@pytest.mark.parametrize("exact", [0, 1])
def test_map_exact_ties_and_max_paths_edges_with_the_sa_walk(U, exact):
    prefix, sigs = T._reads("g4m7", T.MAPS + T.NEVER)
    with sa_walk():
        K._batch_vs_oracle(U, prefix, sigs, 161, exact)


def test_stream_with_the_sa_walk(U):
    prefix, g = synthdata.get_index("g200k")
    sig, _ = synth.reads(g, 24, 8000, seed=15, frac_random=0.3)
    sigs = [sig[i][:8000 - 53 * i] for i in range(24)] + [sig[0][:200]]
    with sa_walk():
        st = P._stream_vs_oracle(U, prefix, sigs, 8, 450)
    assert (2, 0) in st and (3, 1) in st


def test_map_on_a_reference_with_empty_kmer_ranges(U, built):
    """seeded reads from a 639-base reference whose k-mer ranges are mostly empty, expanded and walked, as the oracle"""
    prefix = built["mod126"]
    seq = open(prefix + ".fa", "rb").read().split(b"\n", 1)[1].replace(b"\n", b"")
    g = np.searchsorted(np.frombuffer(b"ACGT", np.uint8), np.frombuffer(seq, np.uint8)).astype(np.uint8)
    sig, _ = synth.reads(g, 8, 1600, seed=3)
    O = orclib.Oracle(prefix)
    for walk in (False, True):
        with (sa_walk() if walk else contextlib.nullcontext()):
            idx = U.Index(prefix, device=0)
        bm = U.BatchMapper(idx, max_reads=8, max_samples=8 * 1600)
        out = bm.map(sig.ravel(), U.make_descs([1600] * 8))
        for i in range(8):
            w = O.map_read(sig[i])
            assert orclib.paf_tuple(w) == U.paf_key(out[i]) and out[i]["status"] == 0, (walk, i)
            assert (w.n_children, w.n_sources, w.n_seeds) == \
                   (int(out[i]["n_children"]), int(out[i]["n_sources"]), int(out[i]["n_seeds"])), (walk, i)
        bm.close()
        idx.close()
