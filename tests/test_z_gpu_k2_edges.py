"""GPU tier: the mapper kernels at the edges tests/test_k2_event_trace_emul.py traces event by event under the emulator.

There is no per-event view of the CUDA build, so these compare what a read ends with -- the PAF fields, n_children,
n_sources, n_seeds, n_clusters and status 0 -- against the oracle, on the same inputs: max_paths on both sides of 32 and
160 and at 32 767 (the largest value the library accepts) on the 200 kb and 4.7 Mb genomes, with the default and the
exact-ties kernels; the streaming mapper with 64 channels at 32 767; and the low-complexity genome.
"""
import numpy as np
import pytest

import orclib
import synth
import synthdata
import test_k2_event_trace_emul as T

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def U():
    import uncalled_b200
    uncalled_b200._native.lib()
    return uncalled_b200


def _counts(r):
    return (int(r.n_children), int(r.n_sources), int(r.n_seeds), int(r.n_clusters))


def _dev_counts(r):
    return (int(r["n_children"]), int(r["n_sources"]), int(r["n_seeds"]), int(r["n_clusters"]))


def _batch_vs_oracle(U, prefix, sigs, max_paths, exact):
    p = U.default_params()
    O = orclib.Oracle(prefix)
    p.max_paths = O.params.max_paths = max_paths
    idx = U.Index(prefix, device=0)
    bm = U.BatchMapper(idx, params=p, max_reads=len(sigs), max_samples=sum(len(s) for s in sigs))
    try:
        bm.set_tie_order(1 if exact else 0)
        out = bm.map(np.concatenate(sigs), U.make_descs([len(s) for s in sigs]))
    finally:
        bm.close()
        idx.close()
    O.lib.orc_set_child_sort(1 if exact else 0)
    try:
        want = [O.map_read(s) for s in sigs]
    finally:
        O.lib.orc_set_child_sort(0)
    for i in range(len(sigs)):
        assert (U.paf_key(out[i]), _dev_counts(out[i]), int(out[i]["status"])) == \
               (orclib.paf_tuple(want[i]), _counts(want[i]), 0), (max_paths, exact, i)
    return out, want


@pytest.mark.parametrize("exact", [0, 1])
@pytest.mark.parametrize("max_paths", [1, 32, 33, 160, 161, 32767])
@pytest.mark.parametrize("name", T.GENOMES)
def test_max_paths_edges(U, name, max_paths, exact):
    """Two reads that map early, two that never map (at 32 767 they sit at the cap for their whole length)."""
    prefix, sigs = T._reads(name, T.MAPS + T.NEVER)
    out, want = _batch_vs_oracle(U, prefix, sigs, max_paths, exact)
    if name == "g4m7" or max_paths <= 161:           # the 200 kb genome holds about 2 300 paths at most
        assert max(w.max_paths_seen for w in want) == max_paths


def test_stream_mapper_64_channels_at_max_paths_32767(U):
    """64 channel slots of the largest buffer; two reads per channel, so that the second continues the channel's state."""
    prefix, g = synthdata.get_index("g4m7")
    sig, truth = synth.reads(g, 128, 2000, seed=17, frac_random=0.15)
    sigs = [np.ascontiguousarray(s, np.float32) for s in sig]
    p = U.default_params()
    O = orclib.Oracle(prefix)
    p.max_paths = O.params.max_paths = 32767
    idx = U.Index(prefix, device=0)
    sm = U.StreamMapper(idx, 64, 450, params=p)
    try:
        res = sm.map_reads(sigs)
    finally:
        sm.close()
        idx.close()
    n_cap = 0
    for c in range(64):
        ids = list(range(c, len(sigs), 64))
        for i, (rec, nu, en) in zip(ids, O.stream_channel([sigs[i] for i in ids], 450)):
            r = res[i]
            assert r is not None and (U.paf_key(r[3]), r[2], r[1]) == (orclib.paf_tuple(rec), nu, en), i
            assert (r[3].n_children, r[3].n_sources, r[3].n_seeds) == (rec.n_children, rec.n_sources, rec.n_seeds), i
            assert r[3].status == 0, i
            n_cap += rec.max_paths_seen == 32767
    assert n_cap > 0 and any(r[3].mapped for r in res)


@pytest.mark.parametrize("exact", [0, 1])
@pytest.mark.parametrize("max_paths", [300, 10000])
def test_low_complexity_genome(U, max_paths, exact):
    prefix, sigs = T._low_complexity_reads()
    _batch_vs_oracle(U, prefix, sigs, max_paths, exact)
