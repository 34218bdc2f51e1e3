"""`events` on the GPU: the C-ABI against the C restatement, bit for bit, on thousands of seeded reads and on every golden
fast5 fixture; its means against unc_events_batch's; match_probs against unc_match_probs; the CLI's TSV."""
import ctypes as C
import glob
import io
import os

import numpy as np
import pytest

import eventslib as E

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAST5 = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "fast5", "*.fast5")))


@pytest.fixture(scope="module")
def proc():
    from uncalled_b200.signal import SignalProcessor
    p = SignalProcessor(device=0)
    yield p
    p.close()


def _check(res, pas, label):
    for i, pa in enumerate(pas):
        E.compare(res.reads[i], res.read(i), E.oracle_read(pa), (label, i))


def test_2000_synthetic_reads_equal_the_restatement(proc):
    sigs = E.synth_reads(1, 1200) + E.synth_reads(2, 800, n_samples=9000)
    res = proc.run(sigs)
    _check(res, sigs, "synth")
    assert len(res.events) > 500000


def test_edges_i16_and_a_long_read(proc):
    edges = list(E.edge_reads(13).values()) + [E.long_read()]
    res = proc.run(edges)
    _check(res, edges, "edges")
    assert int(res.reads["n_events"][-1]) > 50000
    sigs, cals = E.i16_reads(31, 200)
    res = proc.run(sigs, cals)
    _check(res, [E.calibrated(s, c) for s, c in zip(sigs, cals)], "i16")


def _fixture_reads():
    from uncalled_b200.fast5 import Fast5File
    out = []
    for path in FAST5:
        with Fast5File(path) as f:
            out += f.load(0)
    return out


def test_every_golden_fast5_fixture(proc):
    reads = _fixture_reads()
    assert len(reads) > 10
    res = proc.run([r.signal for r in reads], [r.calibration for r in reads])
    _check(res, [r.pa() for r in reads], "fast5")


def test_means_equal_the_mappers_events(proc, example_prefix):
    import uncalled_b200 as U
    sigs = E.synth_reads(4, 64)
    res = proc.run(sigs)
    idx = U.Index(example_prefix, device=0)
    bm = U.BatchMapper(idx, max_reads=64, max_samples=sum(len(s) for s in sigs))
    ev, nm, ne, mel = bm.events(np.concatenate(sigs), U.make_descs([len(s) for s in sigs]))
    for i in range(len(sigs)):
        got = res.read(i)
        assert int(ne[i]) == len(got)
        assert E.same_bits(got["mean"], ev[i, :ne[i]]) and E.same_bits(got["norm_mean"], nm[i, :ne[i]]), i
        assert E.same_bits([res.reads["mean_event_len"][i]], [mel[i]]), i
    rng = np.random.default_rng(3)
    pick = rng.choice(res.events["norm_mean"], 64, replace=False)
    pick = np.concatenate([pick, np.float32([0.0, -5.0, 300.0, 1e-30])])
    mp = proc.match_probs(pick)
    L, M = E.orc()
    for j, x in enumerate(pick):
        assert E.same_bits(mp[j], idx.match_probs(float(x))), j
    for j in range(0, len(pick), 9):
        want = np.array([L.orc_match_prob(C.byref(M), float(pick[j]), k) for k in range(1024)], np.float32)
        assert E.same_bits(mp[j], want), j
    bm.close()


def test_annotate_and_normalize_on_given_means(proc):
    rng = np.random.default_rng(8)
    lists = [rng.normal(90, 12, int(rng.integers(0, 600))).astype(np.float32) for _ in range(300)]
    lists[7][100:200] = np.float32(91.5)
    an = proc.annotate(lists)
    nz = proc.normalize(lists)
    L, M = E.orc()
    for i, m in enumerate(lists):
        n = len(m)
        wm, ws, mk = np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.uint8)
        L.orc_profile_events(m.ctypes.data, n, 5.0, wm.ctypes.data, ws.ctypes.data, mk.ctypes.data)
        assert E.same_bits(an[i]["win_mean"], wm[:n]) and E.same_bits(an[i]["win_stdv"], ws[:n]), i
        assert np.array_equal(an[i]["win_mask"], mk[:n] != 0), i
        if n:
            out, ss = np.zeros(n, np.float32), np.zeros(2, np.float32)
            L.orc_normalize_full(C.byref(M), m.ctypes.data, n, out.ctypes.data, ss.ctypes.data)
            assert E.same_bits(nz[i][2], out) and E.same_bits([nz[i][0], nz[i][1]], ss), i


def test_cli_tsv_equals_the_restatement():
    from uncalled_b200 import cli
    import argparse
    args = argparse.Namespace(fast5s=[os.path.join(ROOT, "tests", "golden", "fast5")], recursive=False, read_list=None,
                              max_reads=None, model=None, batch_reads=7, device=0)
    buf = io.StringIO()
    cli.events_cmd(args, out=buf)
    lines = buf.getvalue().split("\n")
    assert lines[0].split("\t") == list(cli.EVENTS_COLUMNS)
    rows = [l.split("\t") for l in lines[1:] if l]
    from uncalled_b200.fast5 import Fast5File
    want = []
    files = [f for f in cli.load_fast5s(args.fast5s, False) if f is not None]
    for path in files:
        with Fast5File(path) as f:
            for r in f.load(0):
                rd, ev = E.oracle_read(r.pa())
                for j in range(rd["n_events"]):
                    want.append((r.read_id, int(ev["start"][j]), np.float32(ev["length"][j]), ev["mean"][j], ev["stdv"][j],
                                 rd["norm_scale"], rd["norm_shift"], ev["norm_mean"][j], ev["win_mean"][j], ev["win_stdv"][j],
                                 int(ev["win_mask"][j])))
    assert len(rows) == len(want)
    for got, w in zip(rows, want):
        assert got[0] == w[0] and int(got[1]) == w[1] and int(got[10]) == w[10], (got, w)
        for k in range(2, 10):
            assert E.same_bits([np.float32(float(got[k]))], [w[k]]), (k, got, w)


def test_single_read_calls_chain(proc):
    """detect_events of one signal feeds annotate / normalize as one read, as the batched run computes it"""
    from uncalled_b200 import signal as S
    sig = E.synth_reads(12, 1)[0]
    ev = proc.detect_events(sig)
    batch = proc.run([sig]).read(0)
    assert len(ev) == len(batch) > 100
    an = proc.annotate(ev)
    assert len(an) == len(ev)
    assert E.same_values(an["win_mean"], batch["win_mean"]) and np.array_equal(an["win_mask"], batch["win_mask"] != 0)
    sc, sh, nm = proc.normalize(ev)
    assert E.same_bits(nm, batch["norm_mean"]) and np.isfinite(sc)
    assert len(S.annotate(ev)) == len(ev)


def test_pymodule_classes_equal_the_restatement():
    import sys
    import uncalled_b200._native as N
    N.build_pymodule()
    pkg = os.path.join(ROOT, "uncalled_b200")
    if pkg not in sys.path:
        sys.path.insert(0, pkg)
    import _uncalled as U
    L, M = E.orc()
    d = U.EventDetector()
    for sig in E.synth_reads(21, 5) + [E.edge_reads(3)["stall"]]:
        rd, want = E.oracle_read(sig)
        got = d.get_events(sig.tolist())
        assert len(got) == rd["n_events"]
        assert [e.start for e in got] == want["start"].tolist() and [e.length for e in got] == want["length"].astype(int).tolist()
        assert E.same_bits([e.mean for e in got], want["mean"]) and E.same_bits([e.stdv for e in got], want["stdv"])
        assert E.same_bits(d.get_means(sig.tolist()), want["mean"])
        assert E.same_values(d.mean_event_len(), rd["mean_event_len"])
        mask = U.EventProfiler().get_full_mask(got)
        assert mask == (want["win_mask"] != 0).tolist()
    Mt = type(M)()
    L.orc_model_init(C.byref(Mt), E.TAB.ctypes.data_as(C.POINTER(C.c_float)), 0)
    means = np.float32([70.5, 90.0, 101.25, 120.0])
    for model, om in ((U.pmodel_r94_complement, M), (U.pmodel_r94_template, Mt)):
        probs = model.match_prob(means)
        for j, x in enumerate(means):
            want = np.array([L.orc_match_prob(C.byref(om), float(x), k) for k in range(1024)], np.float32)
            assert E.same_bits(probs[j], want), j
            assert E.same_bits([model.match_prob(float(x), 37)], [want[37]])


def test_debug_held_returns(proc):
    import uncalled_b200._native as N
    from uncalled_b200.signal import SignalProcessor
    L = N.lib()
    d0, p0, h0 = C.c_uint64(), C.c_uint64(), C.c_uint32()
    N.check(L.unc_debug_held(C.byref(d0), C.byref(p0), C.byref(h0)))
    p = SignalProcessor(device=0)
    p.run(E.synth_reads(6, 10))
    p.match_probs(np.float32([80.0, 90.0]))
    p.close()
    d1, p1, h1 = C.c_uint64(), C.c_uint64(), C.c_uint32()
    N.check(L.unc_debug_held(C.byref(d1), C.byref(p1), C.byref(h1)))
    assert (d1.value, p1.value, h1.value) == (d0.value, p0.value, h0.value)
