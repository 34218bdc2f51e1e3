"""`events` without a GPU: the C restatement against the reference's own classes and the golden file, the device
routines (unc_events.cuh) under the emulator against the restatement, the compiler's numbers of the kernels `map`
launches, the CLI's argument errors and the C-ABI's answer on a machine without a device."""
import ctypes as C
import json
import os
import shutil
import sys

import numpy as np
import pytest

import eventslib as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import make_events_golden as MG  # noqa: E402

need_ref = pytest.mark.skipif(not E.ref_available(), reason="oracle/_ref/libref_events.so not built")


def _split(reads, events):
    off = [0] + [int(x) for x in np.cumsum(reads["n_events"])]
    return [(reads[i], events[off[i]:off[i + 1]]) for i in range(len(reads))]


def _check_batch(sigs, pas=None, calibration=None, label=""):
    reads, events = E.emulated(sigs, calibration)
    for i, (rd, ev) in enumerate(_split(reads, events)):
        E.compare(rd, ev, E.oracle_read(sigs[i] if pas is None else pas[i]), (label, i))
    return reads, events


# ---------------------------------------------------------------- the restatement
@need_ref
def test_restatement_equals_reference_bitwise():
    sigs = list(MG.golden_reads().values()) + E.synth_reads(7, 30) + list(E.edge_reads(3).values())
    for i, s in enumerate(sigs):
        want, got = E.ref_read(s), E.oracle_read(s)
        for k in ("n_events", "mean_event_len"):
            assert E.same_bits([want[0][k]], [got[0][k]]), (i, k)
        for k in E.FIELDS:
            assert E.same_bits(want[1][k], got[1][k]), (i, k)


def test_restatement_equals_golden():
    gold = json.load(open(E.GOLDEN))["reads"]
    reads = MG.golden_reads()
    assert set(gold) == set(reads)
    for name, sig in reads.items():
        assert MG.summarise(E.oracle_read(sig)) == gold[name], name


def test_golden_covers_masked_and_tail_events():
    gold = json.load(open(E.GOLDEN))["reads"]
    assert gold["example_read"]["n_events"] > 5000
    assert gold["edge_empty"]["n_events"] == 0
    stall = E.oracle_read(MG.golden_reads()["edge_stall"])[1]
    assert (stall["win_mask"] == 0).sum() >= 24 and np.isnan(stall["win_mean"][-24:]).all()


# ---------------------------------------------------------------- the device routines under the emulator
def test_emulated_synthetic_reads():
    _check_batch(E.synth_reads(17, 60), label="synth")


def test_emulated_edge_reads():
    edges = E.edge_reads(41)
    reads, events = _check_batch(list(edges.values()), label="edges")
    by = dict(zip(edges, _split(reads, events)))
    assert int(by["empty"][0]["n_events"]) == 0 and np.isnan(by["empty"][0]["mean_event_len"])
    assert by["empty"][0]["norm_scale"] == 0 and by["empty"][0]["norm_shift"] == 0
    assert int(by["short_5"][0]["n_events"]) == 0
    stall = by["stall"][1]
    assert (stall["win_mask"] == 0).any()                     # the constant stretch is masked
    few = by["few_events"][1]
    assert 0 < len(few) and np.isnan(few["win_mean"][-min(len(few), 24):]).all()


def test_emulated_filters_out_of_range_means():
    sig = E.edge_reads(5)["out_of_range"]
    _, ev = _check_batch([sig], label="range")
    full = E.oracle_read(sig, params=None)[0]["n_events"]
    narrow = E.EventParams(3, 6, 1.4, 9.0, 0.2, 60.0, 120.0, 25, 5.0)
    reads, events = E.emulated([sig], params=narrow)
    assert 0 < int(reads["n_events"][0]) < full
    assert (events["mean"] >= 60).all() and (events["mean"] <= 120).all()
    import orclib
    P = orclib.OrcParams()
    E.orc()[0].orc_params_default(C.byref(P))
    P.min_mean, P.max_mean = 60.0, 120.0
    E.compare(reads[0], events, E.oracle_read(sig, params=P), "narrow")


def test_emulated_i16_with_calibration():
    sigs, cals = E.i16_reads(23, 12)
    pas = [E.calibrated(s, c) for s, c in zip(sigs, cals)]
    _check_batch(sigs, pas=pas, calibration=cals, label="i16")


def test_emulated_read_over_50000_events():
    sig = E.long_read()
    reads, _ = _check_batch([sig], label="long")
    assert int(reads["n_events"][0]) > 50000


def test_warp_routine_equals_the_serial_one():
    """K1's warp routine in its FULL variant and the serial routine give the same records, at several CTA sizes"""
    sigs = E.synth_reads(19, 40, n_samples=6000) + list(E.edge_reads(7).values())
    want = E.emulated(sigs, serial=True)
    for w in (1, 3):
        red = []
        got = E.emulated(sigs, n_warps=w, redone=red)
        assert red == [0]
        assert np.array_equal(got[0]["n_events"], want[0]["n_events"])
        for k in E.FIELDS:
            assert E.same_values(got[1][k], want[1][k]) if k not in ("start", "win_mask") else \
                np.array_equal(got[1][k], want[1][k]), (w, k)


def test_inexact_sums_are_redone_serially():
    """reads whose prefix sums (or sums of squares) round fail K1's exactness check and go to the serial routine"""
    base = E.synth_reads(2, 3, n_samples=5000, ragged=False)
    s = base[0].copy(); s[1000] = 1e-20; s[2000] = 3e7
    t = base[1].copy(); t[10] = np.float32(1e-41)
    red = []
    reads, events = E.emulated([s, t, base[2]], redone=red)
    assert red == [2]
    for i, (rd, ev) in enumerate(_split(reads, events)):
        E.compare(rd, ev, E.oracle_read([s, t, base[2]][i]), ("redo", i))


def test_one_events_array_is_one_read():
    from uncalled_b200.signal import EVENT_DTYPE, _as_list, _means
    ev = np.zeros(5, EVENT_DTYPE)
    ev["mean"] = np.arange(5, dtype=np.float32) + 80
    lst, one = _as_list(ev)
    assert one and len(lst) == 1 and np.array_equal(_means(lst[0]), ev["mean"])
    lst, one = _as_list([ev, ev[:2]])
    assert not one and [len(_means(m)) for m in lst] == [5, 2]


def test_pymodule_window_lengths_are_fixed():
    import uncalled_b200._native as N
    N.build_pymodule()
    pkg = os.path.join(ROOT, "uncalled_b200")
    if pkg not in sys.path:
        sys.path.insert(0, pkg)
    import _uncalled as U
    p = U.EventDetector.Params()
    assert (p.window_length1, p.window_length2) == (3, 6) and np.float32(p.threshold1) == np.float32(1.4)
    for name, v in (("window_length1", 4), ("window_length2", 5)):
        with pytest.raises(ValueError):
            setattr(p, name, v)
    p.window_length1, p.threshold2 = 3, 8.5
    assert p.threshold2 == 8.5
    e = U.Event()
    e.mean, e.length = 91.5, 7
    assert (e.mean, e.length) == (91.5, 7)


def test_emulated_annotate_on_given_means():
    rng = np.random.default_rng(9)
    lists = [rng.normal(90, 12, int(rng.integers(0, 400))).astype(np.float32) for _ in range(20)]
    lists[3][50:120] = np.float32(88.0)                        # a stall
    lists.append(np.zeros(0, np.float32))
    off, nm, wm, ws, mk, sc, sh = E.emulated_annotate(lists)
    L, M = E.orc()
    for i, m in enumerate(lists):
        a, b = int(off[i]), int(off[i + 1])
        n = len(m)
        wwm, wws, wmk = np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.uint8)
        L.orc_profile_events(m.ctypes.data, n, 5.0, wwm.ctypes.data, wws.ctypes.data, wmk.ctypes.data)
        assert E.same_bits(wm[a:b], wwm[:n]) and E.same_bits(ws[a:b], wws[:n]) and E.same_bits(mk[a:b], wmk[:n]), i
        if n:
            out, ss = np.zeros(n, np.float32), np.zeros(2, np.float32)
            L.orc_normalize_full(C.byref(M), m.ctypes.data, n, out.ctypes.data, ss.ctypes.data)
            assert E.same_bits(nm[a:b], out) and E.same_bits([sc[i], sh[i]], ss), i
        else:
            assert sc[i] == 0 and sh[i] == 0


# ---------------------------------------------------------------- the kernels `map` launches are untouched
# ptxas -v for sm_90a (CUDA 12.9) of the parent build (DESIGN.md section 4 lists the mapper kernels' numbers)
MAP_KERNELS = {"k1_events": (128, 0), "k1_fallback": (52, 0), "k2_map": (72, 220), "k2_map_ord": (72, 236),
               "k2_map_stream": (72, 264), "k2_map_exact": (72, 256), "k2_map_stream_exact": (72, 284)}


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_map_kernels_compile_as_before(tmp_path):
    import spill_report
    _, text = spill_report.compile_cubin(str(tmp_path))
    st = spill_report.ptxas_stats(text)
    for k, (regs, spill) in MAP_KERNELS.items():
        assert (st[k]["regs"], st[k]["spill_st"]) == (regs, spill), (k, st[k])
    for k in ("k_events_warp", "k_events_detect", "k_events_annotate", "k_events_gather", "k_match_probs_batch"):
        assert st[k]["spill_st"] == 0 and st[k]["spill_ld"] == 0, (k, st[k])


# ---------------------------------------------------------------- host side
def _run_cli(argv):
    from uncalled_b200 import cli
    with pytest.raises(SystemExit) as e:
        cli.main(argv)
    return e.value.code


def test_cli_argument_errors(tmp_path, capsys):
    fx = os.path.join(ROOT, "tests", "golden", "fast5")
    assert _run_cli(["events", str(tmp_path / "missing")]) == 1
    assert _run_cli(["events", fx, "-n", "-1"]) == 1
    assert _run_cli(["events", fx, "--batch-reads", "0"]) == 1
    assert _run_cli(["events", fx, "-l", str(tmp_path / "no_list.txt")]) == 1
    assert _run_cli(["events", fx, "--model", str(tmp_path / "no_model.f32")]) == 1
    bad = tmp_path / "short_model.f32"
    bad.write_bytes(b"\0" * 100)
    assert _run_cli(["events", fx, "--model", str(bad)]) == 1
    assert _run_cli(["events", fx, "--device", "-2"]) == 1
    err = capsys.readouterr().err
    assert "does not exist" in err and "pore model table" in err


def test_stage_rejects_mixed_and_uncalibrated_batches():
    from uncalled_b200.signal import SignalProcessor
    with pytest.raises(ValueError):
        SignalProcessor.stage([np.zeros(10, np.float32), np.zeros(10, np.int16)])
    with pytest.raises(ValueError):
        SignalProcessor.stage([np.zeros(10, np.int16)])
    flat, d = SignalProcessor.stage([np.arange(5, dtype=np.float32), np.zeros(0, np.float32), np.ones(3, np.float32)])
    assert list(d["offset"]) == [0, 5, 5] and list(d["n_samples"]) == [5, 0, 3] and len(flat) == 8


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs the native library")
def test_no_device_status():
    import uncalled_b200._native as N
    L = N.lib()
    if L.unc_device_count() > 0:
        pytest.skip("a CUDA device is present")
    p = N.EventParams()
    assert L.unc_event_params_default(C.byref(p)) == 0
    assert (p.window_length1, p.window_length2, p.win_len) == (3, 6, 25)
    assert np.float32(p.threshold1) == np.float32(1.4) and p.win_stdv_min == 5.0
    h = C.c_void_p()
    assert L.unc_events_create(N.MODEL_TABLE.encode(), C.byref(p), C.byref(h)) == -4     # UNC_E_NO_DEVICE
    p.window_length2 = 7
    assert L.unc_events_create(N.MODEL_TABLE.encode(), C.byref(p), C.byref(h)) == -1     # UNC_E_ARG comes first
