"""Checkers of `events` (uncalled_b200/csrc/unc_events.cuh): the C restatement (oracle/unc_oracle_events.c), the
reference's own classes (oracle/_ref/libref_events.so), the device routines under the emulator
(tests/emul/emul_events.cpp), and seeded reads that reach the edge cases."""
import ctypes as C
import os
import subprocess

import numpy as np

import orclib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
CSRC = os.path.join(ROOT, "uncalled_b200", "csrc")
GOLDEN = os.path.join(ROOT, "tests", "golden", "events_golden.json")
TAB = np.fromfile(orclib.MODEL_TABLE, dtype=np.float32)
FIELDS = ("start", "length", "mean", "stdv", "norm_mean", "win_mean", "win_stdv", "win_mask")
vp = C.c_void_p


class EventParams(C.Structure):      # unc_event_params
    _fields_ = [("window_length1", C.c_uint32), ("window_length2", C.c_uint32), ("threshold1", C.c_float),
                ("threshold2", C.c_float), ("peak_height", C.c_float), ("min_mean", C.c_float), ("max_mean", C.c_float),
                ("win_len", C.c_uint32), ("win_stdv_min", C.c_float)]


def default_event_params():
    return EventParams(3, 6, 1.4, 9.0, 0.2, 0.0, 400.0, 25, 5.0)


_orc = _model = _ref = _emu = None


def orc():
    """libunc_oracle_events.so and the mapper's model (complement order) as an OrcModel"""
    global _orc, _model
    if _orc is None:
        path = os.path.join(ORACLE_DIR, "libunc_oracle_events.so")
        subprocess.run(["make", "-C", ORACLE_DIR, "-f", "events.mk", "libunc_oracle_events.so"], check=True, capture_output=True)
        L = C.CDLL(path)
        L.orc_params_default.argtypes = [C.POINTER(orclib.OrcParams)]
        L.orc_model_init.argtypes = [C.POINTER(orclib.OrcModel), orclib.f32p, C.c_int]
        L.orc_match_prob.argtypes = [C.POINTER(orclib.OrcModel), C.c_float, C.c_uint16]
        L.orc_match_prob.restype = C.c_float
        L.orc_detect_events_full.argtypes = [C.POINTER(orclib.OrcParams), vp, C.c_uint32, vp, vp, vp, vp, vp]
        L.orc_detect_events_full.restype = C.c_uint32
        L.orc_profile_events.argtypes = [vp, C.c_uint32, C.c_float, vp, vp, vp]
        L.orc_profile_events.restype = None
        L.orc_normalize_full.argtypes = [C.POINTER(orclib.OrcModel), vp, C.c_uint32, vp, vp]
        L.orc_normalize_full.restype = None
        M = orclib.OrcModel()
        L.orc_model_init(C.byref(M), TAB.ctypes.data_as(orclib.f32p), 1)
        _orc, _model = L, M
    return _orc, _model


def ref_available():
    return os.path.exists(os.path.join(ORACLE_DIR, "_ref", "libref_events.so"))


def ref():
    global _ref
    if _ref is None:
        L = C.CDLL(os.path.join(ORACLE_DIR, "_ref", "libref_events.so"))
        L.ref_get_events_full.argtypes = [vp, C.c_uint32, vp, vp, vp, vp, vp]
        L.ref_get_events_full.restype = C.c_uint32
        L.ref_profile_events.argtypes = [vp, C.c_uint32, vp, vp, vp]
        L.ref_profile_events.restype = None
        L.ref_normalize_full.argtypes = [vp, C.c_uint32, vp]
        L.ref_normalize_full.restype = None
        L.ref_match_prob_c.argtypes = [C.c_float, C.c_uint16]
        L.ref_match_prob_c.restype = C.c_float
        _ref = L
    return _ref


def _table(n):
    return {"start": np.zeros(n, np.uint32), "length": np.zeros(n, np.float32), "mean": np.zeros(n, np.float32),
            "stdv": np.zeros(n, np.float32), "norm_mean": np.zeros(n, np.float32), "win_mean": np.zeros(n, np.float32),
            "win_stdv": np.zeros(n, np.float32), "win_mask": np.zeros(n, np.uint8)}


def _one(pa, detect, profile, normalize):
    """(per-read dict, per-event dict) from one pA signal through the three stages"""
    pa = np.ascontiguousarray(pa, np.float32)
    n = len(pa)
    t = _table(max(n, 1))
    lens = np.zeros(max(n, 1), np.uint32)
    mel = C.c_float()
    ne = detect(pa, n, t, lens, mel)
    t = {k: v[:ne].copy() for k, v in t.items()}
    t["length"] = lens[:ne].astype(np.float32)
    ss = np.zeros(2, np.float32)
    if ne:
        normalize(t["mean"], ne, t["norm_mean"], ss)
    profile(t["mean"], ne, t["win_mean"], t["win_stdv"], t["win_mask"])
    return {"n_events": ne, "mean_event_len": np.float32(mel.value), "norm_scale": ss[0], "norm_shift": ss[1]}, t


def oracle_read(pa, win_stdv_min=5.0, params=None):
    L, M = orc()
    P = params or orclib.OrcParams()
    if params is None:
        L.orc_params_default(C.byref(P))
    d = lambda pa, n, t, lens, mel: L.orc_detect_events_full(  # noqa: E731
        C.byref(P), pa.ctypes.data, n, t["mean"].ctypes.data, t["stdv"].ctypes.data, t["start"].ctypes.data,
        lens.ctypes.data, C.byref(mel))
    nz = lambda m, n, out, ss: L.orc_normalize_full(C.byref(M), m.ctypes.data, n, out.ctypes.data, ss.ctypes.data)  # noqa: E731
    pr = lambda m, n, wm, ws, mk: L.orc_profile_events(m.ctypes.data, n, win_stdv_min, wm.ctypes.data, ws.ctypes.data,  # noqa: E731
                                                       mk.ctypes.data)
    return _one(pa, d, pr, nz)


def ref_read(pa):
    """the reference's own classes, default parameters (norm_scale / norm_shift are NaN: the reference keeps them inside
    Normalizer::at; its normalised means are compared instead)"""
    L = ref()
    d = lambda pa, n, t, lens, mel: L.ref_get_events_full(  # noqa: E731
        pa.ctypes.data, n, t["mean"].ctypes.data, t["stdv"].ctypes.data, t["start"].ctypes.data, lens.ctypes.data,
        C.byref(mel))
    def nz(m, n, out, ss):               # the reference's scale / shift are private to its Normalizer: NaN here
        L.ref_normalize_full(m.ctypes.data, n, out.ctypes.data)
        ss[:] = np.nan
    pr = lambda m, n, wm, ws, mk: L.ref_profile_events(m.ctypes.data, n, wm.ctypes.data, ws.ctypes.data, mk.ctypes.data)  # noqa: E731
    return _one(pa, d, pr, nz)


def emu():
    global _emu
    if _emu is None:
        src = os.path.join(EMUL_DIR, "emul_events.cpp")
        out = os.path.join(EMUL_DIR, "libunc_emul_events.so")
        deps = [src, os.path.join(EMUL_DIR, "warp_emul.hpp")] + [os.path.join(CSRC, f) for f in (
            "unc_device.cuh", "unc_events.cuh", "unc_k1.cuh", "unc_stream.cuh", "unc_warp.cuh", "unc_host_index.hpp", "unc_host_params.hpp")]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(x) for x in deps):
            subprocess.run(["g++", "-O2", "-g", "-std=c++17", "-ffp-contract=off", "-DUNC_EMUL", "-DK2_MAXSEG=16u", "-fPIC",
                            "-shared", "-I" + EMUL_DIR, "-I" + CSRC, "-o", out, src], check=True, capture_output=True)
        L = C.CDLL(out)
        L.emu_events_run.argtypes = [C.c_char_p, C.POINTER(EventParams), vp, C.c_uint32, vp, vp, vp, C.c_int, C.c_int,
                                     C.POINTER(C.c_uint32)]
        L.emu_events_annotate.argtypes = [C.c_char_p, C.POINTER(EventParams), C.c_uint32, vp, vp, vp, vp, vp, vp, vp, vp]
        _emu = L
    return _emu


def emulated(signals, calibration=None, params=None, n_warps=2, serial=False, redone=None):
    """the device routines over a batch: (reads READ_DTYPE, events FULL_DTYPE) as unc_events_run + fetch return them.
    serial: every read through the serial routine instead of K1's warp routine; redone (a list): receives the number of
    reads the warp routine handed to the serial one"""
    from uncalled_b200.signal import FULL_DTYPE, READ_DTYPE, SignalProcessor
    flat, descs = SignalProcessor.stage(signals, calibration)
    n = len(descs)
    reads = np.zeros(n, READ_DTYPE)
    events = np.zeros(max(int(descs["n_samples"].sum()), 1), FULL_DTYPE)
    P = params or default_event_params()
    nr = C.c_uint32()
    rc = emu().emu_events_run(orclib.MODEL_TABLE.encode(), C.byref(P), descs.ctypes.data, n, flat.ctypes.data,
                              reads.ctypes.data, events.ctypes.data, n_warps, 1 if serial else 0, C.byref(nr))
    assert rc == 0
    if redone is not None:
        redone.append(nr.value)
    return reads, events[:int(reads["n_events"].sum())]


def emulated_annotate(means_list, params=None):
    off = np.zeros(len(means_list) + 1, np.uint64)
    off[1:] = np.cumsum([len(m) for m in means_list])
    flat = np.ascontiguousarray(np.concatenate([np.asarray(m, np.float32) for m in means_list] + [np.zeros(1, np.float32)]))
    t = int(off[-1]) + 1
    nm, wm, ws = (np.zeros(t, np.float32) for _ in range(3))
    mk = np.zeros(t, np.uint32)
    sc, sh = np.zeros(len(means_list) + 1, np.float32), np.zeros(len(means_list) + 1, np.float32)
    P = params or default_event_params()
    rc = emu().emu_events_annotate(orclib.MODEL_TABLE.encode(), C.byref(P), len(means_list), off.ctypes.data,
                                   flat.ctypes.data, nm.ctypes.data, wm.ctypes.data, ws.ctypes.data, mk.ctypes.data,
                                   sc.ctypes.data, sh.ctypes.data)
    assert rc == 0
    return off, nm, wm, ws, mk, sc, sh


def calibrated(raw_i16, cal):
    """src/read_buffer.cpp:239-242 on the host (u16 reinterpretation), float32 step by step"""
    rng, off, dig = (np.float32(x) for x in cal)
    return (rng * (raw_i16.view(np.uint16).astype(np.float32) + off) / dig).astype(np.float32)


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.kind == "f":
        return a.shape == b.shape and np.array_equal(a.astype(np.float32).view(np.uint32), b.astype(np.float32).view(np.uint32))
    return np.array_equal(a.astype(np.int64), b.astype(np.int64))


def same_values(a, b):
    """bit equality, except that any NaN equals any NaN: a NaN made by arithmetic (0 / 0 for a read without events, inf -
    inf when a read's event means are all equal) has a sign and payload that differ between x86 and the GPU"""
    a, b = np.atleast_1d(np.asarray(a, np.float32)), np.atleast_1d(np.asarray(b, np.float32))
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and same_bits(a[~na], b[~nb])


def compare(got_reads, got_events, want, label=""):
    """got_*: one read's READ_DTYPE row and FULL_DTYPE events; want: oracle_read()'s pair.  Asserts equality of every
    value, bit for bit (same_values)."""
    wr, we = want
    assert int(got_reads["n_events"]) == wr["n_events"], (label, int(got_reads["n_events"]), wr["n_events"])
    for k in ("mean_event_len", "norm_scale", "norm_shift"):
        assert same_values(got_reads[k], wr[k]), (label, k, got_reads[k], wr[k])
    for k in FIELDS:
        ok = same_values(got_events[k], we[k]) if k not in ("start", "win_mask") else same_bits(got_events[k], we[k])
        assert ok, (label, k)


# ---------------------------------------------------------------- seeded reads
def synth_reads(seed, n, n_samples=4000, ragged=True):
    """n reads of the synthetic generator (tools/synth.py), of varied lengths when ragged, float32 pA"""
    import synth
    g = synth.genome(200000, seed=seed)
    sig, _ = synth.reads(g, n, n_samples=n_samples, seed=seed)
    rng = np.random.default_rng(seed)
    return [sig[i, :int(rng.integers(n_samples // 4, n_samples + 1)) if ragged else n_samples].copy() for i in range(n)]


def edge_reads(seed=11):
    """{name: float32 pA signal} that reach the edges of each stage"""
    rng = np.random.default_rng(seed)
    base = synth_reads(seed, 4, ragged=False)
    out = {}
    s = base[0].copy()
    s[600:1200] = np.float32(90.0)                                       # a stall: a constant stretch
    s[2000:2300] = np.float32(85.0) + rng.standard_normal(300).astype(np.float32) * np.float32(0.05)
    out["stall"] = s
    out["all_constant"] = np.full(3000, 77.5, np.float32)
    for L in (0, 1, 5, 6, 7, 11, 12, 13, 30):                             # shorter than the windows
        out["short_%d" % L] = base[1][:L].copy()
    out["empty"] = np.zeros(0, np.float32)
    s = base[2].copy()
    s[::97] += np.float32(500.0)                                         # events above max_mean
    s[1500:1700] = np.float32(-40.0)                                     # and below min_mean
    out["out_of_range"] = s
    few = base[3][:200].copy()                                           # a few events: under the 25-event window
    out["few_events"] = few
    return out


def long_read(seed=5, n_samples=420000):
    """a read of more than 50 000 events"""
    import synth
    g = synth.genome(400000, seed=seed)
    sig, _ = synth.reads(g, 1, n_samples=n_samples, seed=seed, dwell_mean=6.5)
    return sig[0]


def i16_reads(seed, n, n_samples=3000):
    """(int16 DAC signals, calibrations) whose calibrated values look like pA"""
    rng = np.random.default_rng(seed)
    pas = synth_reads(seed, n, n_samples)
    sigs, cals = [], []
    for i, pa in enumerate(pas):
        rngv, dig = np.float32(1400.0 + 50 * i), np.float32(8192.0 if i % 2 == 0 else 8191.0)
        off = np.float32(float(rng.integers(-10, 20)))
        raw = np.clip(np.round(pa * dig / rngv - off), -32768, 32767).astype(np.int16)
        sigs.append(raw)
        cals.append((float(rngv), float(off), float(dig)))
    return sigs, cals
