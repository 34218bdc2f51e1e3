"""Checkers of the DTW sweeps (uncalled_b200/csrc/unc_dtw_band.cuh, unc_dtw.cuh): the C restatement of the band
(oracle/unc_oracle_dtw_band.c orc_dtw_banded), the kernel sources under the warp emulator on the workspace plan of
unc_dtw_plan.hpp (tests/emul/emul_dtw_band.cpp), an independent restatement of that plan's byte count, and seeded problems
that exercise the band's edges."""
import ctypes as C
import os
import subprocess

import numpy as np

import orclib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
CSRC = os.path.join(ROOT, "uncalled_b200", "csrc")
TAB = np.fromfile(orclib.MODEL_TABLE, dtype=np.float32)
# the weights of the DTW_* presets (src/dtw.hpp:15-28), and the dtw_test driver's
WEIGHTS = [(2.0, 1.0, 100.0), (10.0, 1.0, 1000.0), (1.0, 1.0, 1.0)]
vp = C.c_void_p

_orc = None
_model = None
_emu = None


def orc():
    global _orc, _model
    if _orc is None:
        orclib.orc()                                   # builds libunc_oracle.so
        path = os.path.join(ORACLE_DIR, "libunc_oracle_dtw_band.so")
        if not os.path.exists(path):
            subprocess.run(["make", "-C", ORACLE_DIR, "-f", "dtw_band.mk"], check=True, capture_output=True)
        L = C.CDLL(path)
        L.orc_dtw_banded.argtypes = [C.POINTER(orclib.OrcModel), C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, vp, C.c_uint32,
                                     vp, C.c_uint32, C.c_uint32, vp, C.POINTER(C.c_uint64), C.POINTER(C.c_float), vp,
                                     C.POINTER(C.c_uint64)]
        M = orclib.OrcModel()
        orclib.orc().orc_model_init(C.byref(M), TAB.ctypes.data_as(orclib.f32p), 0)
        _orc, _model = L, M
    return _orc, _model


def effective_width(R, C_, W):
    """We of the definition"""
    if C_ == 1:
        return R - 1
    return max(W, -(-(R - 1) // (C_ - 1)))


def band_rows(R, C_, W):
    """(lo, hi) arrays of the definition"""
    we = effective_width(R, C_, W)
    c = (np.arange(C_, dtype=np.uint64) * np.uint64(R - 1)) // np.uint64(max(C_ - 1, 1)) if C_ > 1 else np.zeros(1, np.uint64)
    c = c.astype(np.int64)
    return np.maximum(c - we, 0), np.minimum(c + we, R - 1)


def restated(means, kmers, band, cost_kind=0, w=(1.0, 1.0, 1.0), subseq=0, want_bc=False):
    """orc_dtw_banded: (path [n, 2] of (column, row) from the end cell, score, breadcrumbs or None); rc != 0 raises"""
    L, M = orc()
    means = np.ascontiguousarray(means, np.float32)
    kmers = np.ascontiguousarray(kmers, np.uint16)
    path = np.zeros((len(means) + len(kmers), 2), np.uint64)
    n, s, nc = C.c_uint64(), C.c_float(), C.c_uint64()
    bc = None
    if want_bc:
        lo, hi = band_rows(len(kmers), len(means), band)
        bc = np.zeros(int((hi - lo + 1).sum()), np.uint8)
    rc = L.orc_dtw_banded(C.byref(M), cost_kind, subseq, w[0], w[1], w[2], means.ctypes.data, len(means), kmers.ctypes.data,
                          len(kmers), band, path.ctypes.data, C.byref(n), C.byref(s), None if bc is None else bc.ctypes.data,
                          C.byref(nc))
    if rc != 0:
        raise ValueError("orc_dtw_banded rc=%d" % rc)
    return path[:n.value].copy(), s.value, bc


def emu():
    global _emu
    if _emu is None:
        src = os.path.join(EMUL_DIR, "emul_dtw_band.cpp")
        out = os.path.join(EMUL_DIR, "libunc_emul_dtw_band.so")
        deps = [src, os.path.join(EMUL_DIR, "warp_emul.hpp")] + [os.path.join(CSRC, f) for f in (
            "unc_dtw_plan.hpp", "unc_dtw_band.cuh", "unc_dtw.cuh", "unc_device.cuh", "unc_warp.cuh")]
        if not (os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(x) for x in deps)):
            subprocess.run(["g++", "-O2", "-g", "-std=c++17", "-ffp-contract=off", "-DUNC_EMUL", "-DK2_MAXSEG=16u", "-fPIC",
                            "-shared", "-I" + EMUL_DIR, "-I" + CSRC, "-o", out, src], check=True, capture_output=True)
        L = C.CDLL(out)
        L.emu_dtw_sweep.argtypes = [vp, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_uint32, C.c_uint32] + [vp] * 9 + \
            [C.POINTER(C.c_uint64), C.c_int]
        L.emu_dtw_band_cells.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
        L.emu_dtw_band_cells.restype = C.c_uint64
        L.emu_dtw_plan_bytes.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
        L.emu_dtw_plan_bytes.restype = C.c_uint64
        L.emu_dtw_pack.argtypes = [C.c_uint32, C.c_uint32, vp, vp, C.c_uint64, vp]
        L.emu_dtw_pack.restype = C.c_uint32
        _emu = L
    return _emu


def emulated(problems, band, cost_kind=0, w=(1.0, 1.0, 1.0), n_threads=64, want_bc=False, subseq=0):
    """the kernel source under the emulator (band 0: k_dtw's full sweep, with subseq 0 NONE, 1 ROW or 2 COL):
    [(path, score, breadcrumbs or None)]"""
    L = emu()
    n = len(problems)
    moff = np.zeros(n + 1, np.uint64)
    koff = np.zeros(n + 1, np.uint64)
    poff = np.zeros(n + 1, np.uint64)
    moff[1:] = np.cumsum([len(m) for m, _ in problems])
    koff[1:] = np.cumsum([len(k) for _, k in problems])
    poff[1:] = np.cumsum([len(m) + len(k) for m, k in problems])
    am = np.ascontiguousarray(np.concatenate([m for m, _ in problems]), np.float32)
    ak = np.ascontiguousarray(np.concatenate([k for _, k in problems]), np.uint16)
    path = np.zeros((int(poff[-1]), 2), np.uint64)
    plen = np.zeros(n, np.uint64)
    score = np.zeros(n, np.float32)
    sizes = [int(L.emu_dtw_band_cells(len(k), len(m), band)) if band else len(k) * len(m) for m, k in problems]
    bc = np.zeros(max(sum(sizes), 1), np.uint8) if want_bc else None
    nbc = C.c_uint64()
    rc = L.emu_dtw_sweep(TAB.ctypes.data, cost_kind, subseq, w[0], w[1], w[2], band, n, am.ctypes.data, moff.ctypes.data, ak.ctypes.data,
                         koff.ctypes.data, path.ctypes.data, poff.ctypes.data, plen.ctypes.data, score.ctypes.data,
                         None if bc is None else bc.ctypes.data, C.byref(nbc), n_threads)
    assert rc == 0
    assert nbc.value == sum(sizes)
    out, bo = [], 0
    for i in range(n):
        b = bc[bo:bo + sizes[i]].copy() if want_bc else None
        bo += sizes[i]
        out.append((path[int(poff[i]):int(poff[i]) + int(plen[i])].copy(), float(score[i]), b))
    return out


SKIP = 0xFFFFFFFF


def sweep_bytes(shapes, W):
    """the span aligner's sweep workspace for problems [(R, C)] at half-width W (0: the full sweep), restated from the
    kernels' needs: problem records (56 bytes), breadcrumbs (R x C, or the in-band cells), hrow / vcol / corners
    (C + R + 3 ceil(R / 8) + 8 floats), the last column and row (R + C floats) or the column offsets (C + 1 u64), path room
    (R + C pairs of u64), path lengths, scores, queue; each region 256-byte aligned"""
    a = lambda x: (x + 255) // 256 * 256
    n = len(shapes)
    bc = diag = edge = path = 0
    for R, C_ in shapes:
        if W:
            lo, hi = band_rows(R, C_, W)
            bc += int((hi - lo + 1).sum())
            edge += 8 * (C_ + 1)
        else:
            bc += R * C_
            edge += 4 * (R + C_)
        diag += 4 * (C_ + R + 3 * ((R + 7) // 8) + 8)
        path += 16 * (R + C_)
    return a(56 * n) + a(bc) + a(diag) + a(edge) + a(path) + a(8 * n) + a(4 * n) + a(4)


def pack(shapes, W, budget):
    """the span aligner's launches (dtw_pack) under the emulator: (launch of each problem or SKIP, number of launches)"""
    rows = np.array([r for r, _ in shapes], np.uint32)
    cols = np.array([c for _, c in shapes], np.uint32)
    launch = np.zeros(len(shapes), np.uint32)
    n = emu().emu_dtw_pack(W, len(shapes), rows.ctypes.data, cols.ctypes.data, budget, launch.ctypes.data)
    return [int(x) for x in launch], int(n)


# (k-mers, kept means) of tests/test_z_gpu_dtw_band.py's long reads (its fixture checks them), and the budget its
# test_small_budget_skips_only_the_query_over_it gives the aligner: room for every band at W = 64 but the largest
LONG_READ_SHAPES = [(12546, 19369), (18796, 29123), (28796, 44424), (35046, 54428), (41296, 63875), (49995, 77533),
                    (2546, 3894), (7546, 11652)]


def small_budget(shapes, W):
    need = sorted(sweep_bytes([s], W) for s in shapes)
    return (need[-2] + need[-1]) // 2


def problem(rng, nr, nc, walk=True, noise=2.5):
    """a seeded (means, kmers) pair: events that follow the k-mers with stays and noise, or uniform levels"""
    km = rng.integers(0, 1024, nr).astype(np.uint16)
    if walk:
        idx = np.clip((np.arange(nc) * nr) // max(nc, 1), 0, nr - 1)
        means = (TAB[2 * km[idx].astype(np.int64)] + rng.normal(0, noise, nc)).astype(np.float32)
    else:
        means = rng.uniform(55, 135, nc).astype(np.float32)
    return means, km


# (rows, columns, W): R > C and R < C, C = 1, R = 1, a W the effective width widens (R much larger than C), bands that clip
# at the first and last rows, tile edges (R, C = 0, 1, 7 mod 8), and full bands (W >= R - 1)
SHAPES = [(1, 1, 1), (1, 9, 1), (9, 1, 1), (13, 1, 2), (1, 40, 3), (2, 2, 1), (40, 17, 1), (120, 9, 2), (64, 65, 1),
          (33, 31, 3), (57, 200, 4), (200, 57, 2), (97, 101, 8), (8, 8, 1), (16, 47, 2), (63, 129, 5), (129, 64, 3),
          (72, 73, 71), (40, 90, 39), (90, 40, 200), (7, 300, 2), (300, 7, 1), (120, 360, 12), (81, 161, 6)]


def shape_problems(seed):
    rng = np.random.default_rng(seed)
    return [(problem(rng, r, c, rng.random() < 0.75), w) for r, c, w in SHAPES]
