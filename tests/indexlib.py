"""Test support for the device FM-index builder (never imported by the product).

- `FIXTURES`: the seeded FASTA inputs that the device builder must index exactly as the host builder does;
- `big_fasta`: the seeded 1.1 Gbp genome (2.2e9 FM rows) whose bwa-built files are digested in
  tests/golden/index_build_device_golden.json (made by tools/make_index_device_golden.py);
- `emu_index_build`: the device source run on the CPU under the warp emulator (tests/emul/emul_index_build.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

import masklib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
BIG_GOLDEN = os.path.join(ROOT, "tests", "golden", "index_build_device_golden.json")
EXTS = ("pac", "ann", "amb", "bwt", "sa")

BIG_SPEC = {"n": 1_100_000_000, "seed": 2026, "n_records": 5}


def big_fasta():
    """the 1.1 Gbp genome: masklib.big_genome's repeats, poly-A, lowercase and N runs over five records"""
    return masklib.big_genome(BIG_SPEC["n"], seed=BIG_SPEC["seed"], n_records=BIG_SPEC["n_records"])


# ---------------------------------------------------------------- fixtures (name -> FASTA bytes)

def _rand(rng, n):
    return np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)].tobytes()


def _revcomp(s):
    return s[::-1].translate(bytes.maketrans(b"ACGTacgt", b"TGCAtgca"))


def _wrap(name, seq, width=60):
    return b">" + name + b"\n" + b"".join(seq[i:i + width] + b"\n" for i in range(0, len(seq), width))


def fx_synth(seed):
    import synth
    return _wrap(b"synth%d" % seed, np.frombuffer(b"ACGT", np.uint8)[synth.genome(30000 + 7000 * seed, seed)].tobytes())


def fx_multi_iupac():
    """multi-record FASTA with N runs, IUPAC codes, lowercase, headers with comments"""
    rng = np.random.default_rng(31)
    out = b""
    for r in range(4):
        s = bytearray(_rand(rng, 5000 + 1300 * r))
        for b in b"NNNNRYKMSWBDHVn":
            p, L = int(rng.integers(0, len(s) - 300)), int(rng.integers(1, 300))
            s[p:p + L] = bytes([b]) * L
        s[100:400] = bytes(s[100:400]).lower()
        out += _wrap(b"rec%d some comment %d" % (r, r), bytes(s), 50 + r)
    return out


def fx_polya():
    rng = np.random.default_rng(32)
    return _wrap(b"polya", _rand(rng, 3000) + b"A" * 20000 + _rand(rng, 2000) + b"T" * 20000 + _rand(rng, 500))


def fx_tandem():
    """tandem repeats of period 1 .. 7 between random sequence"""
    rng = np.random.default_rng(33)
    parts = []
    for p in range(1, 8):
        parts.append(_rand(rng, 700))
        parts.append(_rand(rng, p) * (3000 // p))
    return _wrap(b"tandem", b"".join(parts))


def fx_block_repeats():
    """a 10 kb block repeated 8 times, some copies reverse-complemented, with random spacers"""
    rng = np.random.default_rng(34)
    blk = _rand(rng, 10000)
    parts = []
    for c in range(8):
        parts.append(_rand(rng, int(rng.integers(0, 300))))
        parts.append(_revcomp(blk) if c in (2, 5, 6) else blk)
    return _wrap(b"blocks", b"".join(parts))


def fx_palindrome():
    """a record that is its own reverse complement, and a second record"""
    rng = np.random.default_rng(35)
    h = _rand(rng, 12000)
    return _wrap(b"pal", h + _revcomp(h)) + _wrap(b"other", _rand(rng, 3001))


def fx_len(n, seed=36):
    rng = np.random.default_rng(seed + n)
    return _wrap(b"tiny%d" % n, _rand(rng, n))


TINY_LENGTHS = (1, 2, 15, 16, 17, 31, 32, 33, 127, 128, 129)

FIXTURES = {"synth1": lambda: fx_synth(1), "synth2": lambda: fx_synth(2), "synth3": lambda: fx_synth(3),
            "multi_iupac": fx_multi_iupac, "polya": fx_polya, "tandem": fx_tandem, "block_repeats": fx_block_repeats,
            "palindrome": fx_palindrome, "tiny_AAAA": lambda: _wrap(b"a", b"A" * 40),
            "tiny_ACAC": lambda: _wrap(b"ac", b"AC" * 37 + b"A")}
FIXTURES.update({"len%d" % n: (lambda n=n: fx_len(n)) for n in TINY_LENGTHS})


def fixture(name):
    return FIXTURES[name]()


def example():
    """(FASTA bytes, {ext: bytes}) of the shipped example reference and its bwa index files"""
    z = np.load(os.path.join(ROOT, "tests", "golden", "example_index_files.npz"))
    return z["fasta"].tobytes(), {e: z[e].tobytes() for e in EXTS}


# ---------------------------------------------------------------- the emulator

_lib = None


def emu_lib():
    global _lib
    if _lib is None:
        src = os.path.join(EMUL_DIR, "emul_index_build.cpp")
        out = os.path.join(EMUL_DIR, "libunc_emul_index_build.so")
        csrc = os.path.join(ROOT, "uncalled_b200", "csrc")
        deps = [src, os.path.join(EMUL_DIR, "warp_emul.hpp"), os.path.join(ROOT, "include", "unc_b200.h")] + \
            [os.path.join(csrc, f) for f in ("unc_fmb.cuh", "unc_fmb_run.hpp", "unc_index_host.hpp", "unc_device.cuh",
                                             "unc_warp.cuh")]
        if not (os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps)):
            subprocess.run(["g++", "-O2", "-g", "-std=c++17", "-DUNC_EMUL", "-DK2_MAXSEG=16u", "-fPIC", "-shared",
                            "-I" + EMUL_DIR, "-I" + csrc, "-o", out, src], check=True, capture_output=True)
        L = C.CDLL(out)
        L.emu_index_build.argtypes = [C.c_char_p, C.c_char_p, C.c_uint64]
        L.emu_index_build_rounds.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64), C.c_void_p]
        L.emu_index_build_rounds.restype = C.c_uint32
        _lib = L
    return _lib


def emu_index_build(fasta, prefix, ws_rows=0):
    """(status, {"active": [...], "batches": [...], "ws_rows": int, "peak_bytes": int, "model_bytes": int}) of the device
    builder's source on the CPU; model_bytes is the device memory the library checks for before it starts"""
    L = emu_lib()
    rc = L.emu_index_build(fasta.encode(), prefix.encode(), ws_rows)
    act, bat, ws = np.zeros(64, np.uint64), np.zeros(64, np.uint64), C.c_uint64()
    by = np.zeros(2, np.uint64)
    k = L.emu_index_build_rounds(act.ctypes.data, bat.ctypes.data, 64, C.byref(ws), by.ctypes.data)
    return rc, {"active": act[:k].tolist(), "batches": bat[:k].tolist(), "ws_rows": ws.value,
                "peak_bytes": int(by[0]), "model_bytes": int(by[1])}


def read_files(prefix):
    return {e: open(prefix + "." + e, "rb").read() for e in EXTS}
