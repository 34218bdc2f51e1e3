"""Deterministic synthetic indexes for tests and bench: genome from tools/synth.py, FM index
from the PRODUCT's own builder (unc_index_build, byte-identical to bwa), .uncl threshold line
from the committed fixture tests/golden/synth_uncl.json (made by the real reference)."""
import json
import os
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import synth  # noqa: E402

# Outside the source tree, which may be read-only where the benchmark runs; UNC_DATA_DIR overrides.
CACHE = os.environ.get("UNC_DATA_DIR") or os.path.join(tempfile.gettempdir(), "uncalled_b200_data_%d" % os.getuid())
EXTS = (".fa", ".bwt", ".sa", ".ann", ".amb", ".pac", ".uncl")


def get_index(name):
    """Returns (prefix, genome array).  Builds into CACHE on first use: in a private directory first, then moved into
    place with the .uncl file last, so that a concurrent or interrupted build is never taken for a complete one."""
    meta = json.load(open(os.path.join(ROOT, "tests", "golden", "synth_uncl.json")))[name]
    os.makedirs(CACHE, mode=0o700, exist_ok=True)
    prefix = os.path.join(CACHE, name)
    g = synth.genome(meta["size"], meta["seed"])
    if not all(os.path.exists(prefix + e) for e in EXTS):
        work = tempfile.mkdtemp(dir=CACHE)
        try:
            tmp = os.path.join(work, name)
            synth.write_fasta(tmp + ".fa", g)
            from uncalled_b200 import _native as N
            rc = N.lib().unc_index_build((tmp + ".fa").encode(), tmp.encode())
            if rc != 0:
                raise RuntimeError("unc_index_build failed: %d" % rc)
            open(tmp + ".uncl", "w").write(meta["uncl"])
            for e in EXTS:
                os.replace(tmp + e, prefix + e)
        finally:
            shutil.rmtree(work, ignore_errors=True)
    return prefix, g


def low_complexity_genome(seed=77):
    """400 kb of random sequence cut by low-complexity stretches: homopolymer runs of 20..3000 bases, dinucleotide and
    trinucleotide tandem repeats and a 5-base unit repeated, about 40% of the genome in all.  Its FM index has k-mers
    whose ranges span more than 2^16 rows, and many paths that share an fm_start (A^k for every run length k starts where
    the longest run's suffixes do)."""
    import numpy as np
    rng = np.random.default_rng(seed)
    parts, n = [], 0
    while n < 400000:
        r = rng.integers(0, 4, int(rng.integers(200, 1500)), dtype=np.uint8)
        kind = int(rng.integers(0, 4))
        if kind == 0:
            s = np.full(int(rng.integers(20, 3000)), int(rng.integers(0, 4)), np.uint8)
        else:
            unit = rng.integers(0, 4, (2, 3, 5)[kind - 1], dtype=np.uint8)
            s = np.tile(unit, int(rng.integers(10, 400)))
        parts += [r, s]
        n += len(r) + len(s)
    return np.concatenate(parts)


def get_low_complexity_index():
    """(prefix, genome) of low_complexity_genome(), built like get_index; the .uncl threshold line is g200k's."""
    meta = json.load(open(os.path.join(ROOT, "tests", "golden", "synth_uncl.json")))["g200k"]
    name = "lowcomplex77"
    os.makedirs(CACHE, mode=0o700, exist_ok=True)
    prefix = os.path.join(CACHE, name)
    g = low_complexity_genome()
    if not all(os.path.exists(prefix + e) for e in EXTS):
        work = tempfile.mkdtemp(dir=CACHE)
        try:
            tmp = os.path.join(work, name)
            synth.write_fasta(tmp + ".fa", g)
            from uncalled_b200 import _native as N
            rc = N.lib().unc_index_build((tmp + ".fa").encode(), tmp.encode())
            if rc != 0:
                raise RuntimeError("unc_index_build failed: %d" % rc)
            open(tmp + ".uncl", "w").write(meta["uncl"])
            for e in EXTS:
                os.replace(tmp + e, prefix + e)
        finally:
            shutil.rmtree(work, ignore_errors=True)
    return prefix, g
