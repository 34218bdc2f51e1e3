"""CPU sweep of the mapper kernel's worker warps (unc_k2v2.cuh) under the emulator: many bench-like reads per
index, PAF fields and the children / sources / seeds / clusters counters against the oracle, in parallel processes.
    python tools/emul_v2_sweep.py <index name> <first read> <n reads> [seed [noise_mult [max_paths [warps per CTA]]]]"""
import os
import sys
import time
from multiprocessing import Pool
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools"), ROOT]
import numpy as np

name = sys.argv[1] if len(sys.argv) > 1 else "g200k"
first = int(sys.argv[2]) if len(sys.argv) > 2 else 0
n = int(sys.argv[3]) if len(sys.argv) > 3 else 256
seed = int(sys.argv[4]) if len(sys.argv) > 4 else 7
noise = float(sys.argv[5]) if len(sys.argv) > 5 else 1.0
maxp = int(sys.argv[6]) if len(sys.argv) > 6 else 10000
n_warps = int(sys.argv[7]) if len(sys.argv) > 7 else 8


def work(job):
    import emulib, orclib, synth, synthdata
    lo, hi = job
    prefix, g = synthdata.get_index(name)
    sig, _ = synth.reads(g, first + n, 4000, seed=seed, noise_mult=noise)
    E = emulib.Emu(prefix)
    O = orclib.Oracle(prefix)
    E.params.max_paths = O.params.max_paths = maxp
    cnt = lambda r: (r.n_children, r.n_sources, r.n_seeds, r.n_clusters)
    bad = []
    sigs = [sig[i] for i in range(lo, hi)]
    recs = E.map_batch(sigs, n_warps=n_warps)[0]
    for i, r in zip(range(lo, hi), recs):
        w = O.map_read(sig[i])
        if (emulib.paf_tuple(r), cnt(r)) != (orclib.paf_tuple(w), cnt(w)) or r.status != 0:
            bad.append((i, emulib.paf_tuple(r), orclib.paf_tuple(w), cnt(r), cnt(w), r.status))
    return bad


if __name__ == "__main__":
    import emulib
    emulib.build()
    t0 = time.time()
    step = 4
    jobs = [(i, min(i + step, first + n)) for i in range(first, first + n, step)]
    bad = []
    with Pool(min(8, os.cpu_count() or 1)) as p:
        for b in p.imap_unordered(work, jobs):
            bad += b
    for b in sorted(bad):
        print("MISMATCH", b)
    print("SWEEP %s reads [%d, %d) seed %d noise %.1f max_paths %d: %d mismatches, %.0f s" % (name, first, first + n, seed, noise, maxp, len(bad), time.time() - t0))
