"""Throughput of the signal-to-span aligner (`uncalled_b200 dtw`) on seeded reads of realistic length, in one process:

- reads/s and DTW cells/s end to end (host wall clock around DtwAligner.align, which returns after the device is done);
- the CUDA-event time of each stage -- (a) event detection, (b) mask, (c) k-mers, (d) target, (e) normalisation -- and of
  the sweep, summed over the batches;
- the reference's own dtw_test loop body (oracle/_ref ref_dtw_align) on every host CPU, on a subset of the same reads;
- the card's name, power limit and SM clock.

    python tools/bench_dtw_align.py [--reads 512] [--samples 20000:60000] [--out result.json]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import dtwalignlib as D  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().split("\n")[0] if out.returncode == 0 else "unknown"


def reads(prefix, codes, n, lo, hi, seed=7):
    rng = np.random.default_rng(seed)
    names = sorted(codes)
    out = []
    for i in range(n):
        contig = names[i % 3]
        n_samp = int(rng.integers(lo, hi + 1))
        ln = n_samp // 9 + 10
        st = int(rng.integers(0, len(codes[contig]) - ln))
        fwd = bool(rng.integers(0, 2))
        out.append(("r%04d" % i, D.span_signal(codes[contig][st:st + ln], fwd, rng), contig, st, st + ln, fwd))
    return out


def _ref_job(args):
    prefix, sig, contig, rs, re, fwd = args
    return D.ref_align(prefix, sig, contig, rs, re, fwd)["status"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=512)
    ap.add_argument("--samples", default="20000:60000")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--ref-reads", type=int, default=64)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import uncalled_b200._native as N
    from uncalled_b200.dtw import DtwAligner
    lo, hi = (int(x) for x in a.samples.split(":"))
    d = tempfile.mkdtemp()
    prefix, codes = D.multi_contig_genome(d)
    rs = reads(prefix, codes, a.reads, lo, hi)
    N.check(N.lib().unc_init(0))
    A = DtwAligner(prefix)
    q = [(r[0], r[1], None, 0, 0, r[2], r[3], r[4], r[5]) for r in rs]
    A.align(q[:a.batch])                                          # warm-up: module load, buffers, workspace
    keys = ("h2d", "events", "mask", "kmers", "target", "norm", "sweep", "total")
    tot = dict.fromkeys(keys, 0.0)
    cells = launches = 0
    t0 = time.perf_counter()
    for i in range(0, len(q), a.batch):
        res = A.align(q[i:i + a.batch])
        t, la, ce = A.last_times()
        for k in keys:
            tot[k] += t[k]
        cells += ce
        launches += la
        assert all(r.skip is None for r in res)
    wall = time.perf_counter() - t0
    n_cpu = os.cpu_count() or 1
    sub = [(prefix,) + r[1:] for r in rs[:a.ref_reads]]
    t1 = time.perf_counter()
    with ProcessPoolExecutor(n_cpu) as ex:
        st = list(ex.map(_ref_job, sub, chunksize=1))
    ref_wall = time.perf_counter() - t1
    assert all(s == 0 for s in st)
    stages = ("events", "mask", "kmers", "target", "norm")
    out = {"card": card(), "reads": len(q), "samples": a.samples, "batch": a.batch, "wall_s": wall,
           "reads_per_s": len(q) / wall, "cells": cells, "cells_per_s": cells / wall, "sweep_launches": launches,
           "device_ms": tot, "stage_share_of_sweep": {k: tot[k] / tot["sweep"] for k in stages},
           "sweep_cells_per_s": cells / (tot["sweep"] / 1e3),
           "reference": {"cpus": n_cpu, "reads": len(sub), "wall_s": ref_wall, "reads_per_s": len(sub) / ref_wall}}
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
