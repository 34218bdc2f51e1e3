"""Throughput of the banded DTW sweep (`DtwAligner(band=W)`, `dtw --band W`) in one process:

- long reads: seeded reads of 60 000 - 400 000 samples against their spans on the multi-contig test genome, aligned at
  several half-widths (the full sweep skips every read over 50 000 kept means): in-band cells/s of the sweep (CUDA-event
  time), reads/s end to end (host wall clock around DtwAligner.align, which returns after the device is done) and the
  bytes of sweep workspace the reads need;
- short reads: seeded reads under the 50 000-means limit, the full sweep against the banded one on the same reads, with
  the fraction of reads whose banded score equals the full score bit for bit;
- the card's name, power limit and SM clocks, read in the same process.

Every configuration is warmed up, then the configurations are timed in alternation for --rounds rounds.

    python tools/bench_dtw_band.py [--long 48] [--short 256] [--widths 32,64,128] [--out result.json]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import dtwalignlib as D  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().split("\n")[0] if out.returncode == 0 else "unknown"


def reads(codes, n, lo, hi, seed):
    rng = np.random.default_rng(seed)
    names = sorted(codes)
    out = []
    for i in range(n):
        contig = names[i % 3]
        n_samp = int(np.exp(rng.uniform(np.log(lo), np.log(hi))))
        ln = min(n_samp // 9 + 10, len(codes[contig]) - 1)            # the read covers its whole span (about n_samp samples)
        st = int(rng.integers(0, len(codes[contig]) - ln))
        fwd = bool(rng.integers(0, 2))
        sig = D.span_signal(codes[contig][st:st + ln], fwd, rng)
        out.append(("r%04d" % i, sig, None, 0, 0, contig, st, st + ln, fwd))
    return out


def band_bytes(R, C, W):
    """sweep workspace of one banded problem: in-band breadcrumbs, hrow / vcol / corners, column offsets, path room"""
    we = R - 1 if C == 1 else min(max(W, -(-(R - 1) // (C - 1))), R - 1)
    c = (np.arange(C, dtype=np.int64) * (R - 1)) // max(C - 1, 1)
    cells = int((np.minimum(c + we, R - 1) - np.maximum(c - we, 0) + 1).sum())
    return cells + 4 * (C + R + 3 * ((R + 7) // 8) + 8) + 8 * (C + 1) + 16 * (R + C)


def run(A, q, batch):
    """(wall s, sweep ms, cells, results) of aligning q in batches"""
    res, sweep, cells = [], 0.0, 0
    t0 = time.perf_counter()
    for i in range(0, len(q), batch):
        res += A.align(q[i:i + batch])
        t, _, ce = A.last_times()
        sweep += t["sweep"]
        cells += ce
    return time.perf_counter() - t0, sweep, cells, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--long", type=int, default=48)
    ap.add_argument("--short", type=int, default=256)
    ap.add_argument("--widths", default="32,64,128")
    ap.add_argument("--short-width", type=int, default=64)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import uncalled_b200._native as N
    from uncalled_b200.dtw import DtwAligner
    widths = [int(x) for x in a.widths.split(",")]
    d = tempfile.mkdtemp()
    prefix, codes = D.multi_contig_genome(d)
    N.check(N.lib().unc_init(0))
    info = card()
    out = {"card": info}

    # ---- long reads at each width
    lq = reads(codes, a.long, 60000, 400000, seed=11)
    al = {W: DtwAligner(prefix, band=W) for W in widths}
    for W in widths:
        run(al[W], lq[:a.batch], a.batch)                                        # warm-up
    acc = {W: [0.0, 0.0, 0, None] for W in widths}
    for _ in range(a.rounds):
        for W in widths:
            wall, sweep, cells, res = run(al[W], lq, a.batch)
            acc[W][0] += wall; acc[W][1] += sweep; acc[W][2] += cells; acc[W][3] = res
    long_out = {}
    for W in widths:
        wall, sweep, cells, res = acc[W]
        assert all(r.skip is None for r in res), [r.skip for r in res if r.skip]
        ws = [band_bytes(q[7] - q[6] - 4, r.n_kept, W) for q, r in zip(lq, res)]
        long_out[W] = {"reads_per_s": a.rounds * len(lq) / wall, "sweep_cells_per_s": cells / (sweep / 1e3),
                       "sweep_ms_per_round": sweep / a.rounds, "cells_per_round": cells // a.rounds,
                       "workspace_bytes_mean": float(np.mean(ws)), "workspace_bytes_max": int(max(ws))}
    n_over = sum(r.n_kept > D.MAX_MEANS for r in acc[widths[0]][3])
    out["long"] = {"reads": len(lq), "samples": "60000:400000", "kept_means_mean": float(np.mean([r.n_kept for r in acc[widths[0]][3]])),
                   "reads_over_50000_means": n_over, "widths": long_out}

    # ---- short reads: the full sweep against the band on the same reads
    sq = reads(codes, a.short, 20000, 60000, seed=12)
    full, band = DtwAligner(prefix), DtwAligner(prefix, band=a.short_width)
    run(full, sq[:a.batch * 4], a.batch * 4)
    run(band, sq[:a.batch * 4], a.batch * 4)
    tf = [0.0, 0.0, 0]
    tb = [0.0, 0.0, 0]
    for _ in range(a.rounds):
        for acc_, A in ((tf, full), (tb, band)):
            wall, sweep, cells, res = run(A, sq, a.batch * 4)
            acc_[0] += wall; acc_[1] += sweep; acc_[2] += cells
            if A is full:
                rf = res
            else:
                rb = res
    assert all(r.skip is None for r in rf + rb)
    same = sum(np.float32(x.score).view(np.uint32) == np.float32(y.score).view(np.uint32) for x, y in zip(rf, rb))
    out["short"] = {"reads": len(sq), "samples": "20000:60000", "band": a.short_width,
                    "full": {"reads_per_s": a.rounds * len(sq) / tf[0], "sweep_ms_per_round": tf[1] / a.rounds,
                             "sweep_cells_per_s": tf[2] / (tf[1] / 1e3), "cells_per_round": tf[2] // a.rounds},
                    "banded": {"reads_per_s": a.rounds * len(sq) / tb[0], "sweep_ms_per_round": tb[1] / a.rounds,
                               "sweep_cells_per_s": tb[2] / (tb[1] / 1e3), "cells_per_round": tb[2] // a.rounds},
                    "sweep_speedup": tf[1] / tb[1], "fraction_equal_score": same / len(sq),
                    "banded_never_below_full": bool(all(y.score >= x.score for x, y in zip(rf, rb)))}
    out["card_after"] = card()
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
