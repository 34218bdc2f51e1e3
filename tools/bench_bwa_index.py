"""The BwaIndex queries on the GPU: range_to_fms over a whole contig and sa of every row (unc_bwa_range_to_fms,
unc_bwa_sa).

Genome: tools/bench_chr1.py's 230 Mb chr1-sized synthetic (230 masked N runs of 5 kb), indexed on the device in a
temporary directory.  Reported: the CUDA-event time of range_to_fms over the whole contig (both walks, after a warm-up
span) and of sa over every row (in batches of 2^26 rows, summed), with positions/s and rows/s; the wall time of the
range_to_fms call including the copies; and, beside them, the serial walk of the reference's loop as the C restatement
(oracle/unc_oracle_bwa_index.c) runs it on one host core over a 2 Mb span of the same contig, whose lists the GPU's
must equal.  The card's name and power limit are read in the same run.

    python tools/bench_bwa_index.py [--size 230000000] [--serial-span 2000000] [--out result.json]
"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=230_000_000)
    ap.add_argument("--serial-span", type=int, default=2_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import bwaindexlib as B
    import repeatslib as R
    from bench_chr1 import make_genome
    from uncalled_b200 import _native as N
    from uncalled_b200 import index as I
    L = N.lib()
    res = {"card": card(), "genome": "synthetic_chr1", "size": args.size}
    work = tempfile.mkdtemp(prefix="bench_bwa_index_")
    try:
        fa, prefix = os.path.join(work, "chr1.fa"), os.path.join(work, "chr1")
        R.write_fasta(fa, make_genome(args.size, 4242, n_runs=230, run_len=5000)[1], ["synthetic_chr1"])
        N.check(L.unc_index_build_device(fa.encode(), prefix.encode()))
        os.remove(fa)
        X = I.BwaIndex(prefix, True)
        name, ln = X.get_seqs()[0]
        X.range_to_fms(name, 1000, 200_000)                              # warm-up: device image, both kernels
        t = time.time()
        first, second = X.range_to_fms(name, 0, ln)
        wall = time.time() - t
        ms = X.last_kernel_ms()
        res.update(positions=ln, range_to_fms_kernel_ms=ms, range_to_fms_positions_per_s=ln / (ms / 1e3),
                   range_to_fms_wall_s=wall)
        print("range_to_fms", json.dumps(res), flush=True)

        st = ln // 2
        n = args.serial_span
        Rs = B.Restated(prefix)
        t = time.time()
        wa, wb = Rs.range_to_fms(name, st, st + n)
        serial = time.time() - t
        res.update(serial_span=n, serial_restatement_s=serial, serial_positions_per_s=n / serial)
        g1, g2 = X.range_to_fms(name, st, st + n)
        res["serial_span_equal"] = bool(np.array_equal(g1, wa) and np.array_equal(g2, wb))
        res["whole_contig_forward_tail_equal"] = bool(np.array_equal(second[ln - st - n:ln - st], wb))
        del first, second

        rows_total = X.size() + 1
        sa_ms, chunk = 0.0, 1 << 26
        X.sa(np.arange(0, 1 << 20, dtype=np.uint64))                     # warm-up
        for o in range(0, rows_total, chunk):
            X.sa(np.arange(o, min(o + chunk, rows_total), dtype=np.uint64))
            sa_ms += X.last_kernel_ms()
        res.update(sa_rows=rows_total, sa_kernel_ms=sa_ms, sa_rows_per_s=rows_total / (sa_ms / 1e3))
        X.destroy()
    finally:
        shutil.rmtree(work, ignore_errors=True)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
