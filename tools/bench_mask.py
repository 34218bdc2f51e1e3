"""Times `mask-internal` on a chr1-sized seeded genome (default 230 Mb, k = 10, 30 iterations, the setting the
reference's masking/README.md recommends) and prints one JSON line.

    python tools/bench_mask.py [--bases 230000000] [--k 10] [--iters 30] [--repeats 3]

Reported: the CUDA-event time of the device loop (every pass and argmax), the end-to-end time of the call including
reading and writing the FASTA, bases x iterations per second, and the achieved bytes/s of the algorithmic traffic
(per pass n bytes read + n written, plus the 4^k x 4 B histogram read once by the argmax) against the H100 SXM data
sheet's 3.35 TB/s.  The output is checked against the numpy oracle of tests/masklib.py, whose time is reported as
the CPU comparison.  The card name and power limit are read in the same run.  Everything is written to a temporary
directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().split("\n")[0]
        name, watts = [s.strip() for s in out.split(",")]
        return name, watts
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bases", type=int, default=230_000_000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    import masklib as M
    import uncalled_b200 as U
    from uncalled_b200 import mask as UM
    with tempfile.TemporaryDirectory() as tmp:
        data = M.big_genome(a.bases, seed=a.seed)
        fa = os.path.join(tmp, "genome.fa")
        open(fa, "wb").write(data)
        prefix = os.path.join(tmp, "out_")
        U.mask_internal(fa, a.k, min(a.iters, 2), prefix, log=None)          # warm-up: context, module load
        kms, walls = [], []
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            log = U.mask_internal(fa, a.k, a.iters, prefix, log=None)
            walls.append((time.perf_counter() - t0) * 1e3)
            kms.append(UM.last_kernel_ms())
        got = open(prefix + "mask%d.fa" % a.iters, "rb").read()
        t0 = time.perf_counter()
        want, want_log = M.oracle(data, a.k, a.iters)
        cpu_ms = (time.perf_counter() - t0) * 1e3
    n_bases = sum(len(s) for s in M.read_fasta(data)[1])
    kms.sort()
    walls.sort()
    km = kms[len(kms) // 2]
    passes = a.iters + 1
    traffic = passes * 2 * n_bases + a.iters * 4 ** a.k * 4
    name, watts = card()
    print(json.dumps({
        "workload": "mask-internal seeded genome", "bases": n_bases, "k": a.k, "iters": a.iters, "iters_done": len(log),
        "kernel_ms_median": round(km, 3), "kernel_ms_all": [round(x, 3) for x in kms],
        "end_to_end_ms_median": round(walls[len(walls) // 2], 1),
        "bases_x_iters_per_s": n_bases * a.iters / (km / 1e3),
        "algorithmic_bytes": traffic, "achieved_bytes_per_s": traffic / (km / 1e3),
        "fraction_of_3_35_TB_s": traffic / (km / 1e3) / HBM_BYTES_PER_S,
        "oracle_ms": round(cpu_ms, 1), "matches_oracle": got == want and log == want_log,
        "gpu": name, "power_limit": watts}))


if __name__ == "__main__":
    main()
