"""Times `mask-external` on a seeded full reference (default 1 G bases) and a 10 Mb target, at min_len 50 and
min_copy 5 (the setting of the reference's masking/README.md), and prints one JSON line.

    python tools/bench_mask_external.py [--bases 1000000000] [--target 10000000] [--repeats 3] [--check-bases 50000000]

The full reference is tests/masklib.py's big_genome: planted interspersed and tandem repeats, poly-A runs, lowercase and
N runs.  The target is two thirds copied from it and one third random.  Reported: the CUDA-event time of the build,
count and mark kernels; full-reference bases per second in the count kernels; the bytes copied to the device and the
part of the count phase not spent in count kernels (copies and host staging that were not hidden); the end-to-end time
of the call including FASTA I/O; and the achieved bytes/s of the count pass's algorithmic traffic against the H100
SXM data sheet's 3.35 TB/s.  That traffic is counted as 1 byte per full-reference position; the keys read by probes
that pass the filter are not counted, so the figure is a lower bound.  The counts of a smaller run (--check-bases of full
reference, the same target size) are checked against the numpy oracle of tests/test_mask_external.py in the same run.
The card name and power limit are read in the same run.  Everything is written to a temporary directory."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

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


def run(full_fa, target_fa, k, min_copy, prefix, n_target_pos):
    import uncalled_b200._native as N
    L = N.lib()
    counts = np.zeros(n_target_pos, np.uint32)
    sel, bp = C.c_uint64(), C.c_uint64()
    t0 = time.perf_counter()
    N.check(L.unc_mask_external(full_fa.encode(), target_fa.encode(), k, min_copy, (prefix + "m.fa").encode(),
                                (prefix + "m.bed").encode(), 0, counts.ctypes.data, C.byref(sel), C.byref(bp)))
    wall = (time.perf_counter() - t0) * 1e3
    ms = (C.c_float * 4)()
    h2d = C.c_uint64()
    L.unc_mask_external_last_times(ms, C.byref(h2d))
    return {"wall_ms": wall, "build_ms": ms[0], "count_ms": ms[1], "mark_ms": ms[2], "count_phase_ms": ms[3],
            "h2d_bytes": h2d.value, "masked_bp": bp.value, "selected": sel.value}, counts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bases", type=int, default=1_000_000_000)
    ap.add_argument("--target", type=int, default=10_000_000)
    ap.add_argument("--check-bases", type=int, default=50_000_000)
    ap.add_argument("--min-len", type=int, default=50)
    ap.add_argument("--min-copy", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    import test_mask_external as X
    import uncalled_b200._native as N
    N.check(N.lib().unc_init(0))
    k, mc = a.min_len, a.min_copy
    with tempfile.TemporaryDirectory() as tmp:
        # the check: a smaller full reference against the numpy oracle
        full, target = X.big_pair(a.check_bases, a.target, seed=a.seed)
        ffa, tfa = os.path.join(tmp, "full.fa"), os.path.join(tmp, "target.fa")
        open(ffa, "wb").write(full)
        open(tfa, "wb").write(target)
        n_t = len(X._flat(target)[2])
        got, counts = run(ffa, tfa, k, mc, os.path.join(tmp, "c_"), n_t)
        t0 = time.perf_counter()
        want = X.window_counts(full, target, k)
        oracle_ms = (time.perf_counter() - t0) * 1e3
        matches = bool(np.array_equal(counts, want))
        del full
        # the timed workload
        full, target = X.big_pair(a.bases, a.target, seed=a.seed)
        open(ffa, "wb").write(full)
        open(tfa, "wb").write(target)
        n_full = len(X._flat(full)[2])
        del full
        n_t = len(X._flat(target)[2])
        run(ffa, tfa, k, mc, os.path.join(tmp, "w_"), n_t)                   # warm-up: context, module load
        rs = [run(ffa, tfa, k, mc, os.path.join(tmp, "o_"), n_t)[0] for _ in range(a.repeats)]
    rs.sort(key=lambda r: r["count_ms"])
    r = rs[len(rs) // 2]
    traffic = n_full                                                        # 1 B per full-reference position
    name, watts = card()
    print(json.dumps({
        "workload": "mask-external seeded full reference + target", "full_bases": n_full, "target_positions": n_t,
        "min_len": k, "min_copy": mc,
        "build_ms": round(r["build_ms"], 3), "count_ms": round(r["count_ms"], 3), "mark_ms": round(r["mark_ms"], 3),
        "count_ms_all": [round(x["count_ms"], 3) for x in rs],
        "count_phase_ms": round(r["count_phase_ms"], 3),
        "not_hidden_ms": round(r["count_phase_ms"] - r["count_ms"], 3),
        "h2d_bytes": r["h2d_bytes"],
        "full_bases_per_s_count": n_full / (r["count_ms"] / 1e3),
        "end_to_end_ms": [round(x["wall_ms"], 1) for x in rs],
        "count_input_bytes_per_s": traffic / (r["count_ms"] / 1e3),
        "fraction_of_3_35_TB_s": traffic / (r["count_ms"] / 1e3) / HBM_BYTES_PER_S,
        "masked_bp": r["masked_bp"], "selected_windows": r["selected"],
        "check_full_bases": a.check_bases,
        "check_matches_oracle": matches, "oracle_ms": round(oracle_ms, 1),
        "gpu": name, "power_limit": watts}))


if __name__ == "__main__":
    main()
