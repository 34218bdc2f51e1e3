"""Throughput of `events` (uncalled_b200.signal, unc_events_*): reads/s and samples/s.

Workloads: N int16 reads of L samples (default 10 000 x 4 000, synthetic, calibrated on the device), and the golden
fast5 fixtures (tests/golden/fast5).  Per workload:
  device   samples already on the device (a torch tensor), CUDA-event time of the detection + annotation kernels
  e2e      wall time of staging, copy in, kernels, copy back of the per-read results and fetch of every event
  oracle   the C restatement (oracle/unc_oracle_events.c) on all host threads, one read per task
Prints one JSON line per workload.

    python tools/bench_events.py [--reads 10000] [--len 4000] [--reps 5] [--oracle-reads 2000]
"""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import eventslib as E  # noqa: E402
from uncalled_b200.signal import SignalProcessor  # noqa: E402


def measure(proc, sigs, cals, pas, reps, oracle_reads):
    import torch
    flat, descs = proc.stage(sigs, cals)
    n_samp = int(descs["n_samples"].sum())
    dev = torch.from_numpy(flat).cuda()
    torch.cuda.synchronize()
    proc.run_staged(dev.data_ptr(), descs, fetch=False, on_device=True)          # warm-up
    kern = []
    for _ in range(reps):
        proc.run_staged(dev.data_ptr(), descs, fetch=False, on_device=True)
        t = proc.last_times()
        kern.append(t["detect"] + t["annotate"])
    e2e = []
    for _ in range(reps):
        t0 = time.perf_counter()
        res = proc.run(sigs, cals)
        e2e.append(time.perf_counter() - t0)
    k_ms, e_s = float(np.median(kern)), float(np.median(e2e))
    sub = pas[:oracle_reads]
    threads = os.cpu_count() or 1
    t0 = time.perf_counter()
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(E.oracle_read, sub))
    o_s = time.perf_counter() - t0
    o_samp = sum(len(p) for p in sub)
    return {"reads": len(sigs), "samples": n_samp, "events": int(len(res.events)),
            "device_kernels_ms": k_ms, "device_reads_per_s": len(sigs) / (k_ms / 1e3),
            "device_samples_per_s": n_samp / (k_ms / 1e3),
            "e2e_s": e_s, "e2e_reads_per_s": len(sigs) / e_s, "e2e_samples_per_s": n_samp / e_s,
            "oracle_threads": threads, "oracle_reads": len(sub), "oracle_reads_per_s": len(sub) / o_s,
            "oracle_samples_per_s": o_samp / o_s, "times_ms_last_run": proc.last_times()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=10000)
    ap.add_argument("--len", type=int, default=4000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-reads", type=int, default=2000)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--out", type=str, default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    import subprocess
    import torch
    proc = SignalProcessor(device=a.device)
    q = subprocess.run(["nvidia-smi", "-i", str(a.device), "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True).stdout.strip().split(", ")
    head = {"gpu": torch.cuda.get_device_name(a.device), "power_limit_w": float(q[1]) if len(q) > 3 else None,
            "sm_clock_mhz": float(q[2]) if len(q) > 3 else None, "sm_max_clock_mhz": float(q[3]) if len(q) > 3 else None,
            "host_threads": os.cpu_count()}
    lines = [head]

    def emit(d):
        print(json.dumps(d))
        lines.append(d)
    print(json.dumps(head))
    sigs, cals = [], []
    per = 500
    for s0 in range(0, a.reads, per):
        x, c = E.i16_reads(1000 + s0, min(per, a.reads - s0), n_samples=a.len)
        sigs += [np.resize(v, a.len) for v in x]
        cals += c
    pas = [E.calibrated(s, c) for s, c in zip(sigs, cals)]
    emit({"workload": "synthetic_i16_%dx%d" % (a.reads, a.len), **measure(proc, sigs, cals, pas, a.reps, a.oracle_reads)})
    from uncalled_b200.fast5 import Fast5File
    import glob
    reads = []
    for path in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "fast5", "*.fast5"))):
        with Fast5File(path) as f:
            reads += f.load(0)
    emit({"workload": "golden_fast5", **measure(proc, [r.signal for r in reads], [r.calibration for r in reads],
                                                [r.pa() for r in reads], a.reps, a.oracle_reads)})
    t0 = time.perf_counter()
    res = proc.run([r.signal for r in reads], [r.calibration for r in reads])
    import uncalled_b200.cli as cli
    t1 = time.perf_counter()
    text = cli.format_events([r.read_id for r in reads], res)
    t2 = time.perf_counter()
    emit({"workload": "golden_fast5_tsv", "events": len(res.events), "run_s": t1 - t0, "format_s": t2 - t1,
          "format_events_per_s": len(res.events) / (t2 - t1), "bytes": len(text)})
    proc.close()
    if a.out:
        with open(a.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
