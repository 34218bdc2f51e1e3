"""Times the FM-index build (`uncalled index`'s bwa files) on the device builder, and on the host builder for the
smaller genome, and prints one JSON line per genome.

    python tools/bench_index_build.py [--bases 230000000] [--big-bases 1100000000] [--no-host]

Genomes: tests/masklib.py's big_genome (planted interspersed and tandem repeats, poly-A, lowercase and N runs over four
records) of --bases, and of --big-bases (device only: the host builder stops at 2 x 2^30 FM rows; 0 skips it).  For
each: the end-to-end wall time of the call (FASTA in, five files out), the CUDA-event time of the device phases
(initial sort, doubling rounds, BWT / Occ / SA output), the doubling rounds and the active rows of each, the most device
memory the build held, and the achieved bytes/s of each phase against an algorithmic byte count (the model below, also
in DESIGN.md section 4 "FM-index build").  Where both builders run, their files are compared byte for byte.  The card
name and power limit are read in the same run.  Everything is written to a temporary directory.

Algorithmic bytes (N = rows = 2 x bases + 1, M = active rows of a round, P = radix passes of a round):
  initial sort   20.5 N       (hist: 4 B atomic + text; scatter: 4 B atomic, SA, ISA, bucket start)
  a round        (92 + 32 P) M + N / 4   (compaction, snapshot, keys, P passes of 24 B key/value in and out plus the
                 8 B key read of the histogram, write-back, max-scan, rank update; the head bits)
  output         8.5 N        (SA read and text gather per row, packed BWT, Occ counts, SA samples)
P per round is taken as ceil(bits(N + 16) / 8) + ceil(bits(min(M, workspace)) / 8), the passes of a batch whose rows span
its workspace."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

WS_ROWS = 1 << 26            # UNC_FMB_DEFAULT_WS_ROWS


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().split("\n")[0]
        name, watts = [s.strip() for s in out.split(",")]
        return name, watts
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def bits(v):
    return int(v).bit_length()


def device(fa, prefix):
    import uncalled_b200._native as N
    L = N.lib()
    t0 = time.perf_counter()
    N.check(L.unc_index_build_device(fa.encode(), prefix.encode()))
    wall = time.perf_counter() - t0
    ms, rounds, peak = (C.c_float * 3)(), C.c_uint32(), C.c_uint64()
    L.unc_index_build_device_last_times(ms, C.byref(rounds), C.byref(peak))
    act = (C.c_uint64 * 64)()
    k = L.unc_index_build_device_last_active(act, 64)
    return {"wall_s": round(wall, 3), "phase_ms": [round(x, 2) for x in ms], "rounds": rounds.value,
            "active_rows": [int(act[i]) for i in range(min(k, 64))], "peak_device_bytes": peak.value}


def model(n_rows, active):
    init = 20.5 * n_rows
    kp = (bits(n_rows + 16) + 7) // 8
    rounds = sum((92 + 32 * (kp + (bits(min(m, WS_ROWS)) + 7) // 8)) * m + n_rows / 4 for m in active)
    return init, rounds, 8.5 * n_rows


def bench(fa, tmp, tag, host):
    import uncalled_b200._native as N
    r = {"genome": tag}
    d = device(fa, os.path.join(tmp, "dev"))
    r.update(d)
    with open(os.path.join(tmp, "dev.ann")) as f:
        n_rows = 2 * int(f.readline().split()[0]) + 1
    r["rows"] = n_rows
    init, rounds, out = model(n_rows, d["active_rows"])
    ms = d["phase_ms"]
    r["model_bytes"] = [init, rounds, out]
    r["achieved_bytes_per_s"] = [init / (ms[0] / 1e3), rounds / (ms[1] / 1e3) if ms[1] > 0 else None,
                                 out / (ms[2] / 1e3)]
    if host:
        t0 = time.perf_counter()
        N.check(N.lib().unc_index_build(fa.encode(), os.path.join(tmp, "host").encode()))
        r["host_wall_s"] = round(time.perf_counter() - t0, 3)
        r["files_identical"] = all(open(os.path.join(tmp, "dev." + e), "rb").read() ==
                                   open(os.path.join(tmp, "host." + e), "rb").read()
                                   for e in ("pac", "ann", "amb", "bwt", "sa"))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bases", type=int, default=230_000_000)
    ap.add_argument("--big-bases", type=int, default=1_100_000_000)
    ap.add_argument("--no-host", action="store_true")
    a = ap.parse_args()
    import masklib
    import uncalled_b200._native as N
    N.check(N.lib().unc_init(0))
    name, watts = card()
    with tempfile.TemporaryDirectory() as tmp:
        fa = os.path.join(tmp, "g.fa")
        open(fa, "wb").write(masklib.big_genome(1_000_000, seed=1))
        device(fa, os.path.join(tmp, "warm"))                        # warm-up: context, module load
        for bases, host in ((a.bases, not a.no_host), (a.big_bases, False)):
            if not bases:
                continue
            open(fa, "wb").write(masklib.big_genome(bases, seed=1))
            r = bench(fa, tmp, "big_genome(%d, seed=1)" % bases, host)
            r.update({"gpu": name, "power_limit": watts})
            print(json.dumps(r), flush=True)
            for f in os.listdir(tmp):
                if f != "g.fa":
                    os.remove(os.path.join(tmp, f))


if __name__ == "__main__":
    main()
