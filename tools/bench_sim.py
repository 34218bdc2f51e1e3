"""Times `uncalled sim` (uncalled_b200/sim.py run_sim) on the GPU with the wall clock: a synthetic 512-channel control
run whose reads are seeded tools/synth.py signals on the g200k test genome (half on-target, half random sequence, int16
with a calibration, as fast5 reads are), replayed with the activity pattern of a synthetic UNCALLED run.

Prints one JSON line: the card name and power limit (read in the same run), simulated seconds per wall second, signal
seconds mapped per wall second, the p50/p99 of unc_stream_last_step_ms and of the chunks per step, the share of the
loop's wall time spent outside unc_stream_step (host gather, copies issued by the step excluded), and the counts of
ejected / kept / ended reads.  Fails without a GPU.

    python tools/bench_sim.py [--seconds 60] [--reads 2048] [--sim-speed 1.0] [--channels 512]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip().split("\n")[0]
    name, watts = [s.strip() for s in out.split(",")]
    return name, watts


class TimedStream:
    """The GPU StreamMapper with every step timed on the host (a step returns after its results are copied back)."""

    def __init__(self, inner):
        self.inner, self.step_s, self.step_ms, self.chunks = inner, 0.0, [], []

    def step(self, descs, n, flat, res):
        t = time.perf_counter()
        self.inner.step(descs, n, flat, res)
        self.step_s += time.perf_counter() - t
        self.step_ms.append(self.inner.last_step_ms())
        self.chunks.append(sum(1 for i in range(n) if descs[i].n_samples))

    def close(self):
        self.inner.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=60.0, help="simulated sequencing time after the first mux scan")
    ap.add_argument("--reads", type=int, default=2048)
    ap.add_argument("--read-samples", type=int, default=16000)
    ap.add_argument("--channels", type=int, default=512)
    ap.add_argument("--sim-speed", type=float, default=1.0)
    ap.add_argument("--seed", type=int, default=5)
    a = ap.parse_args()

    import uncalled_b200._native as N
    if N.lib().unc_device_count() < 1:
        raise SystemExit("bench_sim needs a CUDA device")
    name, watts = card()

    import synth
    import synthdata
    import test_sim
    from uncalled_b200 import sim, stream
    from uncalled_b200.api import Conf, RealtimePool
    from uncalled_b200.mapper import Index

    prefix, g = synthdata.get_index("g200k")
    on, _ = synth.reads(g, a.reads, a.read_samples, seed=a.seed, frac_random=0.0)
    off, _ = synth.reads(g, a.reads, a.read_samples, seed=a.seed + 1, frac_random=1.0)
    is_on = np.arange(a.reads) % 2 == 0
    cal = test_sim.CAL
    dac = np.round(np.where(is_on[:, None], on, off) * cal[2] / cal[0] - cal[1]).astype(np.int16)
    ids = ["%s%d" % ("on" if is_on[i] else "off", i) for i in range(a.reads)]
    reads = [(ids[i], 1000 + i, dac[i], cal) for i in range(a.reads)]

    with tempfile.TemporaryDirectory() as d:
        paths = test_sim.write_run_fixture(d, ids, a.channels, seq_time=a.seconds, read_time=a.read_samples / 4000.0,
                                           seed=a.seed)
        conf = Conf()
        conf.bwa_prefix, conf.num_channels, conf.sim_speed = prefix, a.channels, a.sim_speed
        conf.realtime_mode, conf.min_ch_reads = RealtimePool.ENRICH, 1
        conf.unc_seqsum, conf.ctl_seqsum, conf.unc_paf = paths["unc_seqsum.txt"], paths["ctl_seqsum.txt"], paths["unc.paf"]
        index = Index(prefix, device=conf.device)
        p = N.default_params()
        p.max_events, p.max_paths, p.seed_len = conf.max_events, conf.max_paths, conf.seed_len
        p.bp_per_sec, p.sample_rate = conf.bp_per_sec, conf.sample_rate
        chunk_len = int(np.float32(conf.chunk_time) * np.float32(conf.sample_rate))
        backend = TimedStream(stream.StreamMapper(index, a.channels, chunk_len, max_chunks=conf.max_chunks, params=p))
        out = io.StringIO()
        t0 = time.perf_counter()
        client = sim.run_sim(conf, [], out, log=io.StringIO(), backend=backend, index=index, reads=reads)
        wall = time.perf_counter() - t0
        loop_s = time.monotonic() - client._t0          # from run(): the pattern and the reads are loaded before
        runtime = client.get_runtime()

    tags = [[x[:2] for x in l.split("\t")[12:]] for l in out.getvalue().splitlines() if not l.startswith("#")]
    steps = np.array(backend.step_ms) if backend.step_ms else np.zeros(1)
    per = np.array(backend.chunks) if backend.chunks else np.zeros(1)
    print(json.dumps({
        "gpu": name, "power_limit": watts, "channels": a.channels, "reads": a.reads, "sim_speed": a.sim_speed,
        "sim_seconds": round(runtime, 2), "loop_wall_seconds": round(loop_s, 2), "total_wall_seconds": round(wall, 2),
        "sim_seconds_per_wall_second": round(runtime / loop_s, 3) if loop_s else None,
        "signal_seconds_mapped_per_wall_second": round(int(per.sum()) * chunk_len / conf.sample_rate / loop_s, 1),
        "steps": len(backend.step_ms), "step_ms_p50": round(float(np.percentile(steps, 50)), 3),
        "step_ms_p99": round(float(np.percentile(steps, 99)), 3),
        "chunks_per_step_p50": float(np.percentile(per, 50)), "chunks_per_step_p99": float(np.percentile(per, 99)),
        "share_outside_stream_step": round(1.0 - backend.step_s / loop_s, 3) if loop_s else None,
        "ejected": sum("ej" in t for t in tags), "kept": sum("kp" in t for t in tags), "ended": sum("en" in t for t in tags),
    }))


if __name__ == "__main__":
    main()
