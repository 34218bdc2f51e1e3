"""Times `map-ord` on the GPU: the device replay (api.MapPoolOrd over unc_stream_replay) against the host-stepped
MapPoolOrd loop over api.RealtimePool (one unc_stream_step per update, tests/replaylib.py host_map_ord), alternating
the two in one run, on a seeded synthetic run: 512 channels, several int16 reads per channel with increasing start times,
about half of them from the genome, at 0.1125 s and 1 s chunks.

Prints one JSON line per chunk time: the card name and power limit (read in the same run), and for each path the wall
seconds of every repetition, chunks/s, reads/s and seconds of signal replayed per wall second; `identical` says whether
both paths gave the same Paf lines in the same order.  Fails without a GPU.

    python tools/bench_map_ord.py [--channels 512] [--reads-per-channel 3] [--samples 16000] [--genome g200k] [--reps 2]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from bench_sim import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=512)
    ap.add_argument("--reads-per-channel", type=int, default=3)
    ap.add_argument("--samples", type=int, default=16000)
    ap.add_argument("--genome", default="g200k")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--chunk-times", default="0.1125,1.0")
    a = ap.parse_args()

    import numpy as np
    import replaylib as RL
    import synthdata
    from uncalled_b200 import api, _native as N

    N.check(N.lib().unc_init(0))
    prefix, g = synthdata.get_index(a.genome)
    reads = RL.synthetic_run(g, a.channels, a.reads_per_channel, a.samples, seed=2024, int16=True)
    name, watts = card()
    for ct in (float(x) for x in a.chunk_times.split(",")):
        conf = api.Conf()
        conf.bwa_prefix, conf.num_channels, conf.chunk_time = prefix, a.channels, ct
        L = int(np.float32(ct) * np.float32(conf.sample_rate)) & 0xFFFF
        chans = RL.order_channels(reads, a.channels, conf.max_chunks * L)
        n_samples = sum(len(r.signal) for q in chans for r in q)
        index = api.Index(prefix, device=0)

        def device():
            pool = api.MapPoolOrd(conf, index=index)
            from uncalled_b200.stream import StreamMapper
            p = N.default_params()
            pool.backend = StreamMapper(index, a.channels, L, params=p)
            for r in reads:
                pool.queue_read(r.id, r.signal, r.channel, r.number, r.start, r.cal)
            pool.load_fast5s()
            t0 = time.perf_counter()
            out = []
            while pool.running():
                out += pool.update()
            dt = time.perf_counter() - t0
            pool.stop()
            return dt, out

        def host():
            from uncalled_b200.stream import StreamMapper
            p = N.default_params()
            pool = api.RealtimePool(conf, backend=StreamMapper(index, a.channels, L, params=p), index=index)
            t0 = time.perf_counter()
            out = [p for _, p in RL.host_map_ord(pool, chans, L)]
            dt = time.perf_counter() - t0
            pool.stop_all()
            return dt, out

        device()                                            # warm-up: module load, first launches
        res = {"device": [], "host": []}
        outs = {}
        for _ in range(a.reps):
            for k, fn in (("host", host), ("device", device)):
                dt, out = fn()
                res[k].append(dt)
                outs[k] = out
        chunks = sum(p.chunks for p in outs["device"])
        n_reads = len(outs["device"])
        row = {"bench": "map_ord", "card": name, "power_limit": watts, "channels": a.channels, "reads": n_reads,
               "chunk_time": ct, "chunks": chunks, "signal_s": n_samples / conf.sample_rate,
               "identical": [RL.paf_fields(p) for p in outs["device"]] == [RL.paf_fields(p) for p in outs["host"]]}
        for k, ts in res.items():
            best = min(ts)
            row[k] = {"wall_s": [round(t, 3) for t in ts], "chunks_per_s": round(chunks / best, 1),
                      "reads_per_s": round(n_reads / best, 1),
                      "signal_s_per_wall_s": round(n_samples / conf.sample_rate / best, 1)}
        row["speedup"] = round(min(res["host"]) / min(res["device"]), 3)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
