"""Builds the simulator fixtures and goldens under tests/golden/sim/ (needs the reference tree for parts 1 and 2):

1. seqsum/PAF fixtures: synthetic control and UNCALLED sequencing summaries with 4-mux scan blocks, long gaps and
   several channels, and an UNCALLED PAF with ej / ub tags.  The reference's own uncalled/sim_utils.py load_sim runs
   on them against a recording client; the call sequence goes to load_sim_golden.json.
2. a ClientSim scenario (intervals, a mux scan, wrapping gaps and delays, unblocks, stop_receiving_read, a read that
   is missing): run through the reference's own src/client_sim.cpp, built with tools/sim_ref/ and its clock set by the
   script; every get_read_chunks / unblock_read result goes to client_golden.json.
3. (--emul) the end-to-end run_sim scenario of tests/test_sim.py on the emulated device; its PAF lines without the
   timing tags go to run_golden.json, which the GPU test compares against.

    python tools/make_sim_golden.py [--ref /root/reference] [--emul]
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "sim")
HEADER = ["filename", "read_id", "run_id", "channel", "mux", "start_time", "duration", "num_events", "passes_filtering",
          "template_start", "num_events_template", "template_duration", "sequence_length_template", "mean_qscore_template"]


def _rid(rng):
    h = "".join("0123456789abcdef"[i] for i in rng.integers(0, 16, 32))
    return "%s-%s-%s-%s-%s" % (h[:8], h[8:12], h[12:16], h[16:20], h[20:])


def _scan(rows, rng, t0, chans, prefix):
    """A mux scan: four blocks (mux 1..4) of overlapping reads on every channel, 3 s apart."""
    t = t0
    for mux in (1, 2, 3, 4):
        for ch in chans:
            for k in range(2):
                st = t + 0.5 * k + 0.1 * (ch % 3)
                rows.append((prefix, _rid(rng), ch, mux, st, 2.0 + 0.2 * k))
        t += 6.0
    return t


def _seq(rows, rng, t0, t1, chans, muxes, prefix, long_gap_chans=()):
    """Sequencing between scans: every channel keeps one mux and reads one read after another with short gaps; the
    channels in `long_gap_chans` pause for a long time once."""
    for ch in chans:
        t = t0 + rng.uniform(0, 0.5)
        paused = False
        while True:
            ln = rng.uniform(4, 25)
            if t + ln > t1:
                break
            rows.append((prefix, _rid(rng), ch, muxes[ch], t, ln))
            t += ln + rng.uniform(0.2, 2.0)
            if ch in long_gap_chans and not paused and t > (t0 + t1) / 2:
                t += 120.0
                paused = True


def make_seqsum(path, seed, chans, muxes, long_gap_chans, periods):
    rng = np.random.default_rng(seed)
    rows = []
    t = 0.0
    for k, (t_len) in enumerate(periods):
        t = _scan(rows, rng, t, chans, "scan")
        _seq(rows, rng, t + 1.5, t + 1.5 + t_len, chans, muxes, "seq", long_gap_chans if k == 0 else ())
        t += 1.5 + t_len + 1.5
    with open(path, "w") as f:
        f.write("\t".join(HEADER) + "\n")
        for _, rid, ch, mux, st, ln in rows:
            tm = st + round(rng.uniform(0.05, 0.6), 4)
            vals = {"filename": "run_%d.fast5" % (ch % 4), "read_id": rid, "run_id": "r0", "channel": ch, "mux": mux,
                    "start_time": "%.4f" % st, "duration": "%.4f" % ln, "num_events": int(ln * 1800), "passes_filtering": "TRUE",
                    "template_start": "%.4f" % tm, "num_events_template": int(ln * 1700),
                    "template_duration": "%.4f" % (st + ln - tm), "sequence_length_template": int(ln * 420),
                    "mean_qscore_template": "9.5"}
            f.write("\t".join(str(vals[h]) for h in HEADER) + "\n")
    return rows


def make_paf(path, rows, seed):
    """UNCALLED PAF lines for the sequencing reads: ejected ones (ej, or ub as older versions wrote), kept ones."""
    rng = np.random.default_rng(seed)
    with open(path, "w") as f:
        f.write("# a comment line\n")
        for k, (prefix, rid, ch, mux, st, ln) in enumerate(rows):
            if prefix != "seq":
                continue
            qlen = int(rng.integers(200, 1800))
            tags = ["ch:i:%d" % ch, "st:i:%d" % int(st * 4000), "mt:f:%.6f" % rng.uniform(50, 500)]
            u = rng.uniform()
            if u < 0.4:
                tags.append("ej:f:%.6f" % rng.uniform(0.01, 0.3))
            elif u < 0.55:
                tags.append("ub:f:%.6f" % rng.uniform(0.01, 0.3))
            else:
                tags.append("kp:f:%.6f" % rng.uniform(0.01, 0.3))
            if rng.uniform() < 0.5:
                cols = [rid, str(qlen)] + ["*"] * 9 + ["255"]
            else:
                cols = [rid, str(qlen), "10", str(qlen), "+", "chr1", "100000", "500", "900", "300", "401", "255"]
            f.write("\t".join(cols + tags) + "\n")


class Recorder:
    def __init__(self):
        self.calls = []

    def _rec(self, *a):
        self.calls.append([a[0]] + [int(x) if isinstance(x, (int, np.integer)) else str(x) for x in a[1:]])

    def add_intv(self, ch, i, st, en):
        self._rec("add_intv", ch, i, st, en)

    def add_gap(self, ch, i, ln):
        self._rec("add_gap", ch, i, ln)

    def add_delay(self, ch, i, ln):
        self._rec("add_delay", ch, i, ln)

    def add_read(self, ch, rd, offs):
        self._rec("add_read", ch, rd, offs)


LOAD_SIM_CASES = {
    "defaults": {"sim_speed": 1.0, "scan_intv_time": 5400.0, "min_ch_reads": 10},
    "short_intervals": {"sim_speed": 0.5, "scan_intv_time": 150.0, "min_ch_reads": 3},
}


def make_fixtures():
    os.makedirs(OUT, exist_ok=True)
    unc_chans = [1, 2, 3, 5, 8, 13]
    unc = make_seqsum(os.path.join(OUT, "unc_seqsum.txt"), 7, unc_chans, {c: 1 + c % 4 for c in unc_chans}, (2, 5),
                      (300.0, 240.0))
    make_paf(os.path.join(OUT, "unc.paf"), unc, 8)
    ctl_chans = [1, 2, 3, 4, 5, 8, 13, 21]
    make_seqsum(os.path.join(OUT, "ctl_seqsum.txt"), 9, ctl_chans, {c: 1 + (c + 1) % 4 for c in ctl_chans}, (3,),
                (260.0, 200.0))


def reference_load_sim(ref):
    """The reference's sim_utils.load_sim, imported by path (its package __init__ needs the compiled module)."""
    pkg = types.ModuleType("uncalled")
    pkg.__path__ = []
    sys.modules["uncalled"] = pkg
    for name in ("pafstats", "sim_utils"):
        spec = importlib.util.spec_from_file_location("uncalled." + name, os.path.join(ref, "uncalled", name + ".py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules["uncalled." + name] = mod
        spec.loader.exec_module(mod)
        setattr(pkg, name, mod)
    return sys.modules["uncalled.sim_utils"].load_sim


def make_load_sim_golden(ref):
    load_sim = reference_load_sim(ref)
    gold = {}
    for key, prm in LOAD_SIM_CASES.items():
        conf = types.SimpleNamespace(unc_seqsum=os.path.join(OUT, "unc_seqsum.txt"), unc_paf=os.path.join(OUT, "unc.paf"),
                                     ctl_seqsum=os.path.join(OUT, "ctl_seqsum.txt"), **prm)
        rec = Recorder()
        load_sim(rec, conf)
        gold[key] = {"conf": prm, "calls": rec.calls}
    json.dump(gold, open(os.path.join(OUT, "load_sim_golden.json"), "w"), indent=0)


def client_script():
    """The ClientSim scenario.  4 channels, chunk_len 1000 samples, max_chunks 6, scan 2 s, eject time 0.1 s."""
    s = ["conf 4 4000 0.25 6 2.0 0.1"]
    # channel 1: active from the start with two gaps and two delays (both wrap); interval 1 starts late
    s += ["intv 1 0 0 60000", "gap 1 0 3000", "gap 1 0 5000", "delay 1 0 700", "delay 1 0 1300",
          "intv 1 1 2000 30000", "gap 1 1 4000"]
    # channel 2: two active stretches in interval 0; three gaps in interval 1
    s += ["intv 2 0 5000 20000", "intv 2 0 30000 50000", "gap 2 0 2500", "delay 2 0 1000",
          "intv 2 1 0 40000", "gap 2 1 1000", "gap 2 1 2000", "gap 2 1 3000", "delay 2 1 900"]
    # channel 3: an interval without gaps (it ends at its first read); channel 4: reads but no interval (dead)
    s += ["intv 3 0 0 40000", "intv 3 1 0 8000", "gap 3 1 1500"]
    reads = [(1, "r1a", 500, 101, 5500), (1, "r1b", 0, 102, 9000), (1, "r1c", 0, 103, None), (1, "r1d", 1200, 104, 3000),
             (2, "r2a", 0, 201, 4200), (2, "r2b", 300, 202, 6100), (2, "r2c", 0, 203, 2500),
             (3, "r3a", 0, 301, 7000), (3, "r3b", 250, 302, 3300), (4, "r4a", 0, 401, 5000)]
    s += ["read %d %s %d" % (ch, rid, offs) for ch, rid, offs, _, _ in reads]
    s += ["load %s %d %d" % (rid, num, n) for _, rid, _, num, n in reads if n is not None]   # r1c is missing
    s.append("run")
    events = {1100: ["unblock 1 101"], 2300: ["stop 2 201"], 3000: ["unblock 2 999"], 4100: ["unblock 1 102"],
              5200: ["unblock 2 202"], 6000: ["stop 1 104"], 7700: ["unblock 1 104", "unblock 1 101"],
              9100: ["unblock 3 301"], 10900: ["stop 2 203"], 13300: ["unblock 2 201"], 15800: ["unblock 1 101"],
              18800: ["unblock 2 202", "stop 1 102"], 21500: ["unblock 1 104"], 24000: ["unblock 2 203"]}
    for ms in range(0, 32000, 137):
        s.append("tick %d" % ms)
        for k in sorted(events):
            if ms <= k < ms + 137:
                s += events[k]
    return s


def make_client_golden(ref):
    here = os.path.join(ROOT, "tools", "sim_ref")
    lib = os.path.join(ROOT, "oracle", "_ref", "libuncalled_ref.so")
    if not os.path.exists(lib):
        raise SystemExit("build oracle/_ref first (make -C oracle ref)")
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "client_sim_driver")
        cmd = ["g++", "-std=c++11", "-O2", "-w", "-pthread", "-include", os.path.join(here, "fake_clock.hpp"),
               "-I" + os.path.join(here, "stubs"), "-I" + os.path.join(ROOT, "oracle", "ref_build", "stubs"),
               "-I" + os.path.join(ref, "src"), "-I" + os.path.join(ref, "submods"),
               "-I" + os.path.join(ref, "submods", "toml11"), "-I" + os.path.join(ref, "submods", "pdqsort"),
               os.path.join(here, "client_sim_driver.cpp"), os.path.join(ref, "src", "client_sim.cpp"),
               os.path.join(ref, "src", "fast5_reader.cpp"), lib, "-Wl,-rpath," + os.path.dirname(lib), "-o", exe]
        subprocess.run(cmd, check=True)
        script = client_script()
        res = subprocess.run([exe], input="\n".join(script) + "\n", capture_output=True, text=True, check=True)
    out = res.stdout.splitlines()
    json.dump({"script": script, "out": out}, open(os.path.join(OUT, "client_golden.json"), "w"), indent=0)
    print("client scenario: %d chunks, %d unblocks" % (sum(l.startswith("chunk") for l in out),
                                                       sum(l.startswith("unblock") for l in out)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    ap.add_argument("--emul", action="store_true", help="only write the emulated end-to-end golden")
    a = ap.parse_args()
    if a.emul:
        sys.path.insert(0, ROOT)
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        import test_sim
        test_sim.write_run_golden(os.path.join(OUT, "run_golden.json"))
        return
    make_fixtures()
    make_load_sim_golden(a.ref)
    make_client_golden(a.ref)


if __name__ == "__main__":
    main()
