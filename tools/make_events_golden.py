"""Writes tests/golden/events_golden.json from the reference's own classes (oracle/_ref/libref_events.so: EventDetector,
EventProfiler, Normalizer), for the checkers of `events`.

Reads: the golden example read (tests/golden/example_read.npz) and seeded synthetic reads (tests/eventslib.py), among
them a stall and reads with events outside min_mean / max_mean.  Per read: the event count, mean_event_len as a float32
bit pattern, the first events in full, and a SHA-256 of every per-event column (little-endian bytes; win_mask as u8).
The reference's scale and shift stay inside its Normalizer; the normalised means carry them.

    python tools/make_events_golden.py        # needs oracle/_ref (built by __graft_entry__.build())
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools"), ROOT]

import eventslib as E  # noqa: E402

N_FULL = 12


def golden_reads():
    """{name: float32 pA signal}: the inputs the golden file covers, regenerated the same way by the tests"""
    g = np.load(os.path.join(ROOT, "tests", "golden", "example_read.npz"))
    out = {"example_read": np.asarray(g["raw"], np.float32)}
    for i, s in enumerate(E.synth_reads(101, 4)):
        out["synth_%d" % i] = s
    edges = E.edge_reads(29)
    for k in ("stall", "out_of_range", "few_events", "short_13", "empty"):
        out["edge_" + k] = edges[k]
    return out


def bits(x):
    return int(np.float32(x).view(np.uint32))


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def summarise(res):
    rd, ev = res
    out = {"n_events": int(rd["n_events"]), "mean_event_len": bits(rd["mean_event_len"]),
           "digest": {k: digest(np.asarray(ev[k], np.uint8 if k == "win_mask" else (np.uint32 if k == "start" else np.float32)))
                      for k in E.FIELDS},
           "first": {k: [int(v) if k in ("start", "win_mask") else bits(v) for v in ev[k][:N_FULL]] for k in E.FIELDS}}
    return out


def main():
    if not E.ref_available():
        sys.exit("oracle/_ref/libref_events.so is missing: build it first (make -C oracle -f events.mk)")
    doc = {"about": "events of the reference's own EventDetector / EventProfiler / Normalizer (tools/make_events_golden.py)",
           "reads": {name: summarise(E.ref_read(sig)) for name, sig in golden_reads().items()}}
    path = os.path.join(ROOT, "tests", "golden", "events_golden.json")
    with open(path, "w") as f:
        json.dump(doc, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", path, len(doc["reads"]), "reads")


if __name__ == "__main__":
    main()
