"""Debug: per-phase cycle breakdown of the mapper kernel (needs the -DUNC_PHASE_TIMING build
uncalled_b200/libunc_b200_pt.so; see DESIGN.md 'measurement')."""
import ctypes as C, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import uncalled_b200._native as N
N.LIB_PATH = sys.argv[3] if len(sys.argv) > 3 else os.path.join(ROOT, "uncalled_b200", "libunc_b200_pt.so")
import uncalled_b200 as U
import synth, synthdata
name = sys.argv[1] if len(sys.argv) > 1 else "g4m7"
n_reads = int(sys.argv[2]) if len(sys.argv) > 2 else 2368
prefix, g = synthdata.get_index(name)
sig, truth = synth.reads(g, n_reads, 4000, seed=7)
idx = U.Index(prefix, device=0)
bm = U.BatchMapper(idx, max_reads=n_reads, max_samples=n_reads * 4000)
d = U.make_descs([4000] * n_reads)
for it in range(2):
    out = bm.map(sig.ravel(), d)
    print("iter", it, bm.timing())
ph2 = np.zeros((n_reads, 64), np.uint64)
L = N.lib()
L.unc_pool_debug_phases.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
N.check(L.unc_pool_debug_phases(bm.h, n_reads, ph2.ctypes.data))
names = ["A probs + counter reset", "B extension", "C1 scatter into k-mer buckets", "C2 bucket sort + count", "(unused)", "D1 dedup/sources/seeds + E fresh",
         "X barrier wait (slowest warp of D1/E, tracker)", "head: event load + scaling", "head: verdict + bookkeeping", "head: loop back-edge",
         "B2 chunk scan / ended rows / bucket offsets / deferred seed_prob", "D0 bucket prefix + flags + fresh plan | S1 SA of ended rows",
         "cut-case recount", "", "", "",
         "  wait at the barrier after A", "  wait after B", "  wait after C1", "  wait after C2", "", "", "", "", "", "", "  wait after B2", "  wait after D0", "", "", "", ""]
ev = out["events_used"].astype(np.float64) + 1
for title, ph in (("worker warp 0, thread 0 (also runs the single-warp sections)", ph2[:, :32]),
                  ("last worker warp, lane 0 (its barrier waits expose the single-warp sections)", ph2[:, 32:64])):
    tot = ph.sum(axis=0).astype(np.float64)
    per_warp = tot.copy()
    tot[[13, 14, 15, 20, 21, 22, 23, 24, 25]] = 0      # not intervals: the worker warps' own times (slowest / mean), below
    ph = ph.copy(); ph[:, [13, 14, 15, 20, 21, 22, 23, 24, 25]] = 0
    if title.startswith("last"):
        ph[:, 28:32] = 0; tot[28:32] = 0           # the tracker's counters
    print("--", title)
    print("total events", ev.sum())
    for i, nm in enumerate(names):
        if not nm or i >= ph.shape[1]:
            continue
        print("%-36s %6.1f%%  %8.0f cycles/event" % (nm, 100 * tot[i] / max(tot.sum(), 1), tot[i] / ev.sum()))
    print("cycles/event total %.0f" % (tot.sum() / ev.sum()))
    if title.startswith("worker"):
        print("   event barrier: now - release stamp of the last-released worker warp %.0f, of the first-released %.0f" % (per_warp[13] / ev.sum(), per_warp[14] / ev.sum()))
        for nm, a, b in (("C2 sort + count", 15, 20), ("D1 emit", 21, 22)):
            print("   %-18s slowest worker warp %8.0f cycles/event, mean warp %8.0f" % (nm, per_warp[a] / ev.sum(), per_warp[b] / ev.sum()))
        print("   event barrier: released %.0f cycles after the last worker warp arrived, %.0f after the first, %.0f after the tracker warp" % (per_warp[23] / ev.sum(), per_warp[24] / ev.sum(), per_warp[25] / ev.sum()))
    if ph.shape[1] >= 32 and title.startswith("last"):
        t = ph2[:, 60:64].astype(np.float64)
        ns = max(t[:, 3].sum(), 1)
        print("tracker warp: %.1f seeds/event; cycles per seed: search %.0f, scan %.0f, update/insert %.0f" % (t[:, 3].sum() / ev.sum(), t[:, 0].sum() / ns, t[:, 1].sum() / ns, t[:, 2].sum() / ns))
    nm_ = out["mapped"] == 0
    print("non-mapping reads: cycles/event %.0f ; mapping: %.0f" % (ph[nm_].sum() / ev[nm_].sum(), ph[~nm_].sum() / ev[~nm_].sum()))
