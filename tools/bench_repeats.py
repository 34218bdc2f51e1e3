"""`find-repeats` on the GPU: the repeat length of every reference position (unc_repeats_lengths, k_repeat_lengths).

Genomes, each indexed on the device (unc_index_build_device) in a temporary directory:
  g4m7     4.7 Mb of seeded random sequence (the size of an E. coli genome);
  fam4m7   4.7 Mb with planted repeat families (repeatslib.family_genome: 300-base and 6 kb elements, a 20 kb segmental
           duplication, a 171-base tandem array), so that the walks are not only those of random sequence;
  chr1     230 Mb with 230 masked N runs of 5 kb (BASELINE.json config 4, tools/bench_chr1.py's genome).
Per genome: the whole-genome kernel time (CUDA events, summed over windows, after one warm-up pass), positions/s, steps/s
(sum of L + 1 over all positions, from the output), how the kernel time splits between windows whose longest walk is
above 1000 steps and the rest (at 2^18-position windows), and the end-to-end wall time of `find-repeats <prefix> 30
--bed`.  Beside them, the reference's own self_align at sample_dist 1 from oracle/_ref (single-threaded, as
find_repeats.cpp is) on g4m7, when oracle/_ref was built.  The card's name and power limit are read in the same run.

    python tools/bench_repeats.py [--genomes g4m7,fam4m7,chr1] [--out result.json]
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

SPLIT_WINDOW = 1 << 18
LONG = 1000


def genome(name):
    """(ACGT-or-N codes, record names)"""
    import repeatslib as R
    from bench_chr1 import make_genome
    if name == "g4m7":
        return np.random.default_rng(4700).integers(0, 4, 4_700_000, dtype=np.uint8), ["g4m7"]
    if name == "fam4m7":
        return R.family_genome(4_700_000, 4701, families=((300, 600), (6000, 40)), dup=20000, tandem=200), ["famA", "famB"]
    if name == "chr1":
        return make_genome(230_000_000, 4242, n_runs=230, run_len=5000)[1], ["synthetic_chr1"]
    raise SystemExit("unknown genome " + name)


def sweep(finder, window):
    """one pass over the reference in windows: (kernel ms per window, sum of L + 1 per window, max L per window)"""
    L = finder._L
    buf = np.empty(window, np.uint32)
    ms, steps, longest = [], [], []
    t = C.c_float()
    for o in range(0, finder.l_pac, window):
        k = min(window, finder.l_pac - o)
        rc = L.unc_repeats_lengths(finder._h, o, k, buf.ctypes.data)
        if rc:
            raise RuntimeError(L.unc_last_error().decode())
        L.unc_repeats_last_kernel_ms(finder._h, C.byref(t))
        ms.append(t.value)
        steps.append(int(buf[:k].astype(np.int64).sum()) + k)
        longest.append(int(buf[:k].max()))
    return np.array(ms), np.array(steps), np.array(longest)


def ref_self_align_seconds(prefix):
    """the reference's own self_align at sample_dist 1 in a child process (oracle/_ref holds one static index)"""
    import orclib
    if not orclib.ref_available():
        return None
    code = ("import sys, time; sys.path[:0] = [%r]; import orclib\n"
            "t = time.time(); orclib.ref_self_align(%r, 1); print('SECONDS', time.time() - t)") % (
        os.path.join(ROOT, "tests"), prefix)
    out = orclib.run_in_subprocess(code, timeout=3600)
    return float(out.split("SECONDS")[1].split()[0])


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genomes", default="g4m7,fam4m7,chr1")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import repeatslib as R
    import uncalled_b200 as U
    from uncalled_b200 import _native as N
    L = N.lib()
    N.check(L.unc_init(0))
    res = {"card": card(), "genomes": {}}
    work = tempfile.mkdtemp(prefix="bench_repeats_")
    try:
        for name in args.genomes.split(","):
            codes, names = genome(name)
            fa, prefix = os.path.join(work, name + ".fa"), os.path.join(work, name)
            R.write_fasta(fa, codes, names)
            del codes
            t = time.time()
            N.check(L.unc_index_build_device(fa.encode(), prefix.encode()))
            r = {"index_build_s": time.time() - t}
            os.remove(fa)
            with U.RepeatFinder(prefix) as f:
                sweep(f, f.window)                                        # warm-up
                ms, steps, _ = sweep(f, f.window)
                sms, ssteps, slong = sweep(f, SPLIT_WINDOW)
                n = f.l_pac
            total_steps = int(steps.sum())
            assert total_steps == int(ssteps.sum())
            long_w = slong > LONG
            r.update(positions=n, kernel_ms=float(ms.sum()), positions_per_s=n / (ms.sum() / 1e3),
                     steps=total_steps, steps_per_s=total_steps / (ms.sum() / 1e3),
                     split_windows=int(len(sms)), split_kernel_ms=float(sms.sum()),
                     long_windows=int(long_w.sum()), long_window_time_share=float(sms[long_w].sum() / sms.sum()),
                     long_window_step_share=float(ssteps[long_w].sum() / ssteps.sum()), max_L=int(slong.max()))
            t = time.time()
            with open(os.devnull, "w") as dn:
                subprocess.run([sys.executable, "-m", "uncalled_b200", "find-repeats", prefix, "30", "--bed"], stdout=dn,
                               check=True, cwd=ROOT)
            r["cli_bed_min_k30_wall_s"] = time.time() - t
            if name == "g4m7":
                r["reference_self_align_sd1_s"] = ref_self_align_seconds(prefix)
            res["genomes"][name] = r
            print(name, json.dumps(r), flush=True)
            for e in (".bwt", ".sa", ".pac", ".ann", ".amb"):
                os.remove(prefix + e)
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
