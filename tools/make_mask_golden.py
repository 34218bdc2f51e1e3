"""Writes tests/golden/mask_golden.json: for every `mask-internal` case of tests/masklib.py, the k-mer of each
iteration and the SHA-256 of the FASTA after it, as the reference's own pipeline produces them.

    python tools/make_mask_golden.py <UNCALLED source tree>

Each iteration's k-mer is chosen by brute-force counting (a dict over every window; ties to the smallest code, since
jellyfish's own choice is its hash order), and the masking is done by the reference's masking/mask_kmers.py itself,
run on the previous iteration's output as masking/mask_internal.sh runs it.  Its unused matplotlib import is served
by an empty stub module.  The loop stops where no k-mer is left, where the shell script would call mask_kmers.py
with an empty k-mer."""
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import masklib as M  # noqa: E402


def stub_matplotlib(d):
    os.makedirs(os.path.join(d, "matplotlib"))
    open(os.path.join(d, "matplotlib", "__init__.py"), "w").close()
    open(os.path.join(d, "matplotlib", "pyplot.py"), "w").close()


def run_case(script, stub, data, k, iters, work):
    steps = []
    cur = os.path.join(work, "mask0.fa")
    open(cur, "wb").write(data)
    for i in range(iters):
        choice = M.brute_force_choice(open(cur, "rb").read(), k)
        if choice is None:
            break
        kmer, count = choice
        nxt = os.path.join(work, "mask%d.fa" % (i + 1))
        with open(nxt, "wb") as out:
            r = subprocess.run([sys.executable, script, cur, "-k", kmer], stdout=out, stderr=subprocess.PIPE,
                               env=dict(os.environ, PYTHONPATH=stub), check=True)
        log = r.stderr.decode()
        m = re.fullmatch(r"masked (\d+) occurences of ([ACGT]+)\n", log)
        assert m and int(m.group(1)) == count and m.group(2) == kmer, (log, kmer, count)
        steps.append({"kmer": kmer, "count": count, "sha256": M.sha256(open(nxt, "rb").read())})
        cur = nxt
    return steps


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    script = os.path.join(sys.argv[1], "masking", "mask_kmers.py")
    assert os.path.isfile(script), script
    gold = {"tie_rule": "smallest 2-bit code", "cases": {}}
    with tempfile.TemporaryDirectory() as tmp:
        stub = os.path.join(tmp, "stub")
        stub_matplotlib(stub)
        for name, k, iters in M.CASES:
            data = M.fixture(name)
            work = tempfile.mkdtemp(dir=tmp)
            key = "%s_k%d_i%d" % (name, k, iters)
            gold["cases"][key] = {"fixture": name, "k": k, "iters": iters, "input_sha256": M.sha256(data),
                                  "steps": run_case(script, stub, data, k, iters, work)}
            print(key, len(gold["cases"][key]["steps"]), "iterations")
    with open(M.GOLDEN, "w") as f:
        json.dump(gold, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
