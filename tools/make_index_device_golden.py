"""Writes tests/golden/index_build_device_golden.json: the SHA-256 of the five files that bwa itself (oracle/_ref's
ref_index_build, the reference's BwaIndex::create -> bwa_idx_build, `bwtsw` at this size) writes for the seeded
1.1 Gbp genome of tests/indexlib.py (2.2e9 FM rows, above 2^31).  The host builder cannot index a text this long,
so bwa is the only reference for the device builder there.

    python tools/make_index_device_golden.py [work_dir]

A long CPU job: bwa's bwtsw on one thread took 1385 s on an 8-CPU development box (the FASTA, 1.1 GB, is made in 15 s)."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import indexlib as I  # noqa: E402


def sha256_file(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 24), b""):
            h.update(blk)
    return h.hexdigest()


def main():
    work = sys.argv[1] if len(sys.argv) > 1 else tempfile.mkdtemp()
    os.makedirs(work, exist_ok=True)
    fa, prefix = os.path.join(work, "big.fa"), os.path.join(work, "big")
    t = time.time()
    data = I.big_fasta()
    with open(fa, "wb") as f:
        f.write(data)
    gold = {"genome": I.BIG_SPEC, "fasta_sha256": hashlib.sha256(data).hexdigest(), "fasta_bytes": len(data)}
    del data
    print("fasta written in %.1f s" % (time.time() - t), flush=True)
    t = time.time()
    code = "import sys; sys.path.insert(0, %r); import orclib; orclib.ref().ref_index_build(%r, %r)" % (
        os.path.join(ROOT, "tests"), fa.encode(), prefix.encode())
    subprocess.run([sys.executable, "-c", code], check=True)
    print("bwa_idx_build in %.1f s" % (time.time() - t), flush=True)
    gold["files"] = {ext: sha256_file(prefix + "." + ext) for ext in I.EXTS}
    with open(I.BIG_GOLDEN, "w") as f:
        json.dump(gold, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(gold, indent=1))


if __name__ == "__main__":
    main()
