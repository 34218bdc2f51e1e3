"""Writes tests/golden/bwa_index_golden.json: what the reference's own BwaIndex<k5> (oracle/_ref/libref_bwa_index.so,
built by `make -C oracle -f bwa_index.mk`) computes on the fixtures of tests/bwaindexlib.py, and checks the C
restatement (oracle/unc_oracle_bwa_index.c) against it before writing.

Per fixture: sa of every row and get_neighbor of every row x 4 bases with start 0, start size() + 1 and inverted ranges
(as digests), range_to_fms over the spans of bwaindexlib.spans (digest of both lists), get_kmers with kmers_revcomp over
bwaindexlib.kmer_spans, and translate_loc at contig edges (values).  Plus the k = 5 helpers of bp.hpp for all 1024
k-mers (digest).

    python tools/make_bwa_index_golden.py
"""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import bwaindexlib as B  # noqa: E402
from orclib import digest  # noqa: E402


def main():
    if not B.Ref.available():
        raise SystemExit("oracle/_ref/libref_bwa_index.so is not built (make -C oracle -f bwa_index.mk)")
    out = {"fixtures": {}}
    d = tempfile.mkdtemp(prefix="bwa_index_golden_")
    for name in B.FIXTURES:
        os.makedirs(os.path.join(d, name))
        prefix = B.build(name, os.path.join(d, name))
        rec = B.golden_record(prefix, B.Ref(prefix))
        mine = B.golden_record(prefix, B.Restated(prefix))
        for k in ("size", "sa", "neighbor", "fms"):
            assert mine[k] == rec[k], (name, k, "the C restatement differs from the reference")
        out["fixtures"][name] = rec
        print(name, "size", rec["size"], "spans", len(rec["fms"]), flush=True)
    h = B.Ref.kmer_helpers()
    out["kmer_helpers"] = digest(*(h[k] for k in sorted(h)))
    with open(B.GOLDEN, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
    print("wrote", B.GOLDEN)


if __name__ == "__main__":
    main()
