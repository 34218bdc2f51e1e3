"""Writes tests/golden/dtw_align_golden.json from the reference's own dtw_test loop body (oracle/_ref ref_dtw_align): per
query the event and kept-mean counts, the target's bits, digests of the normalised means and of the span's k-mers, and for
aligned queries the score and mean score bits, the path length and the SHA-256 of the path's index columns.  Inputs: the
example read against the example index (tests/dtwalignlib.example_queries) and seeded reads of the multi-contig test
genome (synthetic_cases).  Every entry is checked against the C oracle before it is written.

    python tools/make_dtw_align_golden.py"""
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import dtwalignlib as D  # noqa: E402
import orclib  # noqa: E402


def main():
    d = tempfile.mkdtemp()
    out = {"example": {}, "synthetic": {}}
    ex = orclib.materialise_example_index(d)
    raw = np.load(os.path.join(ROOT, "tests", "golden", "example_read.npz"))["raw"]
    g = D.read_genome(ex)
    contig, (_, clen) = next(iter(g[1].items()))
    for name, rd_st, rd_en, rf_st, rf_en, fwd in D.example_queries(len(raw), clen):
        sig = raw[rd_st:(rd_en or len(raw))]
        want = D.ref_align(ex, sig, contig, rf_st, rf_en, fwd)
        got = D.oracle_align(g, sig, contig, rf_st, rf_en, fwd)
        assert D.public(want) == D.public(got), (name, D.public(want), D.public(got))
        out["example"][name] = D.public(want)
    prefix, codes = D.multi_contig_genome(d)
    g = D.read_genome(prefix)
    for name, sig, contig, rf_st, rf_en, fwd in D.synthetic_cases(codes):
        want = D.ref_align(prefix, sig, contig, rf_st, rf_en, fwd)
        got = D.oracle_align(g, sig, contig, rf_st, rf_en, fwd)
        assert D.public(want) == D.public(got), (name, D.public(want), D.public(got))
        out["synthetic"][name] = D.public(want)
    masked = sum(v["n_kept"] < v["n_events"] for v in out["synthetic"].values())
    assert masked >= 4, "the synthetic reads must exercise the mask"
    with open(D.GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", D.GOLDEN, len(out["example"]), "example and", len(out["synthetic"]), "synthetic queries;", masked, "masked")


if __name__ == "__main__":
    main()
