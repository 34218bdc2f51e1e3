"""`mask-internal`: iterative masking of the most frequent k-mer (masking/mask_internal.sh + mask_kmers.py).

CPU: the numpy oracle (tests/masklib.py) against the digests of the reference's own pipeline
(tests/golden/mask_golden.json, tools/make_mask_golden.py); the device source under the warp emulator against the
oracle at two tile sizes; the tie rule; rejected inputs.  GPU: the library against the golden data and the oracle,
a 20 Mb genome, early stop, and `mask-internal` -> `index` -> `map` end to end."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

import masklib as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(M.GOLDEN))["cases"]


def _want(case):
    return [(s["kmer"], s["count"]) for s in case["steps"]]


def _write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


def boundary_fasta(seed=3):
    """records whose separators and planted k-mers sit on, just before and just after the edges of 1024- and
    2048-position tiles and inside the 32-byte halo; overlapping occurrences (tandem copies) included"""
    rng = np.random.default_rng(seed)
    unit = b"GATTACAGTC"
    s = bytearray(b"ACGT"[i] for i in rng.integers(0, 4, 9000))
    for edge in (1024, 2048, 3072, 4096, 6144):
        for d in (-11, -10, -9, -5, -1, 0, 1, 7, 21, 30, 31, 33):
            p = edge + d
            s[p:p + len(unit)] = unit
    s[5000:5000 + 40] = unit[:4] * 10                                      # overlapping occurrences of GATT / ATTG..
    cuts = [1023, 2047, 2048 + 700, 4095, 6143 - 3]                       # positions of record separators
    recs, a = [], 0
    for c in cuts + [len(s)]:
        recs.append(bytes(s[a:c]))
        a = c + 1                                                          # the separator occupies one position
    return b"".join(b">r%d\n" % i + r + b"\n" for i, r in enumerate(recs))


# ---------------------------------------------------------------- CPU

@pytest.mark.parametrize("key", sorted(GOLD))
def test_oracle_matches_the_reference_pipeline(key):
    case = GOLD[key]
    data = M.fixture(case["fixture"])
    assert M.sha256(data) == case["input_sha256"]
    for it in sorted({1, case["iters"]}):
        out, log = M.oracle(data, case["k"], it)
        want = _want(case)[:it]
        assert log == want
        if want:
            assert M.sha256(out) == case["steps"][len(want) - 1]["sha256"]


def test_oracle_quirks():
    # case-insensitive counting, non-ACGT bytes and record ends break k-mers, other bytes kept, CRLF normalised
    data = b">a x \r\nacGTN\r\nAC  gt\r\n>b\r\nAC\r\n"
    out, log = M.oracle(data, 2, 1)
    assert log == [("AC", 3)]
    assert out == b">a x\nNNGTNNN  gt\n>b\nNN\n"
    out, log = M.oracle(b">a\nAAAA\n", 2, 3)                               # overlapping occurrences all masked
    assert log == [("AA", 3)] and out == b">a\nNNNN\n"


@pytest.mark.parametrize("n_threads", [32, 64])
@pytest.mark.parametrize("key", ["repeats_k5_i1", "mixed_k5_i5", "mixed_k13_i5", "crlf_k3_i5", "crlf_k13_i1",
                                 "polya_k13_i5", "polya_k1_i1", "tiny_k1_i30", "tiny_k3_i30"])
def test_emulated_device_source_matches_golden(key, n_threads, tmp_path):
    case = GOLD[key]
    fa = _write(tmp_path, "in.fa", M.fixture(case["fixture"]))
    out = str(tmp_path / "out.fa")
    rc, log = M.emu_mask_internal(fa, out, case["k"], case["iters"], n_threads)
    assert rc == 0 and log == _want(case)
    assert M.sha256(open(out, "rb").read()) == case["steps"][-1]["sha256"]


@pytest.mark.parametrize("n_threads", [32, 64])
@pytest.mark.parametrize("k,iters", [(10, 8), (4, 6), (13, 3), (1, 2)])
def test_emulated_tile_edges_and_halo(k, iters, n_threads, tmp_path):
    data = boundary_fasta()
    fa = _write(tmp_path, "in.fa", data)
    out = str(tmp_path / "out.fa")
    rc, log = M.emu_mask_internal(fa, out, k, iters, n_threads)
    want_out, want_log = M.oracle(data, k, iters)
    assert rc == 0 and log == want_log
    assert open(out, "rb").read() == want_out
    if k == 10:
        assert want_log[0][0] == "GATTACAGTC"                             # the planted copies are masked first


def test_ties_choose_the_smallest_code(tmp_path):
    for data, want in ((b">a\nTTGGCCAA\n>b\nCATG\n", [("CA", 2), ("TG", 2)]),      # CA and TG twice: CA < TG
                       (b">a\nTTGGCCAA\n", [("AA", 1), ("CC", 1)])):                  # every 2-mer once
        assert M.oracle(data, 2, 2)[1] == want
        fa = _write(tmp_path, "in.fa", data)
        for nt in (32, 64):
            rc, log = M.emu_mask_internal(fa, str(tmp_path / "out.fa"), 2, 2, nt)
            assert rc == 0 and log == want
    assert GOLD["tiny_k3_i30"]["steps"][0]["kmer"] == "AAC"                  # every 3-mer once: the smallest


def _native_call(fasta, out, k, iters):
    import uncalled_b200._native as N
    codes, counts, done = np.zeros(max(iters, 1), np.uint64), np.zeros(max(iters, 1), np.uint64), C.c_uint32()
    rc = N.lib().unc_mask_internal(fasta.encode(), out.encode(), k, iters, codes.ctypes.data, counts.ctypes.data,
                                   C.byref(done))
    return rc, N.lib().unc_last_error().decode()


@pytest.mark.parametrize("what,data,k,iters", [
    ("k0", b">a\nACGT\n", 0, 1),
    ("k14", b">a\nACGT\n", 14, 1),
    ("iters0", b">a\nACGT\n", 3, 0),
    ("empty", b"", 3, 1),
    ("no_header", b"ACGT\n>a\nACGT\n", 3, 1),
    ("blank_first_line", b"\n>a\nACGT\n", 3, 1),
    ("record_without_sequence", b">a\n>b\nACGT\n", 3, 1),
    ("last_record_without_sequence", b">a\nACGT\n>b\n  \n", 3, 1),
])
def test_rejected_inputs(what, data, k, iters, tmp_path):
    import uncalled_b200._native as N
    fa = _write(tmp_path, "in.fa", data)
    out = str(tmp_path / "out.fa")
    rc, msg = _native_call(fa, out, k, iters)
    assert rc == -1, (what, rc, msg)                                      # UNC_E_ARG
    assert msg and not os.path.exists(out)
    assert M.emu_mask_internal(fa, out, k, iters, 32)[0] == -1
    with pytest.raises(N.UncError, match="bad argument"):
        import uncalled_b200 as U
        U.mask_internal(fa, k, iters, str(tmp_path / "x_"), log=None)
    assert not os.path.exists(str(tmp_path / ("x_mask%d.fa" % iters)))


def test_missing_file_is_an_io_error(tmp_path):
    rc, msg = _native_call(str(tmp_path / "nope.fa"), str(tmp_path / "out.fa"), 3, 1)
    assert rc == -2 and "nope.fa" in msg


def test_fails_loudly_without_a_gpu(tmp_path):
    """No CPU path: a valid call without a CUDA device reports UNC_E_NO_DEVICE and writes nothing."""
    import uncalled_b200._native as N
    if N.lib().unc_device_count() > 0:
        pytest.skip("a CUDA device is present")
    fa = _write(tmp_path, "in.fa", M.fixture("repeats"))
    assert _native_call(fa, str(tmp_path / "out.fa"), 10, 3)[0] == -4
    assert not os.path.exists(str(tmp_path / "out.fa"))


# ---------------------------------------------------------------- GPU

@pytest.mark.gpu
@pytest.mark.parametrize("key", sorted(GOLD))
def test_gpu_matches_golden_and_oracle(key, tmp_path, capsys):
    import uncalled_b200 as U
    case = GOLD[key]
    data = M.fixture(case["fixture"])
    fa = _write(tmp_path, "in.fa", data)
    prefix = str(tmp_path / "o_")
    log = U.mask_internal(fa, case["k"], case["iters"], prefix)
    assert log == _want(case)
    got = open(prefix + "mask%d.fa" % case["iters"], "rb").read()
    assert M.sha256(got) == case["steps"][-1]["sha256"]
    assert got == M.oracle(data, case["k"], case["iters"])[0]
    err = capsys.readouterr().err
    assert err == "".join("Iteration %d: masked %d occurences of %s\n" % (i, n, km) for i, (km, n) in enumerate(log))


@pytest.mark.gpu
def test_gpu_20mb_k10_30_iterations(tmp_path):
    import uncalled_b200 as U
    data = M.big_genome(20_000_000, seed=7)
    fa = _write(tmp_path, "g20m.fa", data)
    prefix = str(tmp_path / "g_")
    log = U.mask_internal(fa, 10, 30, prefix, log=None)
    want_out, want_log = M.oracle(data, 10, 30)
    assert log == want_log and len(log) == 30
    assert open(prefix + "mask30.fa", "rb").read() == want_out


@pytest.mark.gpu
def test_gpu_k13_and_tile_edges(tmp_path):
    import uncalled_b200 as U
    for data, k, iters in ((boundary_fasta(), 13, 4), (boundary_fasta(), 10, 8), (M.big_genome(300_000, seed=2), 13, 5)):
        fa = _write(tmp_path, "in.fa", data)
        log = U.mask_internal(fa, k, iters, str(tmp_path / "o_"), log=None)
        want_out, want_log = M.oracle(data, k, iters)
        assert log == want_log
        assert open(str(tmp_path / ("o_mask%d.fa" % iters)), "rb").read() == want_out


@pytest.mark.gpu
def test_gpu_early_stop(tmp_path, capsys):
    from uncalled_b200 import cli
    fa = _write(tmp_path, "tiny.fa", b">t1\nACGTTTAC\n>t2\nGGGAAC\n")
    assert cli.main(["mask-internal", fa, "1", "30", str(tmp_path / "t_")]) == 0
    err = capsys.readouterr().err
    assert re.findall(r"Iteration (\d+): masked (\d+) occurences of ([ACGT]+)\n", err) == \
        [("0", "4", "A"), ("1", "4", "G"), ("2", "3", "C"), ("3", "3", "T")]
    assert "No k-mer left to mask after 4 iterations" in err
    assert open(str(tmp_path / "t_mask30.fa"), "rb").read() == b">t1\nNNNNNNNN\n>t2\nNNNNNN\n"


@pytest.mark.gpu
def test_gpu_mask_then_index_then_map(tmp_path, capsys):
    """`mask-internal` on the example reference, `index` of its output, `map` of the example read: valid PAF"""
    import orclib
    from uncalled_b200 import cli
    os.makedirs(tmp_path / "src")
    src = orclib.materialise_example_index(str(tmp_path / "src"))
    fa = _write(tmp_path, "ref.fa", open(src + ".fa", "rb").read())
    assert cli.main(["mask-internal", fa, "10", "5", str(tmp_path / "ref_")]) == 0
    masked = str(tmp_path / "ref_mask5.fa")
    assert open(masked, "rb").read() == M.oracle(open(fa, "rb").read(), 10, 5)[0]
    assert cli.main(["index", masked]) == 0
    capsys.readouterr()
    assert cli.main(["map", masked, os.path.join(ROOT, "tests", "golden", "fast5", "example_single.fast5")]) == 0
    lines = capsys.readouterr().out.strip().split("\n")
    assert len(lines) == 1
    f = lines[0].split("\t")
    assert len(f) >= 12 and f[4] in "+-*"
    if f[4] != "*":
        assert int(f[6]) > 0 and 0 <= int(f[7]) <= int(f[8]) <= int(f[6])
