"""CPU tier of `find-repeats`: the device function (unc_repeat_length in unc_selfalign.cuh) under the emulator, against
L derived from the reference's own self_align at sample_dist 1 (live where oracle/_ref is built, else through stored
digests), against the oracle's orc_repeat_lengths, and against the definition counted in numpy; window independence;
`RepeatFinder` and the `find-repeats` command end to end with the C-ABI replaced by the emulator; the C-ABI's argument
and no-device errors.  tests/test_z_gpu_repeats.py runs the same comparisons through unc_repeats_lengths on the GPU."""
import ctypes as C
import os

import numpy as np
import pytest

import fmsteplib as F
import orclib
import repeatslib as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = sorted(F.FIXTURES)


@pytest.fixture(scope="module")
def work(tmp_path_factory):
    return tmp_path_factory.mktemp("repeats")


@pytest.fixture(scope="module")
def small(work):
    return {name: F.build(name, work) for name in SMALL}


@pytest.fixture(scope="module")
def example(work):
    return orclib.materialise_example_index(str(work))


@pytest.fixture(scope="module")
def multi(work):
    """three contigs with planted repeats, palindromes and a repeat across a contig end"""
    fa = str(work / "multi.fa")
    R.genome_fasta(fa, 11)
    return R.build(fa, str(work / "multi"))


@pytest.fixture(scope="module")
def multi_n(work):
    """contigs with N runs (.amb holes), one of them at a contig's start and one at its end"""
    rng = np.random.default_rng(12)
    seqs = []
    for k in range(3):
        s = bytearray(b"".join(b"ACGT"[v:v + 1] for v in rng.integers(0, 4, 500 + 60 * k)))
        s[100:130] = b"N" * 30
        if k == 1:
            s[:7] = b"N" * 7
        if k == 2:
            s[-9:] = b"N" * 9
        seqs.append(bytes(s))
    fa = str(work / "holes.fa")
    with open(fa, "wb") as f:
        for k, s in enumerate(seqs):
            f.write(b">h%d\n%s\n" % (k, s))
    return R.build(fa, str(work / "holes"))


LIVE = r"""
import sys
sys.path[:0] = [%r]
import numpy as np, orclib, repeatslib as R
for prefix in %r:
    off, val = orclib.ref_self_align(prefix, 1)
    L = R.from_self_align(off, val, R.remaining(prefix))
    print("REF", prefix, orclib.digest(L))
"""


def _ref_digests(prefixes):
    """{prefix: digest of L from the reference's own self_align}, computed in a child (oracle/_ref's index is static)"""
    out = orclib.run_in_subprocess(LIVE % (os.path.join(ROOT, "tests"), list(prefixes)), timeout=1800)
    return {ln.split()[1]: ln.split()[2] for ln in out.splitlines() if ln.startswith("REF ")}


def _against_reference(key, prefixes):
    """emulated L == oracle L == L from the oracle's self_align at every position; and == L from the reference's own
    self_align (live where oracle/_ref is built; through digests stored under `key` otherwise)"""
    got = []
    for p in prefixes:
        emu = R.repeat_lengths(p, 0, R.layout(p)[0])
        orc = R.oracle_lengths(p)
        off, val = orclib.self_align(p, 1)
        via_sa = R.from_self_align(off, val, R.remaining(p))
        assert np.array_equal(emu, orc), (p, np.flatnonzero(emu != orc)[:5])
        assert np.array_equal(orc, via_sa), (p, np.flatnonzero(orc != via_sa)[:5])
        got.append(emu)
    live = orclib.ref_available()
    if live:
        ref = _ref_digests(prefixes)
        for p, L in zip(prefixes, got):
            assert ref[p] == orclib.digest(L), p
    R.expect_reference(key, tuple(got), live=live)


def test_example_index_against_reference(example):
    _against_reference("find_repeats/example", [example])


def test_small_indexes_against_reference(small):
    _against_reference("find_repeats/fm_step_fixtures", [small[n] for n in SMALL])


def test_multi_contig_against_reference(multi, multi_n):
    _against_reference("find_repeats/multi_contig", [multi, multi_n])


def test_self_align_relation(multi, multi_n, small, example):
    """the relation from_self_align relies on, checked path by path on the oracle's self_align: a path has L + 1
    lengths, or L when its walk ended on an empty range (its last length > 1 and fewer than lim - p lengths).  bwa builds
    the BWT from the .pac it writes, random bases of the N runs included, so a walk along the .pac never empties its
    range: on these indexes, holes included, every path has L + 1 lengths"""
    for p in [multi, multi_n, example] + [small[n] for n in ("multi_n", "poly", "palindrome", "tiny1", "tiny2")]:
        off, val = orclib.self_align(p, 1)
        off = off.astype(np.int64)
        L = R.oracle_lengths(p).astype(np.int64)
        cnt = np.diff(off)
        rem = R.remaining(p)
        last = val.astype(np.int64)[off[1:] - 1]
        assert np.array_equal(cnt, L + 1), p
        assert ((last <= 1) | (cnt == rem)).all(), p        # the walk stops on a unique range or at the contig end
        assert (val > 0).all() and (np.minimum.reduceat(val.astype(np.int64), off[:-1]) == last).all()
        assert np.array_equal(R.from_self_align(off, val, rem), L.astype(np.uint32))


@pytest.mark.parametrize("seed", [11, 21, 31])
def test_meaning_brute_force(work, seed):
    """L(p) is the least t >= 1 for which the t + 1 bases from p occur at most once in forward + reverse complement,
    capped by the contig end; the walk's first range also holds row L2[c] (the get_base_range quirk), which can add one
    occurrence: the brute force counts it and its effect is shown to occur"""
    fa = str(work / ("bf%d.fa" % seed))
    R.genome_fasta(fa, seed)
    p = R.build(fa, str(work / ("bf%d" % seed)))
    emu = R.repeat_lengths(p, 0, R.layout(p)[0])
    assert np.array_equal(emu, R.brute_lengths(p, quirk=True))
    plain = R.brute_lengths(p, quirk=False)
    assert (emu >= plain).all()
    # planted repeats: the palindrome, the copies and the text across the end of contig 0 give long walks
    _, contigs, _ = R.layout(p)
    o1, o2 = contigs[1][1], contigs[2][1]
    assert emu[100] >= 59 and emu[o1 + 50] >= 59 and emu[o1 + 300] >= 59      # the 60-base unit, forward and revcomp
    assert emu[400] >= 39                                                     # the palindrome
    assert emu[o2 + 750] >= 59                                                # the copy across the end of contig 0
    assert emu[contigs[0][2] - 1] == 0 and emu[o1 - 2] == 1


def test_quirk_changes_lengths_somewhere(work):
    """the extra row of get_base_range does change L on random 2 kb references: the definition without it is not what
    the reference's walk computes, and the emulated walk follows the reference"""
    for seed in (0, 1):
        rng = np.random.default_rng(seed)
        fa = str(work / ("q%d.fa" % seed))
        open(fa, "w").write(">r\n" + "".join("ACGT"[v] for v in rng.integers(0, 4, 2000)) + "\n")
        p = R.build(fa, str(work / ("q%d" % seed)))
        emu = R.repeat_lengths(p, 0, 2000)
        plain = R.brute_lengths(p, quirk=False)
        assert np.array_equal(emu, R.brute_lengths(p, quirk=True)) and np.array_equal(emu, R.oracle_lengths(p))
        assert 1 <= int((emu != plain).sum()) <= 3 and ((emu == plain) | (emu > plain)).all()


@pytest.mark.parametrize("which", ["multi", "multi_n", "poly"])
def test_windows(which, multi, multi_n, small):
    """every window size from 1 position to the whole reference, windows across contig ends: the same array"""
    p = {"multi": multi, "multi_n": multi_n, "poly": small["poly"]}[which]
    n = R.layout(p)[0]
    whole = R.repeat_lengths(p, 0, n)
    assert np.array_equal(whole, R.oracle_lengths(p))
    for w in (1, 2, 3, 7, 64, 127, 128, 129, 1000, n - 1, n):
        got = np.concatenate([R.repeat_lengths(p, st, min(w, n - st)) for st in range(0, n, w)])
        assert np.array_equal(got, whole), w
    for st, k in [(0, 0), (n, 0), (n - 1, 1), (890, 40), (1, n - 1)]:
        assert np.array_equal(R.repeat_lengths(p, st, k), whole[st:st + k]), (st, k)
        assert np.array_equal(R.oracle_lengths(p, st, k), whole[st:st + k]), (st, k)
    for st, k in [(n, 1), (n + 1, 0), (0, n + 1)]:
        with pytest.raises(RuntimeError):
            R.repeat_lengths(p, st, k)


# ---------------------------------------------------------------- Python and CLI over the emulated device

@pytest.fixture
def emu(monkeypatch):
    from uncalled_b200 import _native as N
    fake = R.EmuLib()
    monkeypatch.setattr(N, "lib", lambda: fake)
    return fake


def _run(args, capsys):
    from uncalled_b200 import cli
    cli.main(["find-repeats"] + args)
    return capsys.readouterr().out


@pytest.mark.parametrize("which", ["multi", "multi_n"])
def test_cli_lines_and_bed(emu, capsys, which, multi, multi_n):
    p = {"multi": multi, "multi_n": multi_n}[which]
    L = R.oracle_lengths(p)
    for min_k in (0, 1, 9, 12, 40, int(L.max()), int(L.max()) + 1):
        assert _run([p, str(min_k)], capsys) == R.expected_lines(p, L, min_k), min_k
        assert _run([p, str(min_k), "--bed"], capsys) == R.expected_bed(p, L, min_k), min_k
    assert _run([p, str(int(L.max()) + 1)], capsys) == "" and _run([p, str(int(L.max()) + 1), "--bed"], capsys) == ""
    lines = _run([p, "0"], capsys).splitlines()
    hole = np.zeros(len(L), bool)
    for o, ln in R.layout(p)[2]:
        hole[o:o + ln] = True
    assert len(lines) == int((~hole).sum())                 # min_k 0: every position outside the holes
    if which == "multi_n":
        assert hole.any() and any("N" in ln.split("\t")[4] for ln in lines if len(ln.split("\t")) == 5)
        assert not any(ln.split("\t")[1] == "h0" and 100 <= int(ln.split("\t")[2]) < 130 for ln in lines)
    assert emu.calls.count("unc_repeats_create") == emu.calls.count("unc_repeats_destroy")


def test_bed_merges_overlapping_and_book_ended(emu, multi):
    """with small windows the runs are cut and carried across windows; book-ended intervals [a, b) [b, c) join"""
    from uncalled_b200 import repeats as RP
    st, en = RP.merge_intervals([0, 2, 5, 9, 9, 20], [5, 4, 9, 9, 12, 21])
    assert st.tolist() == [0, 20] and en.tolist() == [12, 21]
    L = R.oracle_lengths(multi)
    for w in (1, 5, 100, 10 ** 6):
        f = RP.RepeatFinder(multi, window=w)
        out = []
        class W:
            write = out.append
        RP.write_bed(f, 8, W)
        f.close()
        assert "".join(out) == R.expected_bed(multi, L, 8), w


def test_python_api(emu, multi_n):
    import uncalled_b200 as U
    p = multi_n
    L = R.oracle_lengths(p)
    f = U.RepeatFinder(p)
    try:
        _, contigs, _ = R.layout(p)
        assert f.contigs == [(n, ln) for n, _, ln in contigs]
        for name, off, ln in contigs:
            whole = f.lengths(name)
            assert whole.dtype == np.uint32 and np.array_equal(whole, L[off:off + ln])
            for st, en in [(0, 0), (0, 1), (3, 50), (ln - 1, ln), (ln, ln), (99, 131)]:
                assert np.array_equal(f.lengths(name, st, en), whole[st:en]), (name, st, en)
        recs = list(f.records(10))
        want = [ln.split("\t") for ln in R.expected_lines(p, L, 10).splitlines()]
        assert recs == [(int(w[0]), w[1], int(w[2])) for w in want]
        n_calls = len(emu.calls)
        for bad in [("nope",), ("h0", -1, 5), ("h0", 5, 4), ("h0", 0, contigs[0][2] + 1)]:
            with pytest.raises((KeyError, ValueError)):
                f.lengths(*bad)
        for bad in (-1, 1.5, True):
            with pytest.raises(ValueError):
                f.records(bad)
        assert len(emu.calls) == n_calls                     # refused before any device work
    finally:
        f.close()


def test_errors_before_the_device(emu, capsys, multi, tmp_path):
    from uncalled_b200 import cli
    for args in ([multi, "-1"], [str(tmp_path / "missing"), "5"]):
        with pytest.raises(SystemExit) as e:
            cli.main(["find-repeats"] + args)
        assert e.value.code == 1
    err = capsys.readouterr().err
    assert "min_k" in err and "does not exist" in err
    # inconsistent files: an .ann whose lengths do not add up, a .bwt of another reference, a short .pac
    import shutil
    for ext, mutate in [(".ann", lambda b: b.replace(b"\n0 900 0", b"\n0 901 0", 1)),
                        (".bwt", lambda b: b[:32] + (int.from_bytes(b[32:40], "little") + 2).to_bytes(8, "little") + b[40:]),
                        (".pac", lambda b: b[:10]), (".amb", lambda b: b"1 1 0\n")]:
        bad = str(tmp_path / ("bad" + ext.strip(".")))
        for e2 in (".bwt", ".sa", ".pac", ".ann", ".amb"):
            shutil.copy(multi + e2, bad + e2)
        open(bad + ext, "wb").write(mutate(open(multi + ext, "rb").read()))
        with pytest.raises(SystemExit) as e:
            cli.main(["find-repeats", bad, "3"])
        assert e.value.code == 1, ext
    assert emu.calls == []


# ---------------------------------------------------------------- the C-ABI without a device

def test_abi_arguments_and_no_device(multi):
    from uncalled_b200 import _native as N
    L = N.lib()
    h = C.c_void_p()
    assert L.unc_repeats_create(None, C.byref(h)) == -1
    assert L.unc_repeats_create(multi.encode(), None) == -1
    assert L.unc_repeats_lengths(None, 0, 1, None) == -1
    assert L.unc_repeats_last_kernel_ms(None, None) == -1
    L.unc_repeats_destroy(None)
    if L.unc_device_count() == 0:
        assert L.unc_repeats_create(multi.encode(), C.byref(h)) == -4 and not h.value
        with pytest.raises(N.UncError):
            N.check(-4)
