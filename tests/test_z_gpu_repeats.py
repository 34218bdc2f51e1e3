"""GPU tier of `find-repeats`: unc_repeats_lengths (k_repeat_lengths) on the H100 against the oracle and the reference's
own self_align at every position of the example index, the small indexes and a 4.7 Mb seeded genome with planted repeat
families; the command's output there against the output built from the oracle's arrays; the 1.1 Gbp index (2.2e9 FM
rows) against a walk restated from the .bwt file; device memory after every call."""
import ctypes as C
import os
import tempfile
import time

import numpy as np
import pytest

import fmsteplib as F
import orclib
import repeatslib as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def U():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import uncalled_b200 as U
    return U


def _held():
    from uncalled_b200 import _native as N
    d, p, h = C.c_uint64(), C.c_uint64(), C.c_uint32()
    N.check(N.lib().unc_debug_held(C.byref(d), C.byref(p), C.byref(h)))
    return d.value, h.value


def _all(U, prefix):
    with U.RepeatFinder(prefix) as f:
        return f._raw(0, f.l_pac)


def test_bit_for_bit_small_indexes(U, tmp_path):
    """every position of the example index and of the FM-step fixtures: the oracle, and the digests of the reference's
    own self_align that tests/test_repeats.py checks live"""
    ex = orclib.materialise_example_index(str(tmp_path))
    L = _all(U, ex)
    assert np.array_equal(L, R.oracle_lengths(ex))
    R.expect_reference("find_repeats/example", (L,))
    got = []
    for name in sorted(F.FIXTURES):
        p = F.build(name, tmp_path)
        got.append(_all(U, p))
        assert np.array_equal(got[-1], R.oracle_lengths(p)), name
    R.expect_reference("find_repeats/fm_step_fixtures", tuple(got))


def test_seeded_genome_with_repeat_families_and_cli(U, tmp_path, capsys):
    from uncalled_b200 import _native as N
    from uncalled_b200 import cli
    fa, prefix = str(tmp_path / "fam.fa"), str(tmp_path / "fam")
    R.write_fasta(fa, R.family_genome(4_700_000, 47), ["famA", "famB"])
    N.check(N.lib().unc_init(0))
    N.check(N.lib().unc_index_build_device(fa.encode(), prefix.encode()))
    t = time.time()
    L = _all(U, prefix)
    t_gpu = time.time() - t
    t = time.time()
    want = R.oracle_lengths(prefix)
    with capsys.disabled():
        print("4.7 Mb with families: GPU %.2f s, oracle %.2f s, sum(L + 1) = %d, max L = %d" %
              (t_gpu, time.time() - t, int(L.astype(np.int64).sum()) + len(L), int(L.max())))
    assert np.array_equal(L, want), np.flatnonzero(L != want)[:5]
    assert L.max() >= 5000
    for min_k in (25, 1000):
        cli.main(["find-repeats", prefix, str(min_k)])
        assert capsys.readouterr().out == R.expected_lines(prefix, want, min_k), min_k
        cli.main(["find-repeats", prefix, str(min_k), "--bed"])
        assert capsys.readouterr().out == R.expected_bed(prefix, want, min_k), min_k


def test_no_leaks(U, tmp_path):
    from uncalled_b200 import _native as N
    L = N.lib()
    ex = orclib.materialise_example_index(str(tmp_path))
    N.check(L.unc_init(0))
    base = _held()
    h = C.c_void_p()
    N.check(L.unc_repeats_create(ex.encode(), C.byref(h)))
    out = np.zeros(10000, np.uint32)
    N.check(L.unc_repeats_lengths(h, 0, 10000, out.ctypes.data))
    ms = C.c_float()
    N.check(L.unc_repeats_last_kernel_ms(h, C.byref(ms)))
    assert ms.value > 0
    assert L.unc_repeats_lengths(h, 1, 10000, out.ctypes.data) == -1       # past the end
    assert L.unc_repeats_lengths(h, 0, 5, None) == -1
    L.unc_repeats_destroy(h)
    assert _held() == base
    assert L.unc_repeats_create((ex + "_missing").encode(), C.byref(h)) == -2 and not h.value
    assert _held() == base
    os.remove(ex + ".pac")
    assert L.unc_repeats_create(ex.encode(), C.byref(h)) == -2
    assert _held() == base


def occ_of_base(prefix, rows, c):
    """bwt_occ(row, c) for one base per row (submods/bwa/bwt.c:107-129), read from the .bwt file: the row's 128-row block
    count of c plus the c symbols of the block up to the row, counted per 16-symbol word with popcounts.  Row -1 gives 0
    (a range starting at row 0), row n the count of c.  fmsteplib.occ_at_rows computes the same for all four bases."""
    head = np.fromfile(prefix + ".bwt", np.uint64, 5)
    primary, L2 = int(head[0]), np.concatenate([[0], head[1:5]]).astype(np.int64)
    n = int(L2[4])
    words = np.memmap(prefix + ".bwt", np.uint32, "r", offset=40)
    k, c = np.asarray(rows, np.int64), np.asarray(c, np.int64)
    out = np.zeros(len(k), np.int64)
    end = k == n
    out[end] = (L2[c + 1] - L2[c])[end]
    m = (k >= 0) & ~end
    kk = k[m] - (k[m] >= primary)
    base, cm = (kk >> 7) * 16, c[m]
    top = len(words) - 1
    cnt = words[np.minimum(base + 2 * cm, top)].astype(np.int64) | (words[np.minimum(base + 2 * cm + 1, top)].astype(np.int64) << 32)
    w = words[np.minimum(base[:, None] + 8 + np.arange(8), top)].astype(np.uint64)
    x = w ^ (cm.astype(np.uint64) * np.uint64(0x55555555))[:, None]
    eq = ~(x | (x >> np.uint64(1))) & np.uint64(0x55555555)              # low bit of every symbol equal to c
    nsym = np.clip((kk & 127)[:, None] - 16 * np.arange(8) + 1, 0, 16).astype(np.uint64)
    keep = (np.uint64(0xFFFFFFFF) << (np.uint64(32) - 2 * nsym)) & np.uint64(0xFFFFFFFF)  # the first nsym symbols
    out[m] = cnt + np.bitwise_count(eq & keep).sum(1).astype(np.int64)
    return out


def _walk_restated(prefix, pac, lim_of, pos, chunk=1 << 18):
    """self_align's walk from each position, restated in numpy with bwt_occ read per row from the .bwt file; returns
    (L, the rows the walks' ranges started and ended at)"""
    head = np.fromfile(prefix + ".bwt", np.uint64, 5)
    L2 = np.concatenate([[0], head[1:5]]).astype(np.int64)

    def comp(q):
        return 3 - ((pac[q >> 2] >> ((3 - (q & 3)) * 2)) & 3).astype(np.int64)

    out = np.zeros(len(pos), np.int64)
    seen = []
    for o in range(0, len(pos), chunk):
        p = np.asarray(pos[o:o + chunk], np.int64)
        lim = lim_of(p)
        b = comp(p)
        rs, re = L2[b], L2[b + 1]
        j = p + 1
        act = np.arange(len(p))
        while True:
            go = (j[act] < lim[act]) & (re[act] - rs[act] + 1 > 1)
            act = act[go]
            if not len(act):
                break
            c = comp(j[act])
            os_, oe = occ_of_base(prefix, rs[act] - 1, c), occ_of_base(prefix, re[act], c)
            rs[act], re[act] = L2[c] + os_ + 1, L2[c] + oe
            seen.append(np.concatenate([rs[act], re[act]]))
            j[act] += 1
        out[o:o + len(p)] = j - p - 1
        print("restated walks: %d of %d positions" % (o + len(p), len(pos)), flush=True)
    return out, np.concatenate(seen)


def test_above_2_31_rows(U, tmp_path):
    """the 1.1 Gbp genome of test_index_build_device.py: a 1 Mb slice and 20 000 random positions against the walk
    restated from the .bwt, with walks through rows near 2^31 and the `$` row; and the whole genome, timed"""
    import indexlib as I
    from uncalled_b200 import _native as N
    work = tempfile.mkdtemp(dir=str(tmp_path))
    fa, prefix = os.path.join(work, "big.fa"), os.path.join(work, "big")
    with open(fa, "wb") as f:
        f.write(I.big_fasta())
    N.check(N.lib().unc_init(0))
    t0 = time.time()
    N.check(N.lib().unc_index_build_device(fa.encode(), prefix.encode()))
    os.remove(fa)
    print("1.1 Gbp index built in %.1f s" % (time.time() - t0), flush=True)
    _, contigs, _ = R.layout(prefix)
    ends = np.cumsum([ln for _, _, ln in contigs])
    l_pac = int(ends[-1])
    assert 2 * l_pac + 1 > 2 ** 31
    pac = np.fromfile(prefix + ".pac", np.uint8)
    rng = np.random.default_rng(31)
    st = int(rng.integers(0, l_pac - 1_000_000))
    pos = np.concatenate([np.arange(st, st + 1_000_000), rng.integers(0, l_pac, 20_000)])
    t0 = time.time()
    with U.RepeatFinder(prefix) as f:
        # the whole genome, window by window
        buf = np.empty(f.window, np.uint32)
        steps, ms, kernel = 0, C.c_float(), 0.0
        for o in range(0, l_pac, f.window):
            k = min(f.window, l_pac - o)
            N.check(f._L.unc_repeats_lengths(f._h, o, k, buf.ctypes.data))
            N.check(f._L.unc_repeats_last_kernel_ms(f._h, C.byref(ms)))
            kernel += ms.value
            steps += int(buf[:k].sum(dtype=np.int64)) + k
            print("  window at %d: %.1f s" % (o, time.time() - t0), flush=True)
        print("1.1 Gbp whole genome: %.1f s wall, %.1f s in the kernel, %d steps" % (time.time() - t0, kernel / 1e3, steps),
              flush=True)
        got = np.concatenate([f._raw(st, 1_000_000), np.array([f._raw(int(q), 1)[0] for q in pos[1_000_000:]])])
    print("1.1 Gbp: GPU lengths of %d positions done" % len(pos), flush=True)
    t0 = time.time()
    want, rows = _walk_restated(prefix, pac, lambda p: ends[np.searchsorted(ends, p, side="right")], pos)
    assert np.array_equal(got.astype(np.int64), want), np.flatnonzero(got != want)[:5]
    primary = int(np.fromfile(prefix + ".bwt", np.uint64, 1)[0])
    near = lambda r: int(np.abs(rows - r).min())
    print("1.1 Gbp: %d positions checked in %.1f s; nearest walk rows to 2^31 and to primary: %d, %d"
          % (len(pos), time.time() - t0, near(2 ** 31), near(primary)))
    assert near(2 ** 31) < 2000 and near(primary) < 2000
