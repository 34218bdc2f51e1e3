"""BwaIndex queries on the H100 (uncalled_b200.index.BwaIndex and `_uncalled.BwaIndex` over unc_bwa_*): every row's
sa, every neighbour, every range_to_fms span, get_kmers and translate_loc of the fixtures against what the reference's
own BwaIndex computed (tests/golden/bwa_index_golden.json) and against the serial C restatement of its loops;
scalar against batched calls, on indexes that have no .uncl."""
import numpy as np
import pytest

import bwaindexlib as B
from uncalled_b200 import index as I

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=B.FIXTURES)
def fixture(request, tmp_path_factory):
    return B.build(request.param, tmp_path_factory.mktemp(request.param))


@pytest.fixture(scope="module")
def X(fixture):
    x = I.BwaIndex(fixture, True)
    yield x
    x.destroy()


def test_sa_every_row(fixture, X):
    R = B.Restated(fixture)
    rows = np.arange(X.size() + 1, dtype=np.uint64)
    got = X.sa(rows)
    assert np.array_equal(got, R.sa(rows))
    assert got[0] == np.uint64(2**64 - 1)
    for r in (0, 1, X.size() // 2, X.size()):
        assert X.sa(r) == int(got[r])


def test_neighbor_every_row(fixture, X):
    R = B.Restated(fixture)
    st, en, base = B.neighbor_queries(X.size(), np.random.default_rng(7))
    got = X.get_neighbor(st, en, base)
    want = R.neighbors(st, en, base)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    for i in np.random.default_rng(1).integers(0, len(st), 50):
        r = X.get_neighbor(I.Range(int(st[i]), int(en[i])), int(base[i]))
        assert (r.start, r.end) == (int(want[0][i]), int(want[1][i]))


def test_range_to_fms_spans(fixture, X):
    R = B.Restated(fixture)
    for name, st, en in B.spans(fixture):
        got, want = X.range_to_fms(name, st, en), R.range_to_fms(name, st, en)
        assert np.array_equal(got[0], want[0]), (name, st, en, "first")
        assert np.array_equal(got[1], want[1]), (name, st, en, "second")


def test_range_to_fms_whole_contig_is_the_inverse_of_sa(fixture, X):
    sa = X.sa(np.arange(X.size() + 1, dtype=np.uint64))
    isa = np.empty(X.size() + 1, np.uint64)
    isa[sa[1:].astype(np.int64)] = np.arange(1, X.size() + 1, dtype=np.uint64)
    for name, off, ln in B.contigs(fixture):
        first, second = X.range_to_fms(name, 0, ln)
        assert np.array_equal(second, isa[np.arange(off + ln - 1, off - 1, -1)])
        # the reverse walk joins the exact chain: row of pac_min + j is the row of text suffix size() - 1 - (pac_min + j)
        exact = isa[X.size() - 1 - np.arange(off, off + ln)]
        assert np.array_equal(first[-min(ln, 64):], exact[-min(ln, 64):])


def test_get_kmers(fixture, X):
    for name, off, ln in B.contigs(fixture):
        for st, en in ((0, ln), (3, 9), (5, 9), (ln - 5, ln), (7, 7 + 257)):
            if en > ln or st < 0:
                continue
            want = B.seq_to_kmers(fixture, off + st, off + en)
            assert np.array_equal(X.get_kmers(off + st, off + en), want)
            assert np.array_equal(X.get_kmers(name, st, en), want)


def test_kmer_ranges_match_the_neighbor_walk(X):
    for k in range(1024):
        r = X.get_base_range(I.kmer_head(k))
        for i in range(1, 5):
            r = X.get_neighbor(r, I.kmer_base(k, i))
        assert X.get_kmer_range(k) == r and X.get_kmer_count(k) == r.length()


def test_uncalled_module_agrees(fixture, X):
    U = B.uncalled_module()
    u = U.BwaIndex(fixture, True)
    for name, st, en in B.spans(fixture)[:6]:
        a, b = u.range_to_fms(name, st, en)
        c, d = X.range_to_fms(name, st, en)
        assert list(a) == c.tolist() and list(b) == d.tolist()
    assert u.sa(5) == X.sa(5)
    r = u.get_neighbor(U.Range(3, 40), 2)
    assert (r.start, r.end) == (lambda q: (q.start, q.end))(X.get_neighbor(I.Range(3, 40), 2))
    name, off, ln = B.contigs(fixture)[0]
    assert list(u.get_kmers(name, 0, min(ln, 60))) == X.get_kmers(name, 0, min(ln, 60)).tolist()
    u.destroy()


class OnDevice:
    """index.BwaIndex in the shape bwaindexlib.golden_record reads"""

    def __init__(self, X):
        self.X, self.size = X, X.size()

    def sa(self, rows):
        return self.X.sa(rows)

    def neighbors(self, st, en, base):
        return self.X.get_neighbor(st, en, base)

    def range_to_fms(self, name, a, b):
        return self.X.range_to_fms(name, a, b)

    def get_kmers(self, a, b):
        k = self.X.get_kmers(a, b)
        return k, np.array([I.kmer_revcomp(int(x)) for x in k[::-1]], np.uint16)

    def translate_loc(self, p):
        return self.X.translate_loc(p)


def test_matches_the_golden(fixture, X):
    import os
    name = os.path.basename(fixture)
    want = B.golden()["fixtures"]["example" if name not in B.golden()["fixtures"] else name]
    got = B.golden_record(fixture, OnDevice(X))
    for k in ("size", "sa", "neighbor", "fms", "kmers", "translate_loc"):
        assert got[k] == want[k], k
