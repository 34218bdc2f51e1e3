"""GPU tier: every entry point gives back the device memory, pinned memory, streams and events it took, on success and
on failure (unc_debug_held).

The DTW workspace is kept between calls by design, so it is released (unc_dtw_release) before each reading.  No case
here exhausts device memory: each failure comes from the library's own size checks or from a request larger than any
device.
"""
import ctypes as C
import os

import numpy as np
import pytest

import dtwalignlib as D
import orclib

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNC_E_CUDA, UNC_E_NOMEM = -3, -6


@pytest.fixture(scope="module")
def U():
    import uncalled_b200
    L = uncalled_b200._native.lib()
    uncalled_b200._native.check(L.unc_init(0))
    return uncalled_b200


def _held(U):
    L = U._native.lib()
    L.unc_dtw_release()
    dev, pinned, handles = C.c_uint64(), C.c_uint64(), C.c_uint32()
    U._native.check(L.unc_debug_held(C.byref(dev), C.byref(pinned), C.byref(handles)))
    return dev.value, pinned.value, handles.value


def _example_reads(golden_read):
    raw = golden_read["raw"]
    return [raw, raw[:4000], raw[4000:8000]]


def _write_fasta(path, seqs):
    with open(path, "w") as f:
        for name, s in seqs:
            f.write(">%s\n%s\n" % (name, s))
    return path


def _random_bases(rng, n):
    return "".join("ACGT"[int(c)] for c in rng.integers(0, 4, n))


def test_every_entry_point_returns_what_it_held(U, example_prefix, golden_read, tmp_path):
    sigs = _example_reads(golden_read)
    rng = np.random.default_rng(7)
    genome = _random_bases(rng, 20000)
    fa = _write_fasta(str(tmp_path / "g.fa"), [("a", genome[:12000] + genome[:3000]), ("b", genome[12000:])])
    target = _write_fasta(str(tmp_path / "t.fa"), [("t", genome[2000:6000])])
    dprefix, codes = D.multi_contig_genome(str(tmp_path))

    def map_batch():
        idx = U.Index(example_prefix, device=0)
        bm = U.BatchMapper(idx, max_reads=8, max_samples=sum(len(s) for s in sigs))
        out = bm.map(np.concatenate(sigs), U.make_descs([len(s) for s in sigs]))
        assert all(r["status"] == 0 for r in out)
        bm.close()
        idx.close()

    def map_stream():
        idx = U.Index(example_prefix, device=0)
        sm = U.StreamMapper(idx, 4, 450)
        assert any(r is not None for r in sm.map_reads(sigs))
        sm.close()
        idx.close()

    def index_queries():
        idx = U.Index(example_prefix, device=0)
        assert np.isfinite(idx.match_probs(90.0)).all()
        st, en = idx.neighbors([1, 5, 9], [40, 60, 90], [0, 1, 2])
        assert len(st) == len(en) == 3
        assert len(idx.sa([1, 2, 3])) == 3
        idx.close()

    def dtw_align():
        from uncalled_b200.dtw import DtwAligner
        A = DtwAligner(dprefix)
        sig = D.span_signal(codes["chrA"][100:1100], True, np.random.default_rng(3))
        got = A.align([("r", sig, None, 0, 0, "chrA", 100, 1100, True)])
        assert got[0].skip is None
        A.close()

    def dtw_batch():
        from uncalled_b200.dtw import DTWParams, dtw_batch
        means = np.random.default_rng(5).uniform(70, 110, 200).astype(np.float32)
        kmers = np.random.default_rng(6).integers(0, 1024, 150).astype(np.uint16)
        assert len(dtw_batch([(means, kmers)], DTWParams())) == 1

    def self_align():
        off, _ = U.index.self_align_csr(example_prefix, 3)
        assert len(off) > 1

    def build_index():
        U.BwaIndex.create(fa, str(tmp_path / "built"))
        assert os.path.getsize(str(tmp_path / "built.bwt")) > 0

    def mask_internal():
        assert len(U.mask_internal(fa, 5, 3, str(tmp_path / "mi_"), log=None)) == 3

    def mask_external():
        U.mask_external(fa, target, 20, 1, str(tmp_path / "mx_"))

    for op in (map_batch, map_stream, index_queries, dtw_align, dtw_batch, self_align, build_index, mask_internal,
               mask_external):
        before = _held(U)
        op()
        assert _held(U) == before, op.__name__


def test_failed_creates_hold_nothing(U, example_prefix):
    L = U._native.lib()
    idx = U.Index(example_prefix, device=0)
    before = _held(U)
    p = U.default_params()
    h = C.c_void_p()
    assert L.unc_pool_create(idx.h, C.byref(p), 8, 1 << 40, C.byref(h)) == UNC_E_NOMEM    # 4 TiB of samples
    assert not h.value and _held(U) == before
    assert L.unc_stream_create(idx.h, C.byref(p), 1000000, 450, 1000000, C.byref(h)) == UNC_E_NOMEM
    assert not h.value and _held(U) == before
    idx.close()


def test_pool_recovers_from_a_failed_events_buffer(U, example_prefix, golden_read):
    """One read of 2^24 samples in a pool of 65 536 reads needs a 4 TiB events buffer: the allocation fails at once and
    the call returns UNC_E_CUDA.  The pool must then map as before: its events buffer is reallocated rather than left
    null, and the failed allocation is not reported as the next launch's error.  The example reads are cut to 4 000
    samples, which keeps the pool's own events buffer at 1 GiB."""
    sigs = _example_reads(golden_read)[1:]
    flat = np.concatenate(sigs)
    descs = U.make_descs([len(s) for s in sigs])
    O = orclib.Oracle(example_prefix)
    want = [orclib.paf_tuple(O.map_read(s)) for s in sigs]
    idx = U.Index(example_prefix, device=0)
    bm = U.BatchMapper(idx, max_reads=65536, max_samples=1 << 24)
    assert [U.paf_key(r) for r in bm.map(flat, descs)] == want
    held = _held(U)
    big = np.zeros(1 << 24, np.float32)
    out = np.zeros(1, dtype=U._native.PAF_DTYPE)
    rc = bm.L.unc_map_batch(bm.h, U.make_descs([1 << 24]).ctypes.data, 1, big.ctypes.data, out.ctypes.data)
    assert rc == UNC_E_CUDA
    assert b"events buffer" in bm.L.unc_last_error()
    assert [U.paf_key(r) for r in bm.map(flat, descs)] == want
    assert _held(U) == held
    bm.close()
    idx.close()
