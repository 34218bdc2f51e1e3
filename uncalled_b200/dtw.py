"""DTW of event means against reference k-mers: the reference's `DTWr94p`, `DTWr94d`, `DTWParams` and the `DTW_*` presets
(src/dtw.hpp:9-28,188-232, bound at src/pybinder.cpp:75-91) over `unc_dtw_batch` (include/unc_b200.h).

    d = DTWr94p(means, kmers, DTW_EVENT_GLOB); d.get_path(); d.score(); d.mean_score()

`dtw_batch` aligns many (means, kmers) pairs in one call (one CTA per problem on the GPU).  There is no CPU path."""
import ctypes as C
import os

import numpy as np

from . import _native as N


class DTWSubSeq:                      # enum class DTWSubSeq {NONE, ROW, COL}, src/dtw.hpp:9
    NONE, ROW, COL = 0, 1, 2


class DTWParams(C.Structure):
    """DTWParams (src/dtw.hpp:10-13): subseq, dw, hw, vw -- the weights of the diagonal, horizontal and vertical moves."""
    _fields_ = [("subseq", C.c_int32), ("dw", C.c_float), ("hw", C.c_float), ("vw", C.c_float)]

    def __init__(self, subseq=DTWSubSeq.NONE, dw=1.0, hw=1.0, vw=1.0):
        super().__init__(int(subseq), float(dw), float(hw), float(vw))


# src/dtw.hpp:15-28
DTW_EVENT_GLOB = DTWParams(DTWSubSeq.NONE, 2, 1, 100)
DTW_EVENT_QSUB = DTWParams(DTWSubSeq.COL, 2, 1, 100)
DTW_EVENT_RSUB = DTWParams(DTWSubSeq.ROW, 2, 1, 100)
DTW_RAW_QSUB = DTWParams(DTWSubSeq.COL, 10, 1, 1000)
DTW_RAW_RSUB = DTWParams(DTWSubSeq.ROW, 10, 1, 1000)
DTW_RAW_GLOB = DTWParams(DTWSubSeq.NONE, 10, 1, 1000)

_model = None


def model_table():
    """The r9.4 template model as (mean, stdv) pairs per 5-mer (src/model_r94.inl)."""
    global _model
    if _model is None:
        _model = np.fromfile(N.MODEL_TABLE, dtype=np.float32)
        assert _model.size == 2048
    return _model


def dtw_batch(problems, prms, cost="r94p", model=None, band=0):
    """problems: sequence of (means, kmers).  Returns a list of (path, score): path = uint64 array [n, 2] of (column =
    event index, row = k-mer index) pairs from the end of the alignment back to its start, as `get_path()` gives them.
    band = 0 fills the whole matrix; band = W >= 1 only the rows within W (widened to the diagonal's slope) of each column's
    point on the diagonal (`unc_dtw_batch_banded`, global alignment only): the score is never below the full one and equals
    it when the full path stays in the band."""
    L = N.lib()
    args = [C.c_void_p, C.c_int, C.POINTER(DTWParams), C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
            C.c_void_p, C.c_void_p, C.c_void_p]
    L.unc_dtw_batch.argtypes = args
    L.unc_dtw_batch_banded.argtypes = args + [C.c_uint32]
    n = len(problems)
    if n == 0:
        return []
    means = [np.ascontiguousarray(m, dtype=np.float32).ravel() for m, _ in problems]
    kmers = [np.ascontiguousarray(k, dtype=np.uint16).ravel() for _, k in problems]
    moff = np.zeros(n + 1, np.uint64)
    koff = np.zeros(n + 1, np.uint64)
    poff = np.zeros(n + 1, np.uint64)
    moff[1:] = np.cumsum([len(m) for m in means])
    koff[1:] = np.cumsum([len(k) for k in kmers])
    poff[1:] = np.cumsum([len(m) + len(k) for m, k in zip(means, kmers)])
    am, ak = np.concatenate(means), np.concatenate(kmers)
    path = np.zeros((int(poff[-1]), 2), np.uint64)
    plen = np.zeros(n, np.uint64)
    score = np.zeros(n, np.float32)
    tab = np.ascontiguousarray(model if model is not None else model_table(), dtype=np.float32)
    kind = {"r94p": 0, "r94d": 1}[cost]
    a = (tab.ctypes.data, kind, C.byref(prms), n, am.ctypes.data, moff.ctypes.data, ak.ctypes.data, koff.ctypes.data,
         path.ctypes.data, poff.ctypes.data, plen.ctypes.data, score.ctypes.data)
    if not 0 <= band < 1 << 32:
        raise ValueError("band must be 0 (the full matrix) or a half-width from 1 to 2^32 - 1")
    N.check(L.unc_dtw_batch_banded(*a, int(band)) if band else L.unc_dtw_batch(*a))
    return [(path[int(poff[i]):int(poff[i]) + int(plen[i])].copy(), float(score[i])) for i in range(n)]


class _DTW:
    _cost = None

    def __init__(self, means, kmers, prms):
        (self._path, self._score), = dtw_batch([(means, kmers)], prms, self._cost)

    def get_path(self):
        """[(event index, k-mer index), ...] from the end of the alignment back to its start (src/dtw.hpp:124-126)."""
        return [(int(a), int(b)) for a, b in self._path]

    def score(self):
        return self._score

    def mean_score(self):             # score_sum_ / path_.size() in float (src/dtw.hpp:132-134)
        return float(np.float32(self._score) / np.float32(len(self._path)))


class DTWr94p(_DTW):
    """cost = -match_prob(event, k-mer) of the r9.4 template model (src/dtw.hpp:188-209)"""
    _cost = "r94p"


class DTWr94d(_DTW):
    """cost = abs(event - model mean of the k-mer), as the reference compiles it: the difference is truncated to an
    integer first (src/dtw.hpp:212-232)"""
    _cost = "r94d"


# ---------------------------------------------------------------- reads against reference spans (the dtw_test driver)

class DtwQuery(C.Structure):
    """unc_dtw_query (include/unc_b200.h)"""
    _fields_ = [("rid", C.c_int32), ("fwd", C.c_uint32), ("rf_st", C.c_uint64), ("rf_en", C.c_uint64)]


class DtwAlignResult(C.Structure):
    """unc_dtw_align_result (include/unc_b200.h)"""
    _fields_ = [("status", C.c_int32), ("n_events", C.c_uint32), ("n_kept", C.c_uint32), ("score", C.c_float),
                ("mean_score", C.c_float), ("pad", C.c_uint32), ("path_len", C.c_uint64)]


MAX_MEANS = 50000                     # src/dtw_test.cpp:156
# why a query is skipped (UNC_DTW_ALIGN_* of include/unc_b200.h)
SKIP_REASONS = {1: "too many means", 2: "no event left after the mask", 3: "the DTW matrix exceeds the workspace budget",
                4: "unknown contig", 5: "rf_en past the end of the contig", 6: "reference span shorter than 5 bases",
                7: "empty sample range"}
RD_EN_PAST_END = "rd_en past the end of the signal"


class Alignment:
    """One query's outcome: `skip` is None when it was aligned, else the reason ("too many means" for the reference's
    own skip above 50 000 means).  With paths: `path` = (event index, k-mer index) pairs from the start cell to the end
    cell, `means` = the normalised kept means, `kmers` = the span's k-mers."""
    __slots__ = ("read_id", "skip", "n_events", "n_kept", "score", "mean_score", "path", "means", "kmers")

    def __init__(self, read_id, skip=None, **kw):
        self.read_id, self.skip = read_id, skip
        for k in self.__slots__[2:]:
            setattr(self, k, kw.get(k))

    def skip_message(self):
        """The stderr line of a skipped query (src/dtw_test.cpp:157 for the > 50 000 means case)."""
        return "Skipping %s" % self.read_id if self.skip == "too many means" else "Skipping %s: %s" % (self.read_id, self.skip)


class DtwAligner:
    """The reference's dtw_test driver (src/dtw_test.cpp:94-175) on the GPU: reads aligned by DTWr94d to their reference
    spans, after event detection, the EventProfiler mask and normalisation to the span's model levels.  Only the .pac and
    .ann of `bwa_prefix` are read.  `budget`: bytes of the DTW sweep's workspace (0 = the free device memory).  `band`: 0
    aligns with the full matrix and skips reads over 50 000 kept means, as the reference does; W >= 1 aligns with the banded
    sweep of half-width W (see `dtw_batch`), where only the budget limits a read's length."""

    def __init__(self, bwa_prefix, budget=0, band=0):
        self._L = N.lib()
        self._h = C.c_void_p()
        N.check(self._L.unc_dtw_aligner_create(os.fsencode(bwa_prefix), os.fsencode(N.MODEL_TABLE), C.byref(self._h)))
        self.set_budget(budget)
        self.set_band(band)

    def close(self):
        if getattr(self, "_h", None):
            self._L.unc_dtw_aligner_free(self._h)
            self._h = None

    __del__ = close

    def set_budget(self, nbytes):
        N.check(self._L.unc_dtw_aligner_set_budget(self._h, int(nbytes)))

    def set_band(self, band):
        """0: the full matrix; W >= 1: the banded sweep of half-width W"""
        if not 0 <= band < 1 << 32:
            raise ValueError("band must be 0 (the full matrix) or a half-width from 1 to 2^32 - 1")
        N.check(self._L.unc_dtw_aligner_set_band(self._h, int(band)))

    def contig(self, name):
        """(rid, length) of a contig of the .ann, or None"""
        rid, ln = C.c_int32(), C.c_uint64()
        N.check(self._L.unc_dtw_aligner_contig(self._h, name.encode(), C.byref(rid), C.byref(ln)))
        return None if rid.value < 0 else (rid.value, ln.value)

    def align(self, queries, paths=False):
        """queries: (read_id, signal, calibration, rd_st, rd_en, contig, rf_st, rf_en, fwd) per read, all with the same
        signal type: float32 pA (calibration None) or int16 DAC values with their (range, offset, digitisation).
        rd_st = rd_en = 0 takes the whole signal; rd_en = 0 runs to its end.  Returns one Alignment per query, in order."""
        n = len(queries)
        out = [None] * n
        descs = (N.ReadDesc * max(n, 1))()
        qs = (DtwQuery * max(n, 1))()
        parts, off = [], 0
        for i, (rid_, sig, cal, rd_st, rd_en, contig, rf_st, rf_en, fwd) in enumerate(queries):
            en = len(sig) if rd_en == 0 else rd_en
            c = self.contig(contig)
            qs[i].rid, qs[i].fwd, qs[i].rf_st, qs[i].rf_en = (c[0] if c else -1), int(bool(fwd)), int(rf_st), int(rf_en)
            d = descs[i]
            d.offset, d.dtype = off, 0 if cal is None else 1
            if cal is not None:
                d.cal_range, d.cal_offset, d.cal_digit = cal
            if en > len(sig) or rd_st >= en:
                out[i] = Alignment(rid_, RD_EN_PAST_END if en > len(sig) else SKIP_REASONS[7])
                d.n_samples = 0
            else:
                part = sig[rd_st:en]
                parts.append(part)
                d.n_samples = len(part)
                off += len(part)
        dtypes = {descs[i].dtype for i in range(n)}
        if len(dtypes) > 1:
            raise ValueError("one batch holds one signal type")
        samples = np.concatenate(parts) if parts else np.zeros(1, np.float32)
        samples = np.ascontiguousarray(samples, dtype=np.int16 if dtypes == {1} else np.float32)
        res = (DtwAlignResult * max(n, 1))()
        N.check(self._L.unc_dtw_align_batch(self._h, n, descs, samples.ctypes.data, qs, 1 if paths else 0, res))
        for i in range(n):
            if out[i] is not None:
                continue
            r = res[i]
            kw = dict(n_events=r.n_events, n_kept=r.n_kept)
            if r.status:
                out[i] = Alignment(queries[i][0], SKIP_REASONS[r.status], **kw)
                continue
            kw.update(score=float(r.score), mean_score=float(r.mean_score))
            if paths:
                p = np.zeros((r.path_len, 2), np.uint64)
                m = np.zeros(max(r.n_kept, 1), np.float32)
                k = np.zeros(max(qs[i].rf_en - qs[i].rf_st - 4, 1), np.uint16)
                N.check(self._L.unc_dtw_align_path(self._h, i, p.ctypes.data, m.ctypes.data, k.ctypes.data))
                kw.update(path=p[::-1].copy(), means=m[:r.n_kept], kmers=k[:qs[i].rf_en - qs[i].rf_st - 4])
            out[i] = Alignment(queries[i][0], **kw)
        return out

    def last_times(self):
        """CUDA-event times of the last batch in ms: h2d, events, mask, kmers, target, norm, sweep, total; then the
        number of sweep launches and of matrix cells (in-band cells with a band)."""
        ms = np.zeros(8, np.float32)
        la, ce = C.c_uint64(), C.c_uint64()
        N.check(self._L.unc_dtw_align_last_times(self._h, ms.ctypes.data, C.byref(la), C.byref(ce)))
        keys = ("h2d", "events", "mask", "kmers", "target", "norm", "sweep", "total")
        return dict(zip(keys, (float(x) for x in ms))), la.value, ce.value


def r94d_cost(kmer, mean):
    """DTWr94d's cost of (k-mer, event mean) as the reference's dtw_test driver compiles it: the float abs of the float
    difference (the driver includes <math.h> before dtw.hpp)."""
    lv = model_table()[0::2]
    return np.abs(np.asarray(mean, np.float32) - lv[np.asarray(kmer, dtype=np.int64)].astype(np.float32)).astype(np.float32)


def format_path(a):
    """The lines of the path file of an Alignment (print_path, src/dtw.hpp:135-143): event index, k-mer index, the
    k-mer of the row, the mean of the column and their cost, each followed by a tab."""
    ev, km = a.path[:, 0].astype(np.int64), a.path[:, 1].astype(np.int64)
    k = a.kmers[km]
    m = a.means[ev]
    c = r94d_cost(k, m)
    return "".join("%d\t%d\t%d\t%g\t%g\t\n" % (e, r, kk, float(mm), float(cc)) for e, r, kk, mm, cc in zip(ev, km, k, m, c))


class QueryError(ValueError):
    pass


def load_queries(fname, aligner):
    """load_queries (src/dtw_test.cpp:27-58): `rd_name rd_st rd_en rf_name rf_st rf_en strand` per line, keyed by read
    name (a later line for a read replaces an earlier one).  Returns {read name: (rd_st, rd_en, contig, rf_st, rf_en,
    fwd)}.  A malformed line, an unknown contig or a strand other than + / - rejects the whole file (QueryError)."""
    out = {}
    with open(fname) as f:
        for ln, line in enumerate(f, 1):
            fields = line.split()
            if not fields:
                continue
            where = "%s:%d: " % (fname, ln)
            if len(fields) != 7:
                raise QueryError(where + "expected 7 fields (rd_name rd_st rd_en rf_name rf_st rf_en strand), got %d" % len(fields))
            name, rd_st, rd_en, contig, rf_st, rf_en, strand = fields
            try:
                nums = [int(x, 10) for x in (rd_st, rd_en, rf_st, rf_en)]
            except ValueError:
                raise QueryError(where + "coordinates must be non-negative integers") from None
            if min(nums) < 0 or max(nums[:2]) >= 1 << 32 or max(nums[2:]) >= 1 << 64:
                raise QueryError(where + "coordinates must be non-negative integers")
            if strand not in ("+", "-"):
                raise QueryError(where + "strand must be + or -, got %r" % strand)
            if aligner.contig(contig) is None:
                raise QueryError(where + "unknown contig %r" % contig)
            out[name] = (nums[0], nums[1], contig, nums[2], nums[3], strand == "+")
    return out


def host_skip(aligner, n_signal, rd_st, rd_en, contig, rf_st, rf_en):
    """The reason a query is skipped before the device, or None (unc_dtw_align_batch applies the same checks)."""
    en = n_signal if rd_en == 0 else rd_en
    if en > n_signal:
        return RD_EN_PAST_END
    if rd_st >= en:
        return SKIP_REASONS[7]
    rid, ln = aligner.contig(contig)
    if rf_en > ln or rf_st > rf_en:
        return SKIP_REASONS[5]
    if rf_en - rf_st < 5:
        return SKIP_REASONS[6]
    return None
