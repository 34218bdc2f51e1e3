"""Host-side objects over the C-ABI: Index (device image of a bwa/UNCALLED index) and
BatchMapper (a device workspace that maps batches of raw reads).

These sit directly under the reference-shaped interface in uncalled_b200/api.py
(Conf / MapPool / Paf, mirroring reference src/pybinder.cpp:14-91); they hold no mapping
logic themselves -- every result comes from the CUDA kernels behind include/unc_b200.h.
"""
import ctypes as C

import numpy as np

from . import _native as N


class Index:
    """unc_index: replaces Mapper::load_static / BwaIndex::load_index
    (reference src/mapper.cpp:109-159, src/bwa_index.hpp:116-135)."""

    def __init__(self, bwa_prefix, preset="default", device=0, model_table=None):
        self.L = N.lib()
        N.check(self.L.unc_init(int(device)))
        self.h = C.c_void_p()
        N.check(self.L.unc_index_load(str(bwa_prefix).encode(), str(preset).encode(),
                                      (model_table or N.MODEL_TABLE).encode(), C.byref(self.h)))
        info = N.IndexInfo()
        N.check(self.L.unc_index_get_info(self.h, C.byref(info)))
        self.n_rows, self.n_seqs, self.device, self.device_bytes = info.n_rows, info.n_seqs, info.device, info.device_bytes
        self.seqs = []
        for i in range(self.n_seqs):
            nm, ln = C.c_char_p(), C.c_uint64()
            N.check(self.L.unc_index_seq(self.h, i, C.byref(nm), C.byref(ln)))
            self.seqs.append((nm.value.decode(), int(ln.value)))

    def kmer_ranges(self):
        st, en = np.zeros(1024, np.uint64), np.zeros(1024, np.uint64)
        a, b = C.c_uint64(), C.c_uint64()
        for k in range(1024):
            N.check(self.L.unc_index_kmer_range(self.h, k, C.byref(a), C.byref(b)))
            st[k], en[k] = a.value, b.value
        return st, en

    def thresholds(self):
        out = np.zeros(64, np.float32)
        N.check(self.L.unc_index_thresholds(self.h, out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def match_probs(self, event):
        out = np.zeros(1024, np.float32)
        N.check(self.L.unc_match_probs(self.h, float(event), out.ctypes.data))
        return out

    def neighbors(self, start, end, base):
        start = np.ascontiguousarray(start, np.uint64)
        end = np.ascontiguousarray(end, np.uint64)
        base = np.ascontiguousarray(base, np.uint8)
        os_, oe = np.zeros_like(start), np.zeros_like(start)
        N.check(self.L.unc_fm_neighbors(self.h, len(start), start.ctypes.data, end.ctypes.data, base.ctypes.data,
                                        os_.ctypes.data, oe.ctypes.data))
        return os_, oe

    def fm_step(self, start, end, want):
        """The mapper's backward step per entry: (ns, ne) of shape (n, 4) for all four bases, and the valid masks."""
        start = np.ascontiguousarray(start, np.uint64)
        end = np.ascontiguousarray(end, np.uint64)
        want = np.ascontiguousarray(want, np.uint8)
        ns, ne, valid = np.zeros((len(start), 4), np.uint64), np.zeros((len(start), 4), np.uint64), np.zeros_like(want)
        N.check(self.L.unc_fm_step(self.h, len(start), start.ctypes.data, end.ctypes.data, want.ctypes.data,
                                   ns.ctypes.data, ne.ctypes.data, valid.ctypes.data))
        return ns, ne, valid

    def sa(self, rows):
        rows = np.ascontiguousarray(rows, np.uint64)
        out = np.zeros_like(rows)
        N.check(self.L.unc_fm_sa(self.h, len(rows), rows.ctypes.data, out.ctypes.data))
        return out

    def close(self):
        if self.h:
            self.L.unc_index_free(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def make_descs(lens, dtype=0, cal=(1.0, 0.0, 1.0), offsets=None):
    lens = np.asarray(lens, dtype=np.uint32)
    d = np.zeros(len(lens), dtype=N.DESC_DTYPE)
    if offsets is None:
        offsets = np.concatenate([[0], np.cumsum(lens[:-1], dtype=np.uint64)]).astype(np.uint64)
    d["offset"] = offsets
    d["n_samples"] = lens
    d["dtype"] = dtype
    d["cal_range"], d["cal_offset"], d["cal_digit"] = cal
    return d


class BatchMapper:
    """unc_pool: the device side of MapPool (reference src/map_pool.cpp:28-69)."""

    def __init__(self, index, params=None, max_reads=4096, max_samples=None):
        self.L = N.lib()
        self.index = index
        self.params = params if params is not None else N.default_params()
        self.max_reads = int(max_reads)
        self.max_samples = int(max_samples if max_samples is not None else self.max_reads * 4000)
        self.h = C.c_void_p()
        N.check(self.L.unc_pool_create(index.h, C.byref(self.params), self.max_reads, self.max_samples, C.byref(self.h)))

    def map(self, samples, descs):
        """samples: contiguous numpy array (f32 pA or i16 raw) in HOST memory."""
        samples = np.ascontiguousarray(samples)
        out = np.zeros(len(descs), dtype=N.PAF_DTYPE)
        rc = self.L.unc_map_batch(self.h, descs.ctypes.data, len(descs), samples.ctypes.data, out.ctypes.data)
        self._last_rc = rc
        if rc != 0 and rc != -7:
            N.check(rc)
        return out

    def map_device(self, d_ptr, descs):
        """d_ptr: integer device pointer to the batch's samples (e.g. torch tensor .data_ptr())."""
        out = np.zeros(len(descs), dtype=N.PAF_DTYPE)
        rc = self.L.unc_map_batch_device(self.h, descs.ctypes.data, len(descs), C.c_void_p(int(d_ptr)), out.ctypes.data)
        self._last_rc = rc
        if rc != 0 and rc != -7:
            N.check(rc)
        return out

    def set_tie_order(self, mode):
        """0: equal children keep emission order (default kernel); 1: the reference's unstable pdqsort reproduced
        (exact-ties kernel; unc_pool_set_tie_order)."""
        N.check(self.L.unc_pool_set_tie_order(self.h, int(mode)))

    def map_ordered(self, samples, descs, carry=None, on_device=False):
        """The batch as ONE long-lived Mapper maps it, read after read (`uncalled map -t 1`; unc_map_batch_ordered).
        carry: 32 uint32 sources_added_ words the previous batch ended with (None = a new Mapper); returns
        (records, carry after the last read, reads mapped again, extra rounds)."""
        if on_device:
            ptr = C.c_void_p(int(samples))
        else:
            samples = np.ascontiguousarray(samples)
            ptr = C.c_void_p(samples.ctypes.data)
        carry = np.zeros(32, np.uint32) if carry is None else np.array(carry, dtype=np.uint32, copy=True)
        assert carry.shape == (32,)
        out = np.zeros(len(descs), dtype=N.PAF_DTYPE)
        nre, nro = C.c_uint32(), C.c_uint32()
        rc = self.L.unc_map_batch_ordered(self.h, descs.ctypes.data, len(descs), ptr, 1 if on_device else 0,
                                          carry.ctypes.data, out.ctypes.data, C.byref(nre), C.byref(nro))
        self._last_rc = rc
        if rc != 0 and rc != -7:
            N.check(rc)
        return out, carry, int(nre.value), int(nro.value)

    def submit(self, samples, descs, on_device=False):
        """First half of map()/map_device(): queue the batch on this pool's stream and return.  `samples`: host numpy
        array, or an integer device pointer with on_device=True; keep it (and `descs`) alive until wait()."""
        if on_device:
            ptr = C.c_void_p(int(samples))
        else:
            samples = np.ascontiguousarray(samples)
            ptr = C.c_void_p(samples.ctypes.data)
        self._pending = (samples, descs)
        N.check(self.L.unc_map_batch_submit(self.h, descs.ctypes.data, len(descs), ptr, 1 if on_device else 0))

    def wait(self):
        """Second half: block until the submitted batch is done; returns its records."""
        if getattr(self, "_pending", None) is None:
            raise N.UncError("no submitted batch to wait for")
        _, descs = self._pending
        out = np.zeros(len(descs), dtype=N.PAF_DTYPE)
        rc = self.L.unc_map_batch_wait(self.h, out.ctypes.data)
        self._pending = None
        self._last_rc = rc
        if rc != 0 and rc != -7:
            N.check(rc)
        return out

    def record(self, slot):
        """Mark event `slot` (0/1) at the current end of this pool's stream (device-side timing across pools)."""
        N.check(self.L.unc_pool_record(self.h, int(slot)))

    def elapsed_ms(self, slot, other, other_slot):
        """Milliseconds from this pool's event `slot` to `other`'s event `other_slot` (waits for both)."""
        ms = C.c_float()
        N.check(self.L.unc_pool_elapsed(self.h, int(slot), other.h, int(other_slot), C.byref(ms)))
        return float(ms.value)

    def events(self, samples, descs):
        samples = np.ascontiguousarray(samples)
        n = len(descs)
        stride = int(descs["n_samples"].max())
        ev = np.zeros((n, stride), np.float32)
        nm = np.zeros((n, stride), np.float32)
        ne = np.zeros(n, np.uint32)
        mel = np.zeros(n, np.float32)
        N.check(self.L.unc_events_batch(self.h, descs.ctypes.data, n, samples.ctypes.data, stride, ev.ctypes.data,
                                        nm.ctypes.data, ne.ctypes.data, mel.ctypes.data))
        return ev, nm, ne, mel

    def k1_stats(self):
        """(tiles, FSM re-run rounds, lanes re-run, reads redone serially) of the last batch's event detection."""
        a = (C.c_uint32 * 4)()
        N.check(self.L.unc_pool_k1_stats(self.h, a))
        return tuple(a)

    def timing(self):
        t = N.Timing()
        N.check(self.L.unc_pool_last_timing(self.h, C.byref(t)))
        return {k: getattr(t, k) for k, _ in N.Timing._fields_}

    def close(self):
        if self.h:
            self.L.unc_pool_free(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def paf_key(r):
    """Comparable PAF fields of one record (numpy void or ctypes struct)."""
    g = (lambda k: int(r[k])) if isinstance(r, np.void) else (lambda k: int(getattr(r, k)))
    if not g("mapped"):
        return (0, g("rd_len"), g("n_events"), g("events_used"))
    return tuple(g(k) for k in ("mapped", "fwd", "rid", "n_events", "events_used", "matches",
                                "rd_len", "rd_st", "rd_en", "rf_st", "rf_en", "rf_len"))
