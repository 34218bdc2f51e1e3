"""The signal front end of the mapper, event by event, from the GPU (include/unc_b200.h, `unc_events_*`).

What the mapper computes from a read's signal before it looks at the index, for every event of the whole signal:

* ``detect_events``: the reference's ``EventDetector::get_events`` (src/event_detector.cpp:114-127,296-319): start,
  length, mean and stdv of every event that passes the min_mean / max_mean filter;
* ``normalize``: the offline ``Normalizer`` the mapper applies to the event means (src/normalizer.cpp:31-44,114-118,
  src/mapper.cpp:193): scale, shift and the normalised means;
* ``annotate``: ``EventProfiler::get_full_mask`` and ``anno_event`` (src/event_profiler.hpp:71-151): the 25-event
  window's mean and stdv and the stall mask;
* ``match_probs``: ``PoreModel::match_prob`` of the mapper's model against all 1024 k-mers.

Every call is batched: it takes a list of reads and makes one pass over them on the device.  ``SignalProcessor``
keeps the device buffers between calls; the module-level functions use one processor per device and model.

Signals are float32 pA, or int16 DAC values with a (range, offset, digitisation) calibration per read, calibrated on
the device exactly as ``map`` does (src/read_buffer.cpp:239-242).  The whole signal is used (no max_events cap).
"""
import ctypes as C

import numpy as np

from . import _native as N

EVENT_DTYPE = np.dtype([("start", "<u4"), ("length", "<f4"), ("mean", "<f4"), ("stdv", "<f4")])
ANNO_DTYPE = np.dtype([("win_mean", "<f4"), ("win_stdv", "<f4"), ("win_mask", "?")])
# unc_event_full: one event and its annotations
FULL_DTYPE = np.dtype([("start", "<u4"), ("length", "<f4"), ("mean", "<f4"), ("stdv", "<f4"), ("norm_mean", "<f4"),
                       ("win_mean", "<f4"), ("win_stdv", "<f4"), ("win_mask", "<u4")])
# unc_event_read: per read
READ_DTYPE = np.dtype([("n_events", "<u4"), ("mean_event_len", "<f4"), ("norm_scale", "<f4"), ("norm_shift", "<f4")])

PARAM_NAMES = ("window_length1", "window_length2", "threshold1", "threshold2", "peak_height", "min_mean", "max_mean",
               "win_len", "win_stdv_min")


def default_params():
    """EventDetector::PRMS_DEF and EventProfiler::PRMS_DEF's win_len / win_stdv_min, as a dict."""
    p = N.EventParams()
    N.check(N.lib().unc_event_params_default(C.byref(p)))
    return {k: getattr(p, k) for k in PARAM_NAMES}


def _as_list(reads):
    """(list of reads, whether one read was given): any 1-D ndarray -- a signal, a list of means or an EVENT_DTYPE /
    FULL_DTYPE array of events -- is one read"""
    if isinstance(reads, np.ndarray) and reads.ndim == 1:
        return [reads], True
    return list(reads), False


def _means(m):
    """the event means of one read: the "mean" field of an events array, or the array itself"""
    if isinstance(m, np.ndarray) and m.dtype.names:
        return np.ascontiguousarray(m["mean"], np.float32)
    return np.ascontiguousarray(m, np.float32).ravel()


class EventBatch:
    """The result of SignalProcessor.run: ``reads`` (READ_DTYPE, one per read), ``events`` (FULL_DTYPE, read i's at
    ``events[offsets[i]:offsets[i + 1]]``)."""

    def __init__(self, reads, events):
        self.reads, self.events = reads, events
        self.offsets = np.zeros(len(reads) + 1, np.uint64)
        np.cumsum(reads["n_events"], out=self.offsets[1:])

    def __len__(self):
        return len(self.reads)

    def read(self, i):
        return self.events[int(self.offsets[i]):int(self.offsets[i + 1])]


class SignalProcessor:
    """unc_events: the detector, profiler and pore model on one device.  ``params`` overrides default_params();
    window lengths 3 / 6 and the 25-event profiler window are fixed (another value raises UncError)."""

    def __init__(self, model_path=None, device=0, **params):
        self.L = N.lib()
        unknown = set(params) - set(PARAM_NAMES)
        if unknown:
            raise TypeError("unknown parameter(s): " + ", ".join(sorted(unknown)))
        p = N.EventParams()
        N.check(self.L.unc_event_params_default(C.byref(p)))
        for k, v in params.items():
            setattr(p, k, v)
        self.params = {k: getattr(p, k) for k in PARAM_NAMES}
        N.check(self.L.unc_init(int(device)))
        self.h = C.c_void_p()
        N.check(self.L.unc_events_create((model_path or N.MODEL_TABLE).encode(), C.byref(p), C.byref(self.h)))
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.L.unc_events_free(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def stage(signals, calibration=None):
        """(flat samples, descriptors) of a list of signals, as unc_map_batch takes them"""
        sigs, _ = _as_list(signals)
        if not sigs:
            return np.zeros(1, np.float32), np.zeros(0, N.DESC_DTYPE)
        i16 = sigs[0].dtype == np.int16
        if any((s.dtype == np.int16) != i16 for s in sigs):
            raise ValueError("all signals of a batch are float32 pA or all are int16 DAC values")
        if i16 and calibration is None:
            raise ValueError("int16 signals need a (range, offset, digitisation) calibration per read")
        flat = np.concatenate([np.asarray(s, np.int16 if i16 else np.float32).ravel() for s in sigs] + [np.zeros(0, np.int16 if i16 else np.float32)])
        descs = np.zeros(len(sigs), N.DESC_DTYPE)
        lens = np.array([len(s) for s in sigs], np.uint64)
        if lens.size and lens.max() >= 1 << 32:
            raise ValueError("a read of 2^32 samples or more")
        descs["offset"][1:] = np.cumsum(lens)[:-1]
        descs["n_samples"] = lens
        descs["dtype"] = 1 if i16 else 0
        if i16:
            cal = np.asarray(calibration, np.float32).reshape(len(sigs), 3)
            descs["cal_range"], descs["cal_offset"], descs["cal_digit"] = cal[:, 0], cal[:, 1], cal[:, 2]
        else:
            descs["cal_range"], descs["cal_digit"] = 1.0, 1.0
        return np.ascontiguousarray(flat), descs

    def run(self, signals, calibration=None, fetch=True):
        """Detection, normaliser and profiler over every read: an EventBatch (events None when fetch is False; they
        then stay on the device, which is what a device-resident timing measures)."""
        flat, descs = self.stage(signals, calibration)
        return self.run_staged(flat, descs, fetch)

    def run_staged(self, flat, descs, fetch=True, on_device=False):
        """run() on samples already staged by stage(); on_device: `flat` is a device pointer (int) on this device"""
        n = len(descs)
        reads = np.zeros(n, READ_DTYPE)
        ptr = C.c_void_p(int(flat)) if on_device else C.c_void_p(flat.ctypes.data)
        N.check(self.L.unc_events_run(self.h, descs.ctypes.data, n, ptr, 1 if on_device else 0, reads.ctypes.data))
        if not fetch:
            return EventBatch(reads, None)
        events = np.zeros(int(reads["n_events"].sum(dtype=np.uint64)), FULL_DTYPE)
        if len(events):
            N.check(self.L.unc_events_fetch(self.h, events.ctypes.data))
        return EventBatch(reads, events)

    def last_times(self):
        """CUDA-event times of the last run in ms: h2d, detect, annotate (normaliser + profiler), d2h"""
        ms = (C.c_float * 4)()
        N.check(self.L.unc_events_last_times(self.h, ms))
        return dict(zip(("h2d", "detect", "annotate", "d2h"), (float(x) for x in ms)))

    def detect_events(self, signals, calibration=None):
        """EventDetector::get_events of each read: a list of EVENT_DTYPE arrays (one array for one signal)"""
        sigs, one = _as_list(signals)
        b = self.run(sigs, calibration)
        out = [_project(b.read(i), EVENT_DTYPE) for i in range(len(b))]
        return out[0] if one else out

    def _annotate(self, means_list):
        means_list = [_means(m) for m in means_list]
        n = len(means_list)
        off = np.zeros(n + 1, np.uint64)
        off[1:] = np.cumsum([len(m) for m in means_list])
        flat = np.ascontiguousarray(np.concatenate(means_list + [np.zeros(0, np.float32)]))
        tot = int(off[-1])
        nm, wm, ws = (np.zeros(tot, np.float32) for _ in range(3))
        mask = np.zeros(tot, np.uint32)
        sc, sh = np.zeros(n, np.float32), np.zeros(n, np.float32)
        N.check(self.L.unc_events_annotate(self.h, n, off.ctypes.data, flat.ctypes.data, nm.ctypes.data, wm.ctypes.data,
                                           ws.ctypes.data, mask.ctypes.data, sc.ctypes.data, sh.ctypes.data))
        return off, nm, wm, ws, mask, sc, sh

    def annotate(self, events):
        """EventProfiler::get_full_mask with anno_event's window statistics over each read's events (EVENT_DTYPE arrays
        or arrays of means): a list of ANNO_DTYPE arrays.  win_mean / win_stdv are NaN for the events that never become
        the profiler's next event (the last ones of a read)."""
        lst, one = _as_list(events)
        off, _, wm, ws, mask, _, _ = self._annotate(lst)
        out = []
        for i in range(len(lst)):
            a, b = int(off[i]), int(off[i + 1])
            r = np.zeros(b - a, ANNO_DTYPE)
            r["win_mean"], r["win_stdv"], r["win_mask"] = wm[a:b], ws[a:b], mask[a:b] != 0
            out.append(r)
        return out[0] if one else out

    def normalize(self, means):
        """The offline Normalizer towards the model's mean and stdv over each read's event means (EVENT_DTYPE arrays or
        arrays of means): a list of (scale, shift, normalised means); scale = shift = 0 for a read without events."""
        lst, one = _as_list(means)
        off, nm, _, _, _, sc, sh = self._annotate(lst)
        out = [(float(sc[i]), float(sh[i]), nm[int(off[i]):int(off[i + 1])]) for i in range(len(lst))]
        return out[0] if one else out

    def match_probs(self, means):
        """PoreModel::match_prob of the mapper's model: a [len(means), 1024] float32 array, k-mer k in column k (the
        index unc_match_probs uses)"""
        m = np.ascontiguousarray(np.asarray(means, np.float32).ravel())
        out = np.zeros((len(m), 1024), np.float32)
        if len(m):
            N.check(self.L.unc_match_probs_batch(self.h, m.ctypes.data, len(m), out.ctypes.data))
        return out


def _project(a, dtype):
    r = np.zeros(len(a), dtype)
    for k in dtype.names:
        r[k] = a[k]
    return r


_default = {}


def processor(device=0, model_path=None):
    """The module's SignalProcessor with default parameters for this device and model."""
    key = (int(device), model_path)
    if key not in _default:
        _default[key] = SignalProcessor(model_path=model_path, device=device)
    return _default[key]


def detect_events(signals, calibration=None, device=0, model_path=None):
    return processor(device, model_path).detect_events(signals, calibration)


def annotate(events, device=0, model_path=None):
    return processor(device, model_path).annotate(events)


def normalize(means, device=0, model_path=None):
    return processor(device, model_path).normalize(means)


def match_probs(means, device=0, model_path=None):
    return processor(device, model_path).match_probs(means)


def process(signals, calibration=None, device=0, model_path=None):
    """Everything at once: an EventBatch."""
    return processor(device, model_path).run(signals, calibration)


for _f, _m in ((detect_events, "detect_events"), (annotate, "annotate"), (normalize, "normalize"),
               (match_probs, "match_probs")):
    _f.__doc__ = getattr(SignalProcessor, _m).__doc__
