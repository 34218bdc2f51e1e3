"""Streaming path over the C-ABI (unc_stream_create / unc_stream_step / unc_stream_free in
include/unc_b200.h): chunks of many channels with persistent per-channel state on the device --
what RealtimePool does with one Mapper per channel (reference src/realtime_pool.cpp:38-139,316-360,
src/mapper.cpp:210-431).  No mapping logic lives here; `feed_reads` is only the chunk-feeding policy
(next chunk of a channel once the previous one is mapped, an empty chunk when the signal is exhausted)
that the reference's simulator applies (ReadBuffer::get_chunks cuts full chunks, src/read_buffer.cpp:319-332).
"""
import ctypes as C

import numpy as np

from . import _native as N

MAPPING, SUCCESS, FAILURE = 1, 2, 3


class ChunkDesc(C.Structure):
    """unc_chunk_desc"""
    _fields_ = [("channel", C.c_uint32), ("new_read", C.c_uint32), ("offset", C.c_uint64), ("n_samples", C.c_uint32),
                ("dtype", C.c_uint32), ("cal_range", C.c_float), ("cal_offset", C.c_float), ("cal_digit", C.c_float)]


class StreamResult(C.Structure):
    """unc_stream_result"""
    _fields_ = [("state", C.c_int32), ("ended", C.c_int32), ("chunks", C.c_uint32), ("pad_", C.c_uint32),
                ("rec", N.PafRec)]


class ReplayRead(C.Structure):
    """unc_replay_read"""
    _fields_ = [("channel", C.c_uint32), ("number", C.c_uint32), ("offset", C.c_uint64), ("n_samples", C.c_uint64),
                ("dtype", C.c_uint32), ("cal_range", C.c_float), ("cal_offset", C.c_float), ("cal_digit", C.c_float)]


class ReplayResult(C.Structure):
    """unc_replay_result"""
    _fields_ = [("read", C.c_uint32), ("number", C.c_uint32), ("step", C.c_uint64), ("kind", C.c_uint32),
                ("pad_", C.c_uint32), ("res", StreamResult)]


def feed_reads(step, n_channels, signals, chunk_len, max_chunks=1000000):
    """Drives `step(descs, n, flat_samples, results)` like a flow cell: read i sits on channel i % n_channels
    (reads sharing a channel follow each other); every round each active channel gets its next FULL chunk, and
    an empty chunk once its signal (or max_chunks) is exhausted.  Returns, per read, (state, ended, chunks, rec)
    or None for a read shorter than one chunk (it never reaches the mapper)."""
    queues = [[] for _ in range(n_channels)]
    for i in range(len(signals)):
        queues[i % n_channels].append(i)
    cur = [None] * n_channels            # [read index, next chunk]
    done = {}
    while True:
        descs, parts, owners = [], [], []
        off = 0
        for c in range(n_channels):
            while cur[c] is None and queues[c]:
                i = queues[c].pop(0)
                if len(signals[i]) // chunk_len == 0 or max_chunks == 0:
                    done[i] = None
                else:
                    cur[c] = [i, 0]
            if cur[c] is None:
                continue
            i, k = cur[c]
            s = signals[i]
            nfull = min(len(s) // chunk_len, max_chunks)
            d = ChunkDesc()
            d.channel, d.new_read, d.offset, d.dtype = c, 1 if k == 0 else 0, off, 0
            d.cal_range, d.cal_offset, d.cal_digit = 1.0, 0.0, 1.0
            if k < nfull:
                d.n_samples = chunk_len
                parts.append(np.ascontiguousarray(s[k * chunk_len:(k + 1) * chunk_len], np.float32))
                off += chunk_len
            else:
                d.n_samples = 0
            descs.append(d)
            owners.append(c)
        if not descs:
            break
        arr = (ChunkDesc * len(descs))(*descs)
        flat = np.concatenate(parts) if parts else np.zeros(1, np.float32)
        res = (StreamResult * len(descs))()
        step(arr, len(descs), flat, res)
        for c, r in zip(owners, res):
            cur[c][1] += 1
            if r.state != MAPPING:
                done[cur[c][0]] = (r.state, r.ended, r.chunks, N.PafRec.from_buffer_copy(bytes(r.rec)))
                cur[c] = None
    return [done.get(i) for i in range(len(signals))]


class StreamMapper:
    """unc_stream: one persistent device-side mapper state per channel."""

    def __init__(self, index, n_channels, chunk_len, max_chunks=1000000, params=None):
        self.L = N.lib()
        self.index, self.n_channels, self.chunk_len, self.max_chunks = index, int(n_channels), int(chunk_len), int(max_chunks)
        self.params = params if params is not None else N.default_params()
        self.h = C.c_void_p()
        N.check(self.L.unc_stream_create(index.h, C.byref(self.params), self.n_channels, self.chunk_len,
                                         self.max_chunks, C.byref(self.h)))

    def set_tie_order(self, mode):
        """1: the reference's unstable child sort reproduced (exact-ties kernel), 0: emission order (default)."""
        N.check(self.L.unc_stream_set_tie_order(self.h, int(mode)))

    def set_chunk_timeout(self, ms):
        """Mapper::PRMS.chunk_timeout (reference src/mapper.cpp:40,384-390): reads still mapping after a step that took
        longer than `ms` of wall-clock time fail and are marked ended.  Off until set."""
        N.check(self.L.unc_stream_set_chunk_timeout(self.h, float(ms)))

    def last_step_ms(self):
        """Wall-clock time of the last step (copies included): the decision latency of its chunks."""
        return float(self.L.unc_stream_last_step_ms(self.h))

    def norm_state(self, channel):
        """The channel's streaming normaliser after the last step: (mean, varsum, n, wr), n being the events in its
        window (at most 6000) and wr its ring cursor."""
        m, v, n, w = C.c_double(), C.c_double(), C.c_uint32(), C.c_uint32()
        N.check(self.L.unc_stream_channel_norm(self.h, int(channel), C.byref(m), C.byref(v), C.byref(n), C.byref(w)))
        return m.value, v.value, n.value, w.value

    def step(self, descs, n, flat, res):
        flat = np.ascontiguousarray(flat)
        rc = self.L.unc_stream_step(self.h, descs, n, flat.ctypes.data, res)
        if rc != 0 and rc != -7:
            N.check(rc)

    def replay(self, reads, n, flat, out):
        """unc_stream_replay: a window of whole reads (ReplayRead array) run to completion on the device; `out` (ReplayResult
        array of n) receives them in completion order.  Returns 0 or UNC_E_OVERFLOW (-7, reported per read in
        rec.status); other errors raise."""
        flat = np.ascontiguousarray(flat)
        rc = self.L.unc_stream_replay(self.h, reads, n, flat.ctypes.data, out)
        if rc != 0 and rc != -7:
            N.check(rc)
        return rc

    def map_reads(self, signals):
        """Streams whole reads through the channels (feed_reads policy); one result per read."""
        return feed_reads(self.step, self.n_channels, signals, self.chunk_len, self.max_chunks)

    def close(self):
        if self.h:
            self.L.unc_stream_free(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
