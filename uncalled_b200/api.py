"""Host-side mirror of the reference's Python surface for the map path: `Conf`, `Paf`, `MapPool`
(what `_uncalled` exports through reference src/pybinder.cpp:14-91 and what `scripts/uncalled
map` drives, scripts/uncalled:127-167).

Same names, argument meaning and error behaviour; every mapping result comes from the CUDA
kernels behind include/unc_b200.h (uncalled_b200/libunc_b200.so).  There is no CPU fallback:
constructing a MapPool without a usable CUDA device raises UncError.

Differences a caller can observe (documented, not hidden):
  * `MapPool(conf)` maps batches on the GPU instead of one read per CPU thread; `conf.threads`
    is accepted and ignored by the mapper (reference src/map_pool.cpp:31).
    `conf.exact_ties = 1` (CLI `--exact-ties`) selects the kernel that reproduces the reference's unstable child sort
    (DESIGN.md section 2, divergence 1); with both switches the output is the unmodified reference's `-t 1` output.
    `conf.ordered = 1` (CLI `--ordered`) reproduces what the reference prints with ONE thread for a multi-read
    input: reads mapped in input order by one long-lived Mapper (DESIGN.md section 2, divergence 2).
  * fast5 files are read by the library's own HDF5 subset reader (uncalled_b200/csrc/unc_fast5.cpp; the
    reference vendors libhdf5).  VBZ-compressed files are rejected with a clear error (the reference's
    vendored libhdf5 cannot read them either without an external plugin).  Reads can also be queued as
    arrays with `add_read()`, which is what `Fast5Reader` hands to `MapPool::update` after decoding
    (reference src/read_buffer.cpp:160-246).
"""
import enum
import sys
import time

import numpy as np

from . import _native as N
from .mapper import BatchMapper, Index, make_descs


class Conf:
    """reference src/conf.hpp:296-340 -- the attributes `uncalled map` sets (uncalled/args.py:296-302).
    They are real properties so that `Conf.<name>.__doc__` works as uncalled/args.py:223-260 expects."""

    _FIELDS = {
        # name: (default, doc)           defaults: src/mapper.cpp:29-52, read_buffer.cpp:26-32, fast5_reader.cpp:26-31
        "threads": (1, "Number of threads (the GPU mapper has no CPU mapping threads; used as fast5 decoding threads)"),
        "bwa_prefix": ("", "BWA prefix to map to"),
        "idx_preset": ("default", "Mapping mode preset line of the .uncl file"),
        "model_path": ("", "k-mer model file (empty: built-in r9.4 5-mer template model)"),
        "max_events": (30000, "Will give up on a read after this many events have been processed"),
        "seed_len": (22, "Seed length in events"),
        "max_paths": (10000, "Maximum number of paths to consider per event"),
        "chunk_time": (1.0, "Length of chunks in seconds"),
        "max_chunks": (1000000, "Will give up on a read after this many chunks have been processed"),
        "sample_rate": (4000.0, "Raw samples per second"),
        "bp_per_sec": (450.0, "Expected bases sequenced per second"),
        "num_channels": (512, "Number of channels used in sequencing"),
        "fast5_list": ("", "File containing a list of paths to fast5 files, one per line"),
        "read_list": ("", "Only map reads listed in this file"),
        "max_reads": (0, "Maximum number of reads to map"),
        "max_buffer": (100, "Maximum number of reads to store in memory"),
        "realtime_mode": (0, "RealtimePool.DEPLETE or RealtimePool.ENRICH"),
        "active_chs": (0, "RealtimePool.FULL, EVEN or ODD"),
        "host": ("127.0.0.1", "MinKNOW host address"),
        "port": (8000, "MinKNOW port"),
        "duration": (72.0, "Duration to map real-time run in hours"),
        "max_active_reads": (512, "Maximum number of reads being mapped at once"),
        "min_active_reads": (0, "map-ord: stop once fewer channels than this have a read in progress after a step "
                                "(0: never)"),
        "device": (0, "CUDA device of this process (one process per GPU)"),
        "batch_reads": (4096, "Reads per GPU batch"),
        "exact_ties": (0, "1: children that compare equal in the per-event sort are ordered exactly as the reference's "
                          "unstable pdqsort orders them (exact-ties kernel, slower); 0: emission order (default)"),
        "ordered": (0, "1: map the reads in input order as ONE long-lived Mapper does, i.e. exactly what the reference "
                       "prints with `-t 1` (a read inherits the source flags its predecessor left set); "
                       "0: every read is mapped by a new Mapper (batch order free, fastest)"),
        # read-until simulator (`uncalled sim`); defaults: the [simulator] section of the reference's conf/defaults.toml
        "ctl_seqsum": ("", "Sequencing summary of the control run whose reads are replayed"),
        "unc_seqsum": ("", "Sequencing summary of the UNCALLED run that gives the channel activity pattern"),
        "unc_paf": ("", "PAF of the UNCALLED run (its ej/ub tags give the eject delay)"),
        "sim_speed": (1.0, "Scale factor applied to the scan interval boundaries"),
        "scan_time": (10.0, "Length of a simulated mux scan in seconds"),
        "scan_intv_time": (5400.0, "Time between mux scans in seconds"),
        "ej_time": (0.1, "Extra gap after an ejected read in seconds"),
        "min_ch_reads": (10, "Minimum number of control reads given to a channel that had reads in the UNCALLED run"),
    }

    def __init__(self):
        self._v = {k: d for k, (d, _) in self._FIELDS.items()}


def _conf_prop(name, doc):
    def g(self):
        return self._v[name]

    def s(self, val):
        self._v[name] = type(Conf._FIELDS[name][0])(val)
    return property(g, s, doc=doc)


for _n, (_d, _doc) in Conf._FIELDS.items():
    setattr(Conf, _n, _conf_prop(_n, _doc))


class Paf:
    """reference src/read_buffer.hpp:40-128, src/read_buffer.cpp:34-155."""

    class Tag(enum.IntEnum):
        MAP_TIME = 0
        WAIT_TIME = 1
        QUEUE_TIME = 2
        RECEIVE_TIME = 3
        CHANNEL = 4
        EJECT = 5
        READ_START = 6
        IN_SCAN = 7
        TOP_RATIO = 8
        MEAN_RATIO = 9
        ENDED = 10
        KEEP = 11
        DELAY = 12
        SEED_CLUSTER = 13
        CONFIDENT_EVENT = 14

    PAF_TAGS = ["mt", "wt", "qt", "rt", "ch", "ej", "st", "mx", "tr", "mr", "en", "kp", "dl", "sc", "ce"]

    def __init__(self, rd_name="", channel=None, start_sample=None):
        self.rd_name, self.rf_name = rd_name, ""
        self._mapped = self._ended = False
        self.rd_st = self.rd_en = self.rd_len = self.rf_st = self.rf_en = self.rf_len = 0
        self.fwd, self.matches = False, 0
        self.int_tags, self.float_tags, self.str_tags = [], [], []
        if channel is not None:                         # Paf(rd_name, channel, start_sample), :66-82
            self.set_int(Paf.Tag.CHANNEL, channel)
            self.set_int(Paf.Tag.READ_START, start_sample or 0)

    def is_mapped(self):
        return self._mapped

    def is_ended(self):
        return self._ended

    def set_read_len(self, n):
        self.rd_len = int(n)

    def set_mapped(self, rd_st, rd_en, rf_name, rf_st, rf_en, rf_len, fwd, matches):
        self._mapped = True
        self.rd_st, self.rd_en, self.rf_name = int(rd_st), int(rd_en), rf_name
        self.rf_st, self.rf_en, self.rf_len = int(rf_st), int(rf_en), int(rf_len)
        self.fwd, self.matches = bool(fwd), int(matches) & 0xFFFF

    def set_int(self, t, v):
        self.int_tags.append((int(t), int(v)))

    def set_float(self, t, v):
        self.float_tags.append((int(t), float(np.float32(v))))

    def set_str(self, t, v):
        self.str_tags.append((int(t), str(v)))

    def fields(self):
        """The 12 PAF columns as strings (src/read_buffer.cpp:92-126)."""
        f = [self.rd_name, str(self.rd_len)]
        if self._mapped:
            f += [str(self.rd_st), str(self.rd_en), "+" if self.fwd else "-", self.rf_name, str(self.rf_len),
                  str(self.rf_st), str(self.rf_en), str(self.matches), str(self.rf_en - self.rf_st + 1), "255"]
        else:
            f += ["*"] * 9 + ["255"]
        return f

    def line(self):
        f = self.fields()
        f += ["%s:i:%d" % (self.PAF_TAGS[t], v) for t, v in self.int_tags]
        f += ["%s:f:%.6f" % (self.PAF_TAGS[t], v) for t, v in self.float_tags]      # std::fixed
        f += ["%s:Z:%s" % (self.PAF_TAGS[t], v) for t, v in self.str_tags]
        return "\t".join(f)

    def print_paf(self, file=None):
        (file or sys.stdout).write(self.line() + "\n")


# export the enum values into class scope like pybind11's export_values() (read_buffer.hpp:104-112)
for _t in Paf.Tag:
    setattr(Paf, _t.name, _t)


def _paf_from_rec(seqs, rec, read_id, channel, start):
    """Paf as Mapper::set_ref_loc / set_failed leave it (reference src/mapper.cpp:365-372,708-728)."""
    g = (lambda k: rec[k]) if isinstance(rec, np.void) else (lambda k: getattr(rec, k))
    p = Paf(read_id, channel, start)
    p.set_read_len(int(g("rd_len")))
    if g("mapped"):
        rid = int(g("rid"))
        name = seqs[rid][0] if 0 <= rid < len(seqs) else ""
        p.set_mapped(g("rd_st"), g("rd_en"), name, g("rf_st"), g("rf_en"), g("rf_len"), bool(g("fwd")), int(g("matches")))
    return p


class _Read:
    __slots__ = ("id", "channel", "number", "start", "signal", "dtype", "cal")

    def __init__(self, rid, signal, channel, number, start, dtype, cal):
        self.id, self.signal, self.channel, self.number, self.start = rid, signal, channel, number, start
        self.dtype, self.cal = dtype, cal


class MapPool:
    """reference src/map_pool.hpp:33-53: MapPool(conf), add_fast5, update() -> [Paf], running(), stop()."""

    def __init__(self, conf, backend=None, index=None):
        """`backend` (tests): an object with map(samples, descs) -> records standing in for the GPU BatchMapper,
        with `index.seqs` = [(name, length)]; by default the index is loaded onto conf.device."""
        self.conf = conf
        self._backend = backend
        if backend is None:
            if not conf.bwa_prefix:
                raise RuntimeError("Conf.bwa_prefix is not set")
            index = Index(conf.bwa_prefix, preset=conf.idx_preset, device=conf.device,
                          model_table=conf.model_path or None)
        self.index = index
        p = N.default_params()
        p.max_events, p.max_paths, p.seed_len = conf.max_events, conf.max_paths, conf.seed_len
        p.bp_per_sec, p.sample_rate = conf.bp_per_sec, conf.sample_rate
        self.params = p
        self._queue = []
        self._mappers, self._caps, self._inflight = [None, None], [(0, 0), (0, 0)], None   # two pools: batches overlap
        self._n_added, self._stopped = 0, False
        self.n_overflowed = 0                                 # reads whose device workspace overflowed (warned about, reported unmapped)
        self._carry = None                                    # conf.ordered: sources_added_ words after the last read mapped
        self._files, self._open, self._next = [], None, 0
        self._future, self._executor = None, None          # fast5 decoding of the NEXT batch overlaps the mapping
        if conf.fast5_list:                                   # Fast5Reader::load_fast5_list (src/fast5_reader.cpp:77-92)
            self._files = [l.rstrip("\n") for l in open(conf.fast5_list) if l.strip()]
        self._read_filter = None
        if conf.read_list:
            self._read_filter = set(l.strip() for l in open(conf.read_list) if l.strip())

    # -- input ---------------------------------------------------------------------------
    def _max_len(self):
        # the fast5 constructor truncates the signal to max_chunks * chunk_len samples
        # (reference src/read_buffer.cpp:229-234; chunk_len = chunk_time * sample_rate, read_buffer.hpp:135-137)
        chunk_len = int(np.float32(self.conf.chunk_time) * np.float32(self.conf.sample_rate)) & 0xFFFF   # chunk_len() returns u16
        return int(self.conf.max_chunks) * chunk_len

    def add_read(self, read_id, signal, channel=0, number=0, start_sample=0, calibration=None):
        """Queue one read.  signal: float32 pA, or int16 DAC values with calibration=(range, offset, digitisation)
        (calibrated on the device exactly as reference src/read_buffer.cpp:239-242)."""
        if self._read_filter is not None and read_id not in self._read_filter:
            return False
        if self.conf.max_reads and self._n_added >= self.conf.max_reads:
            return False
        sig = np.asarray(signal)
        if calibration is None:
            sig, dtype, cal = np.ascontiguousarray(sig, np.float32), 0, (1.0, 0.0, 1.0)
        else:
            if sig.dtype != np.int16:
                raise TypeError("calibration given: the signal must be int16 DAC values")
            sig, dtype, cal = np.ascontiguousarray(sig), 1, tuple(float(np.float32(x)) for x in calibration)
        sig = sig[:self._max_len()]
        self._queue.append(_Read(read_id, sig, int(channel), int(number), int(start_sample), dtype, cal))
        self._n_added += 1
        return True

    def add_fast5(self, fast5_name):
        """Fast5Reader::add_fast5 (src/fast5_reader.cpp:73-75): the file is queued and read when update() needs
        reads.  A file that cannot be read raises RuntimeError from update(), as the reference's reader throws
        from its fill_buffer()."""
        self._files.append(fast5_name)

    def _decode_next(self, want):
        """Fast5Reader::fill_buffer (src/fast5_reader.cpp:179-229): decode up to `want` reads from the pending
        files (conf.threads host threads inside unc_fast5_load).  Runs on the prefetch thread while the GPU maps."""
        from .fast5 import Fast5File
        out = []
        while len(out) < want and (self._open is not None or self._files):
            if self._open is None:
                self._open, self._next = Fast5File(self._files.pop(0)), 0
            f = self._open
            n = min(want - len(out), f.n_reads - self._next)
            out += f.load(self._next, n, max_samples_per_read=self._max_len(), threads=self.conf.threads)
            self._next += n
            if self._next >= f.n_reads:
                f.close()
                self._open = None
        return out

    def _files_pending(self):
        if self.conf.max_reads and self._n_added >= self.conf.max_reads:      # Fast5Reader::all_buffered
            if self._open is not None:
                self._open.close()
            self._files, self._open = [], None
        return self._open is not None or len(self._files) > 0

    def _queue_decoded(self, reads):
        for r in reads:
            self.add_read(r.read_id, r.signal, r.channel, r.number, r.start_sample, calibration=r.calibration)

    def _fill_from_fast5(self):
        want = self.conf.batch_reads
        if self._future is not None:                     # decoded while the previous batch was on the GPU
            fut, self._future = self._future, None
            self._queue_decoded(fut.result())
        while len(self._queue) < want and self._files_pending():
            self._queue_decoded(self._decode_next(want - len(self._queue)))
        if self._files_pending():                        # start on the next batch before this one is mapped
            if self._executor is None:
                from concurrent.futures import ThreadPoolExecutor
                self._executor = ThreadPoolExecutor(max_workers=1)
            self._future = self._executor.submit(self._decode_next, want)

    # -- output --------------------------------------------------------------------------
    def _take_batch(self):
        """The leading reads of one sample type, at most conf.batch_reads (a device batch has one sample type)."""
        if not self._queue:
            return None
        dtype, n = self._queue[0].dtype, 0
        while n < len(self._queue) and n < self.conf.batch_reads and self._queue[n].dtype == dtype:
            n += 1
        batch = self._queue[:n]
        del self._queue[:n]
        return batch

    def _mapper_for(self, slot, n_reads, total):
        if self._backend is not None:
            return self._backend
        m, cap = self._mappers[slot], self._caps[slot]
        if m is None or n_reads > cap[0] or total > cap[1]:
            cap = (max(n_reads, cap[0], 64), max(total, cap[1], 1 << 20))
            if m is not None:
                m.close()
            m = BatchMapper(self.index, params=self.params, max_reads=cap[0], max_samples=cap[1])
            if self.conf.exact_ties:
                m.set_tie_order(1)
            self._mappers[slot], self._caps[slot] = m, cap
        return m

    def _launch(self, batch):
        """Put a batch on the GPU (unc_map_batch_submit on the pool that is not in flight) and return at once.
        The CTAs take reads from the batch in order, so the longest signals go first: the batch then ends on short
        reads instead of leaving most SMs idle behind one long read (results are matched by read, not by position)."""
        ordered = bool(self.conf.ordered)
        if not ordered:
            batch.sort(key=lambda r: -len(r.signal))
        lens = [len(r.signal) for r in batch]
        total = int(sum(lens))
        dtype = batch[0].dtype
        d = make_descs(lens, dtype=dtype)
        for i, r in enumerate(batch):              # descriptors carry the calibration per read
            d["cal_range"][i], d["cal_offset"][i], d["cal_digit"][i] = r.cal
        flat = np.concatenate([r.signal for r in batch]) if total else np.zeros(1, np.float32 if dtype == 0 else np.int16)
        slot = 1 - self._inflight["slot"] if self._inflight is not None else 0
        m = self._mapper_for(slot, len(batch), total)
        job = {"slot": slot, "batch": batch, "flat": flat, "descs": d, "t0": time.time(), "mapper": m, "recs": None}
        if ordered:
            # one Mapper, read after read (reference src/map_pool.cpp:104-158 with one thread): the chain through the
            # flags is resolved inside unc_map_batch_ordered; batches follow each other, linked by the carry
            job["recs"], self._carry, _, _ = m.map_ordered(flat, d, carry=self._carry)
        elif hasattr(m, "submit"):
            m.submit(flat, d)
        else:                                      # a test backend without the two-call form
            job["recs"] = m.map(flat, d)
        return job

    def _collect(self, job):
        recs = job["recs"] if job["recs"] is not None else job["mapper"].wait()
        batch = job["batch"]
        ms = (time.time() - job["t0"]) * 1e3 / len(batch)
        out = []
        for r, rec in zip(batch, recs):
            if int(rec["status"] if isinstance(rec, np.void) else rec.status) != 0:
                # the read overflowed its per-read device workspace (seed rows of one event / cluster blocks): its record
                # is an unmapped one, and that must not pass silently -- the reference would have gone on mapping it
                self.n_overflowed += 1
                sys.stderr.write("Warning: read %s overflowed its device workspace (status %d); reported unmapped\n"
                                 % (r.id, int(rec["status"] if isinstance(rec, np.void) else rec.status)))
            p = _paf_from_rec(self.index.seqs, rec, r.id, r.channel, r.start)
            p.set_float(Paf.Tag.MAP_TIME, ms)
            out.append(p)
        return out

    def update(self):
        """Returns the Paf records that are ready (the reference returns whatever its threads finished since the
        last call, src/map_pool.cpp:45-69).  Batches of conf.batch_reads reads are mapped on the GPU; when more input
        is waiting, the next batch is submitted (on a second pool) BEFORE the call waits for the one in flight, so that
        its CTAs fill the SMs which the tail of the previous batch leaves idle, and fast5 decoding runs alongside."""
        if self._stopped:
            return []
        self._fill_from_fast5()
        nxt = self._take_batch()
        job = self._launch(nxt) if nxt else None
        out = []
        if self._inflight is not None:
            out = self._collect(self._inflight)
            self._inflight = None
        if job is not None:
            more = bool(self._queue) or self._future is not None or self._open is not None or bool(self._files)
            if more:
                self._inflight = job               # collected by the next call, after that call's submit
            else:
                out += self._collect(job)
        return out

    def running(self):
        return not self._stopped and (len(self._queue) > 0 or self._inflight is not None or self._future is not None or
                                      self._open is not None or len(self._files) > 0)

    def stop(self):
        self._stopped = True
        if self._inflight is not None:
            try:
                self._collect(self._inflight)
            except Exception:
                pass
            self._inflight = None
        if self._future is not None:
            try:
                self._future.result()
            except Exception:
                pass
            self._future = None
        if self._executor is not None:
            self._executor.shutdown(wait=True)
            self._executor = None
        if self._open is not None:
            self._open.close()
            self._open = None
        for i, m in enumerate(self._mappers):
            if m is not None:
                m.close()
            self._mappers[i] = None


class Chunk:
    """reference src/chunk.hpp:33-81 (the vector<float> constructor form and the accessors pybind exports).
    With `calibration=(range, offset, digitisation)` the samples are int16 DAC values, kept as they are and
    calibrated on the device when RealtimePool maps them."""

    def __init__(self, read_id="", channel=1, number=0, start=0, raw_data=(), raw_st=0, raw_len=None, calibration=None):
        if calibration is None:
            raw, self.dtype, self.cal = np.asarray(raw_data, dtype=np.float32), 0, (1.0, 0.0, 1.0)
        else:
            raw = np.asarray(raw_data)
            if raw.dtype != np.int16:
                raise TypeError("calibration given: the samples must be int16 DAC values")
            self.dtype, self.cal = 1, tuple(float(np.float32(x)) for x in calibration)
        if raw_len is None:
            raw_len = len(raw) - raw_st
        if raw_st + raw_len > len(raw):                   # Chunk::Chunk clips to the signal (src/chunk.cpp:74-83)
            raw_len = len(raw) - raw_st
        self.id, self.channel, self.number, self.start = read_id, int(channel), int(number), int(start)
        self._raw = np.ascontiguousarray(raw[raw_st:raw_st + raw_len])

    def size(self):
        return len(self._raw)

    def empty(self):
        return len(self._raw) == 0

    def pop(self):
        r, self._raw = self._raw, np.zeros(0, self._raw.dtype)
        return r

    def swap(self, other):
        self.__dict__, other.__dict__ = other.__dict__, self.__dict__

    def print(self):
        for v in self._raw:
            print(v)


class RealtimePool:
    """reference src/realtime_pool.hpp:33-91: RealtimePool(conf), add_chunk, try_add_chunk, update() ->
    [(channel, read number, Paf)], all_finished(), stop_all(), and the mode constants the CLI parser needs
    (uncalled/args.py:160-187).  One persistent device-side mapper state per channel (StreamMapper) replaces
    the per-channel Mapper objects and the worker threads; update() maps the buffered chunks of all channels
    in one unc_stream_step call.  `backend`/`index` exist so the CPU tests can drive this class with the
    emulated device code."""

    DEPLETE, ENRICH = 0, 1                 # RealtimeParams::Mode
    FULL, EVEN, ODD = 0, 1, 2              # RealtimeParams::ActiveChs

    def __init__(self, conf, backend=None, index=None):
        from . import stream as S
        self.conf, self._S = conf, S
        self.chunk_len = int(np.float32(conf.chunk_time) * np.float32(conf.sample_rate)) & 0xFFFF   # u16 chunk_len()
        if backend is None:
            if not conf.bwa_prefix:
                raise RuntimeError("Conf.bwa_prefix is not set")
            index = Index(conf.bwa_prefix, preset=conf.idx_preset, device=conf.device, model_table=conf.model_path or None)
            p = N.default_params()
            p.max_events, p.max_paths, p.seed_len = conf.max_events, conf.max_paths, conf.seed_len
            p.bp_per_sec, p.sample_rate = conf.bp_per_sec, conf.sample_rate
            backend = S.StreamMapper(index, conf.num_channels, self.chunk_len, max_chunks=conf.max_chunks, params=p)
            if conf.exact_ties:
                backend.set_tie_order(1)
        self.backend, self.index = backend, index
        n = conf.num_channels
        self._pending = [None] * n          # chunk waiting for the next update()
        self._read = [None] * n             # (id, number, start) of the read in progress
        self._fresh = [False] * n           # the pending chunk starts a read
        self._reset = [False] * n           # request_reset: the read in progress gets no more signal
        self._stopped = False

    def _active(self, ch):
        return self._read[ch] is not None

    def add_chunk(self, c):
        """RealtimePool::add_chunk (src/realtime_pool.cpp:74-101)."""
        ch = c.channel - 1
        if self._stopped or not (0 <= ch < self.conf.num_channels):
            return False
        if self._active(ch) and self._read[ch][1] != c.number:
            # a different read arrived while the previous one is mapping: it is reset and the chunk is buffered
            self._reset[ch] = True
            self._pending[ch], self._fresh[ch] = c, True
            return True
        if not self._active(ch):
            self._pending[ch], self._fresh[ch] = c, True
            return True
        if self._pending[ch] is not None:   # Mapper::add_chunk refuses while the previous chunk is unprocessed
            return False
        self._pending[ch], self._fresh[ch] = c, False
        return True

    def try_add_chunk(self, c):
        """RealtimePool::try_add_chunk (src/realtime_pool.cpp:108-139): an empty chunk means the read has no more signal."""
        ch = c.channel - 1
        if self._stopped or not (0 <= ch < self.conf.num_channels):
            return False
        if c.empty():
            if self._active(ch) and self._pending[ch] is None:
                self._reset[ch] = True
            return False
        if not self._active(ch):
            if self._pending[ch] is not None:
                return False
            self._pending[ch], self._fresh[ch] = c, True
            return True
        if self._read[ch][1] == c.number and self._pending[ch] is None:
            self._pending[ch], self._fresh[ch] = c, False
            return True
        return False

    def update(self):
        """Maps every buffered chunk (one step) and returns the reads that finished: [(channel, number, Paf)]."""
        S = self._S
        if self._stopped:
            return []
        out = []
        # phase 0: resets of reads in progress; phase 1: the buffered chunks, float32 ones first and then int16
        # ones (a step carries one sample type)
        for phase, dtype in ((0, 0), (1, 0), (1, 1)):
            descs, parts, chans, off = [], [], [], 0
            for ch in range(self.conf.num_channels):
                d = S.ChunkDesc()
                d.channel, d.dtype = ch, dtype
                d.cal_range, d.cal_offset, d.cal_digit = 1.0, 0.0, 1.0
                if phase == 0:
                    if not (self._reset[ch] and self._active(ch)):
                        continue
                    d.new_read, d.offset, d.n_samples = 0, 0, 0
                else:
                    c = self._pending[ch]
                    if c is None or c.dtype != dtype:
                        continue
                    d.cal_range, d.cal_offset, d.cal_digit = c.cal
                    raw = c.pop()
                    d.new_read, d.offset, d.n_samples = (1 if self._fresh[ch] else 0), off, len(raw)
                    if self._fresh[ch]:
                        self._read[ch] = (c.id, c.number, c.start)
                    parts.append(raw)
                    off += len(raw)
                    self._pending[ch] = None
                descs.append(d)
                chans.append(ch)
            if not descs:
                continue
            arr = (S.ChunkDesc * len(descs))(*descs)
            flat = np.concatenate(parts) if parts else np.zeros(1, np.float32 if dtype == 0 else np.int16)
            res = (S.StreamResult * len(descs))()
            self.backend.step(arr, len(descs), flat, res)
            for ch, r in zip(chans, res):
                if phase == 0:
                    self._reset[ch] = False
                if r.state == S.MAPPING or self._read[ch] is None:
                    continue
                rid, number, start = self._read[ch]
                if int(r.rec.status) != 0:          # the channel's device workspace overflowed: never silent
                    sys.stderr.write("Warning: read %s (channel %d) overflowed its device workspace (status %d); reported unmapped\n"
                                     % (rid, ch + 1, int(r.rec.status)))
                p = _paf_from_rec(self.index.seqs if self.index is not None else [], r.rec, rid, ch + 1, start)
                if r.ended:
                    p._ended = True        # Paf::set_ended
                out.append((ch + 1, number, p))
                self._read[ch] = None       # Mapper::deactivate
        return out

    def all_finished(self):
        return all(r is None for r in self._read) and all(p is None for p in self._pending)

    def stop_all(self):
        if not self._stopped:
            self._stopped = True
            if hasattr(self.backend, "close"):
                self.backend.close()


class _OrdRead:
    __slots__ = ("id", "channel", "number", "start", "key", "n", "signal", "cal", "dtype", "src")

    def __init__(self, rid, channel, number, start, key, n, signal, cal, dtype, src):
        self.id, self.channel, self.number, self.start, self.key = rid, channel, number, start, key
        self.n, self.signal, self.cal, self.dtype, self.src = n, signal, cal, dtype, src


class MapPoolOrd:
    """reference src/map_pool_ord.hpp:33-62 (`uncalled_map_ord`): MapPoolOrd(conf), add_fast5, add_read(read_id),
    load_fast5s, update() -> [Paf], running(), stop().  Every channel's reads are replayed in the order they were
    sequenced, through the streaming mapper with its long-lived per-channel state, as UNCALLED would have mapped them in
    real time.  The replay runs on the device (unc_stream_replay): the reads go over in windows of at most
    `window_samples` samples, each channel steps through its chunks without a host round trip, and the next window's
    signals are decoded while the device replays the current one.  The records do not depend on the window size.

    Observable differences from the reference (DESIGN.md section 4):
      * reads of one channel with equal start samples keep the order of their files and of their position in the file
        (the reference's pdqsort leaves that order unspecified);
      * a channel number above conf.num_channels raises ValueError in load_fast5s (out of bounds in the reference);
      * a read without samples is skipped (the reference never finishes it and runs forever);
      * min_active_reads counts, after each step of the lockstep loop, the channels with a read in progress (the
        reference counts at thread-timing-dependent moments);
      * all reads of a run share one sample type (int16 from fast5 files)."""

    def __init__(self, conf, backend=None, index=None, window_samples=1 << 28):
        """`backend`/`index` (tests): an object with replay(reads, n, flat, out) standing in for the StreamMapper, and an
        index with .seqs.  The index is loaded at the first update(), so that input errors are found first."""
        self.conf = conf
        self.chunk_len = int(np.float32(conf.chunk_time) * np.float32(conf.sample_rate)) & 0xFFFF   # u16 chunk_len()
        self.backend, self.index = backend, index
        self.window_samples = int(window_samples)
        self._files, self._ids = [], None
        if conf.fast5_list:                                   # Fast5Reader::load_fast5_list
            self._files = [l.rstrip("\n") for l in open(conf.fast5_list) if l.strip()]
        if conf.read_list:
            self._ids = set(l.strip() for l in open(conf.read_list) if l.strip())
        self._mem = []                                        # queue_read
        self._channels = None                                 # per channel: its reads in replay order
        self._open = {}
        self._future, self._executor = None, None
        self._stopped = False
        n = conf.num_channels
        self._next_start = [0] * n                            # the step at which the channel's next read starts
        self._starts, self._fins = [], []                     # every replayed read's first and last step
        self._held = []                                       # results after the step up to which activity is known
        self._known = -1

    # -- input ---------------------------------------------------------------------------
    def add_fast5(self, fname):
        self._files.append(fname)

    def add_read(self, read_id):
        """Fast5Reader::add_read: only the reads named so are mapped (map_pool_ord.cpp:44)."""
        if self._ids is None:
            self._ids = set()
        self._ids.add(read_id)

    def queue_read(self, read_id, signal, channel, number=0, start_sample=0, calibration=None):
        """Queue one in-memory read (as MapPool.add_read): float32 pA, or int16 DAC values with calibration=(range,
        offset, digitisation).  `channel` is 1-based.  Reads queued so come after those of the fast5 files when start
        samples are equal."""
        sig = np.asarray(signal)
        if calibration is None:
            sig, dtype, cal = np.ascontiguousarray(sig, np.float32), 0, (1.0, 0.0, 1.0)
        else:
            if sig.dtype != np.int16:
                raise TypeError("calibration given: the signal must be int16 DAC values")
            sig, dtype, cal = np.ascontiguousarray(sig), 1, tuple(float(np.float32(x)) for x in calibration)
        self._mem.append((read_id, sig, int(channel), int(number), int(start_sample), dtype, cal))

    def _max_len(self):
        return int(self.conf.max_chunks) * self.chunk_len      # ReadBuffer keeps at most max_chunks chunks

    def load_fast5s(self):
        """MapPoolOrd::load_fast5s (map_pool_ord.cpp:48-59): every read's header is read up front (read list and
        max_reads applied as Fast5Reader does), reads are grouped by channel and each channel is sorted by start sample,
        ties by file order and position in the file.  Signals are decoded window by window.  Raises ValueError for a
        channel outside 1..num_channels."""
        from .fast5 import Fast5File
        n_ch, cap = self.conf.num_channels, self.conf.max_reads
        reads, k = [], 0
        for fi, path in enumerate(self._files):
            if cap and k >= cap:
                break
            with Fast5File(path) as f:
                for i in range(f.n_reads):
                    if cap and k >= cap:
                        break
                    info = f.info(i)
                    if self._ids is not None and info.read_id not in self._ids:
                        continue
                    k += 1
                    n = min(info.n_samples, self._max_len())
                    if n:
                        reads.append(_OrdRead(info.read_id, int(info.channel), int(info.number), int(info.start_sample),
                                              (int(info.start_sample) % (1 << 64), fi, i), n, None, None, 1, (path, i)))
        for j, (rid, sig, ch, nm, st, dtype, cal) in enumerate(self._mem):
            if (self._ids is not None and rid not in self._ids) or (cap and k >= cap):
                continue
            k += 1
            sig = sig[:self._max_len()]
            if len(sig):
                reads.append(_OrdRead(rid, ch, nm, st, (st % (1 << 64), len(self._files), j), len(sig), sig, cal, dtype,
                                      None))
        bad = [r for r in reads if not 1 <= r.channel <= n_ch]
        if bad:
            raise ValueError("read %s is on channel %d, outside 1..%d (--num-channels)" % (bad[0].id, bad[0].channel, n_ch))
        if len(set(r.dtype for r in reads)) > 1:
            raise ValueError("the reads mix float32 and int16 signals")
        self._channels = [[] for _ in range(n_ch)]
        for r in reads:
            self._channels[r.channel - 1].append(r)
        for q in self._channels:
            q.sort(key=lambda r: r.key)
        self._left = [len(q) for q in self._channels]
        self.n_loaded = len(reads)
        return len(reads)

    def _fetch(self, reads):
        """Decodes the signals of a window's fast5 reads (their sample counts after the max_chunks cut)."""
        from .fast5 import Fast5File
        for r in reads:
            if r.signal is None:
                path, i = r.src
                f = self._open.get(path)
                if f is None:
                    f = self._open[path] = Fast5File(path)
                rd = f.load(i, 1, max_samples_per_read=self._max_len(), threads=self.conf.threads)[0]
                r.signal, r.cal, r.n = rd.signal, rd.calibration, len(rd.signal)
        return reads

    def _take_window(self):
        """The next reads of the channels, one per channel per round, while they fit in window_samples (at least one)."""
        win, total = [], 0
        while True:
            took = False
            for q in self._channels:
                if q and (not win or total + q[0].n <= self.window_samples):
                    win.append(q.pop(0))
                    total += win[-1].n
                    took = True
            if not took:
                return win

    # -- output --------------------------------------------------------------------------
    def _ensure_backend(self):
        if self.backend is not None:
            return
        from .stream import StreamMapper
        if not self.conf.bwa_prefix:
            raise RuntimeError("Conf.bwa_prefix is not set")
        self.index = Index(self.conf.bwa_prefix, preset=self.conf.idx_preset, device=self.conf.device,
                           model_table=self.conf.model_path or None)
        p = N.default_params()
        p.max_events, p.max_paths, p.seed_len = self.conf.max_events, self.conf.max_paths, self.conf.seed_len
        p.bp_per_sec, p.sample_rate = self.conf.bp_per_sec, self.conf.sample_rate
        self.backend = StreamMapper(self.index, self.conf.num_channels, self.chunk_len, max_chunks=self.conf.max_chunks,
                                    params=p)
        if self.conf.exact_ties:
            self.backend.set_tie_order(1)

    def _prefetch(self):
        win = self._take_window()
        if not win:
            return None
        if any(r.signal is None for r in win):
            if self._executor is None:
                from concurrent.futures import ThreadPoolExecutor
                self._executor = ThreadPoolExecutor(max_workers=1)
            return self._executor.submit(self._fetch, win)
        return _Done(win)

    def _replay(self, win):
        from . import stream as S
        reads = (S.ReplayRead * len(win))()
        off = 0
        for d, r in zip(reads, win):
            d.channel, d.number, d.offset, d.n_samples, d.dtype = r.channel - 1, r.number & 0xFFFFFFFF, off, r.n, r.dtype
            d.cal_range, d.cal_offset, d.cal_digit = r.cal
            off += r.n
        flat = np.concatenate([r.signal for r in win])
        out = (S.ReplayResult * len(win))()
        self.backend.replay(reads, len(win), flat, out)
        seqs = self.index.seqs if self.index is not None else []
        ret = []
        for o in out:
            r = win[o.read]
            if int(o.res.rec.status) != 0:               # the channel's device workspace overflowed: never silent
                sys.stderr.write("Warning: read %s (channel %d) overflowed its device workspace (status %d); reported "
                                 "unmapped\n" % (r.id, r.channel, int(o.res.rec.status)))
            p = _paf_from_rec(seqs, o.res.rec, r.id, r.channel, r.start)
            if o.res.ended:
                p._ended = True                            # Paf::set_ended
            p.chunks, p.rec = int(o.res.chunks), N.PafRec.from_buffer_copy(bytes(o.res.rec))   # chunks used, raw record
            ch = r.channel - 1
            self._starts.append(self._next_start[ch])
            self._fins.append(int(o.step))
            self._next_start[ch] = int(o.step) + 1
            self._left[ch] -= 1
            ret.append((int(o.step), p))
            r.signal = None
        return ret

    def _gate(self, results):
        """min_active_reads: the run stops after the first step t at which fewer channels than that have a read in progress
        (started at or before t, finished after t).  Results are held back until activity is known up to their step."""
        m = int(self.conf.min_active_reads)
        if m <= 0:
            return [p for _, p in results]
        self._held += results
        pending = [self._next_start[c] - 1 for c, k in enumerate(self._left) if k]
        horizon = min(pending) if pending else max(self._fins, default=0)
        st, fi = np.sort(np.array(self._starts, np.int64)), np.sort(np.array(self._fins, np.int64))
        cand = np.unique(np.concatenate([[0], fi]))
        cand = cand[(cand > self._known) & (cand <= horizon)]
        active = np.searchsorted(st, cand, side="right") - np.searchsorted(fi, cand, side="right")
        low = np.flatnonzero(active < m)
        stop = int(cand[low[0]]) if len(low) else None
        upto = stop if stop is not None else horizon
        out = [p for s, p in self._held if s <= upto]
        self._held = [(s, p) for s, p in self._held if s > upto]
        self._known = max(self._known, upto)
        if stop is not None:
            self._stop_all()
        return out

    def update(self):
        """Replays the next window on the device and returns its reads' Paf records, in completion order.  Each Paf also
        carries `chunks` (chunks the decision took) and `rec` (the device record, unc_paf_rec)."""
        if self._stopped:
            return []
        if self._channels is None:
            self.load_fast5s()
        self._ensure_backend()
        cur = self._future if self._future is not None else self._prefetch()
        self._future = None
        if cur is None:
            self._stopped = True
            return self._gate([]) if self._held else []
        win = cur.result()
        self._future = self._prefetch()                   # decoded while the device replays this window
        return self._gate(self._replay(win))

    def running(self):
        return not self._stopped and (self._channels is None or self._future is not None or bool(self._held) or
                                      any(self._channels))

    def _stop_all(self):
        self._stopped = True
        for q in self._channels or []:
            q.clear()
        self._left = [0] * len(self._left)
        self._held = []

    def stop(self):
        self._stopped = True
        if self._future is not None:
            try:
                self._future.result()
            except Exception:
                pass
            self._future = None
        if self._executor is not None:
            self._executor.shutdown(wait=True)
            self._executor = None
        for f in self._open.values():
            f.close()
        self._open = {}
        if self.backend is not None and hasattr(self.backend, "close"):
            self.backend.close()


class _Done:
    """A window whose signals are already in memory (the Future interface the prefetch uses)."""

    def __init__(self, v):
        self.v = v

    def result(self):
        return self.v
