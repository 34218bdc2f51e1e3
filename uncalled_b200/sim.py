"""`uncalled sim`: predicts what a read-until run with this mapper would enrich or deplete, by replaying the reads of a
control run through the streaming mapper (api.RealtimePool, the sm_90a stream kernels) with the channel activity of
an earlier UNCALLED run.  Restates the reference's simulator (src/client_sim.{hpp,cpp}: ClientSim, SimChannel, SimRead,
ScanIntv; uncalled/sim_utils.py: find_scans, SeqsumProfile, load_sim; the `sim` branch of realtime_cmd in
scripts/uncalled:169-300).

  * load_sim(client, conf) turns the UNCALLED run's sequencing summary and PAF and the control run's summary into
    the add_intv / add_gap / add_delay / add_read calls the reference makes, in the same order.
  * ClientSim(conf, clock=None) is the per-channel state machine.  Times are in samples: clock() * sample_rate / 1000
    rounded to float32, as ClientSim::get_time.  A read keeps only the int16 samples its chunks need, with its
    calibration (the reference holds every read as float chunks).
  * run_sim(conf, fast5s, out) is the decision loop; PAF lines go to `out`.

Differences from the reference are listed in DESIGN.md section 8.
"""
import collections
import os
import sys
import time

import numpy as np

MAX_SLEEP = 0.01
U32 = 0xFFFFFFFF
SEQSUM_COLUMNS = ("channel", "start_time", "duration", "mux", "read_id", "template_start", "template_duration",
                  "sequence_length_template")


class SimError(RuntimeError):
    """A simulator input that cannot be used (missing file or column, too few control reads)."""


def _f32(x):
    return float(np.float32(x))


# ---------------------------------------------------------------------------------------------------------------------
# the activity pattern (reference uncalled/sim_utils.py)

def find_scans(sts, ens, mxs, max_block_gap=1, max_intv_gap=20, min_mux_frac=0.95):
    """The mux scans of a run: (start, end) in seconds of every run of four blocks of reads, each block dominated by
    one mux and the muxes going 1, 2, 3, 4.  A block is a stretch of reads with no gap longer than `max_block_gap`."""
    o = np.argsort(sts)
    sts, ens, mxs = sts[o], ens[o], mxs[o]

    blocks = []
    bst, ben = sts[0], ens[0]
    for rst, ren in zip(sts[1:], ens[1:]):
        if rst - ben > max_block_gap:
            blocks.append((bst, ben))
            bst, ben = rst, ren
        else:
            ben = max(ren, ben)
    blocks.append((bst, ben))

    segs, seg_gaps = [], []
    scan = []
    prev_en, lead_gap = 0, None
    for bst, ben in blocks:
        if scan and bst - scan[-1][1] > max_intv_gap:
            if len(scan) == 4:
                segs.append(scan)
            scan = []

        muxes = collections.Counter(mxs[(sts >= bst) & (sts < ben)])
        top_count, top_mux = max(((c, m) for m, c in muxes.items()), default=(0, 0))
        if muxes and top_count / sum(muxes.values()) >= min_mux_frac:
            if top_mux != 4 and len(scan) == 4:
                segs.append(scan)
                seg_gaps.append((lead_gap, bst - scan[-1][1]))
                scan = []
            if scan and top_mux == len(scan):
                if ben - scan[-1][1] < max_intv_gap:       # the same mux again: the block extends the segment
                    scan[-1] = (scan[-1][0], ben)
                elif top_mux == 1:
                    scan[0] = (bst, ben)
                    lead_gap = bst - prev_en
            elif top_mux - 1 == len(scan):
                scan.append((bst, ben))
                if len(scan) == 1:
                    lead_gap = bst - prev_en
            else:
                scan = []
        else:
            if len(scan) == 4:
                segs.append(scan)
                seg_gaps.append((lead_gap, bst - scan[-1][1]))
            scan = []
        prev_en = ben

    # a scan runs from the end of the block before its first segment to the start of the block after its last
    return [(s[0][0] - g[0], s[-1][1] + g[1]) for s, g in zip(segs, seg_gaps)]


class SeqsumProfile:
    """The reads of one sequencing summary, sorted by start time (seconds)."""
    PROPS = ("chs", "sts", "lns", "mxs", "ids", "ens", "glns", "gsts", "tms", "tds", "bps")

    def __init__(self, fname, n_channels=512):
        if not os.path.isfile(fname):
            raise SimError("sequencing summary \"%s\" does not exist" % fname)
        self.fname, self.n_channels = fname, n_channels
        with open(fname) as infile:
            header = infile.readline().split()
            col = {}
            for name in SEQSUM_COLUMNS:
                if name not in header:
                    raise SimError("sequencing summary \"%s\" has no \"%s\" column" % (fname, name))
                col[name] = header.index(name)
            rows = [line.split() for line in infile if line.strip()]
        if not rows:
            raise SimError("sequencing summary \"%s\" has no reads" % fname)
        try:
            sts = np.array([float(t[col["start_time"]]) for t in rows])
            self.lns = np.array([float(t[col["duration"]]) for t in rows])
            self.chs = np.array([int(t[col["channel"]]) for t in rows])
            self.mxs = np.array([int(t[col["mux"]]) for t in rows])
            self.ids = np.array([t[col["read_id"]] for t in rows])
            self.tms = np.array([float(t[col["template_start"]]) for t in rows]) - sts
            self.tds = np.array([float(t[col["template_duration"]]) for t in rows])
            self.bps = np.array([int(t[col["sequence_length_template"]]) for t in rows])
        except (ValueError, IndexError) as e:
            raise SimError("sequencing summary \"%s\": unreadable row (%s)" % (fname, e))
        bad = (self.chs < 1) | (self.chs > n_channels)
        if np.any(bad):
            raise SimError("sequencing summary \"%s\": channel %d is outside 1..%d" % (fname, self.chs[bad][0], n_channels))
        self.sts, self.ens = sts, sts + self.lns
        self._take(np.argsort(self.sts))
        self.chodr = np.arange(n_channels) + 1
        self.chcts = self._counts()

    def _counts(self):
        return np.bincount(self.chs, minlength=self.n_channels + 1)[1:]

    def _take(self, sel):
        for p in self.PROPS:
            if hasattr(self, p):
                setattr(self, p, getattr(self, p)[sel])

    def rm_scans(self):
        """Removes the reads inside mux scans and closes the time up.  Returns the scan boundaries in the new time:
        the start of every scan, then the end of the last read."""
        bounds, sh = [], 0
        for st, en in find_scans(self.sts, self.ens, self.mxs):
            inside = (self.sts + sh >= st) & (self.ens + sh <= en)
            self._take(~inside)
            ln = en - st
            bounds.append(st - sh)
            self.sts[self.sts + sh >= st] -= ln
            self.ens[self.ens + sh >= st] -= ln
            sh += ln
        bounds.append(np.max(self.ens))
        self.chcts = self._counts()
        return np.array(bounds)

    def compute_gaps(self):
        """gsts/glns: the gap before every read on its channel (the first gap starts at 0)."""
        self.gsts, self.glns = np.zeros(len(self.ids)), np.zeros(len(self.ids))
        for ch in range(1, self.n_channels + 1):
            m = self.chs == ch
            if not np.any(m):
                continue
            gsts = np.insert(self.ens[m][:-1], 0, 0)
            self.gsts[m], self.glns[m] = gsts, self.sts[m] - gsts

    def compute_eject_delays(self, paf):
        """dls: for every read the PAF shows ejected (ej or ub tag), the template time it went on being sequenced
        after the decision; inf for the others."""
        if not os.path.isfile(paf):
            raise SimError("PAF \"%s\" does not exist" % paf)
        self.dls = np.full(len(self.sts), np.inf)
        idx = {r: i for i, r in enumerate(self.ids)}
        tlns = self.lns - self.tms
        with open(paf) as infile:
            for line in infile:
                if line[0] == "#":
                    continue
                t = line.split()
                i = idx.get(t[0])
                if i is None:
                    continue
                tags = {}
                for tag in t[12:]:
                    k, _, v = tag.split(":", 2)
                    tags[k] = v
                ej = tags.get("ej", tags.get("ub"))
                if ej is not None:
                    self.dls[i] = max(0, tlns[i] - (int(t[1]) / 450.0 + float(ej)))

    def chsort(self, order):
        self.chodr, self.chcts = self.chodr[order], self.chcts[order]


def load_sim(client, conf, log=sys.stderr):
    """Builds the simulation pattern into `client` (reference uncalled/sim_utils.py:249-443):
      * scan intervals of every channel from the UNCALLED run, mux scans removed and intervals broken at gaps longer
        than median + stddev of all gaps (ACTIVE_THRESH), scaled by conf.sim_speed;
      * the shorter gaps and, for every ejected read, the median eject delay;
      * the control run's reads, balanced over the channels in proportion to the UNCALLED run's read counts with at
        least conf.min_ch_reads per channel that had reads.
    Every input is read and checked before the first call on `client`."""
    n = conf.num_channels
    sr = float(conf.sample_rate)

    def samp(sec, coef=1.0):
        return int(np.round(sec * sr * coef))

    for f in (conf.unc_seqsum, conf.unc_paf, conf.ctl_seqsum):
        if not os.path.isfile(f):
            raise SimError("\"%s\" does not exist" % f)
    log.write("Loading UNCALLED run\n")
    unc = SeqsumProfile(conf.unc_seqsum, n)
    ctl = SeqsumProfile(conf.ctl_seqsum, n)
    scans = unc.rm_scans()
    unc.compute_gaps()
    unc.compute_eject_delays(conf.unc_paf)
    delay = np.median(unc.dls[unc.dls != np.inf]) if np.any(unc.dls != np.inf) else 0.0
    unc.chsort(np.argsort(unc.chcts))
    thresh = np.median(unc.glns) + np.std(unc.glns)

    log.write("Generating pattern\n")
    speed, intv_time = conf.sim_speed, conf.scan_intv_time
    for ch in range(1, n + 1):
        m = unc.chs == ch
        if not np.any(m):
            continue
        gsts, glns = unc.gsts[m], unc.glns[m]
        sc, itv_st = 0, 0
        for br in np.flatnonzero(glns >= thresh):          # a long gap ends the channel's active stretch
            act_en = gsts[br]
            while scans[sc + 1] < act_en:                  # whole intervals before the gap
                client.add_intv(ch, sc, samp(itv_st - scans[sc], speed), samp(intv_time, speed))
                itv_st = scans[sc + 1]
                sc += 1
            if itv_st != act_en:                            # the part of the gap's interval before it
                client.add_intv(ch, sc, samp(itv_st - scans[sc], speed), samp(act_en - scans[sc], speed))
            itv_st = act_en + glns[br]
            while scans[sc + 1] < itv_st:
                sc += 1
        last = np.max(unc.ens[m])
        while sc < len(scans) - 1 and scans[sc] < last:     # from the last gap to the channel's last read
            client.add_intv(ch, sc, samp(itv_st - scans[sc], speed), samp(min(last - scans[sc], intv_time), speed))
            itv_st = scans[sc + 1]
            sc += 1
        dls = unc.dls[m]
        for sc in range(len(scans) - 1):
            in_sc = (gsts > scans[sc]) & ((gsts + glns) <= scans[sc + 1])
            for ln in glns[in_sc]:
                if 0 < ln < thresh:
                    client.add_gap(ch, sc, samp(ln))
            for dl in dls[in_sc]:
                if dl != np.inf:
                    client.add_delay(ch, sc, samp(delay))

    log.write("Ordering control reads\n")
    ctl.rm_scans()
    ctl.chsort(np.argsort(ctl.chcts))
    # target read count per channel: proportional to the UNCALLED run, with the minimum for channels that had reads
    min_const = np.zeros(n)
    min_const[unc.chcts > 0] = conf.min_ch_reads
    total = np.sum(ctl.chcts)
    remain = total * unc.chcts / np.sum(unc.chcts) - min_const
    remain_clp = np.clip(remain, 0, np.inf)
    tgt = np.round(min_const + np.sum(remain) * remain_clp / np.sum(remain_clp)).astype(int)
    step, i = (-1 if np.sum(tgt) > total else 1), n - 1
    while np.sum(tgt) != total:                             # rounding error, taken from the last channels
        tgt[i] += step
        i -= 1
    diff = ctl.chcts - tgt
    order = np.flip(np.argsort(diff), 0)
    diff, tgt = diff[order], tgt[order]
    ctl.chsort(order)
    unc.chsort(order)

    sim_reads = [None] * n
    extra, e = [], 0                                        # surplus reads of the channels with more than their target
    for i in range(n):
        j = ctl.chs == ctl.chodr[i]
        reads = list(zip(ctl.ids[j], ctl.tms[j]))
        if diff[i] >= 0:
            if diff[i] > 0:
                extra.append(reads[tgt[i]:])
            reads = reads[:tgt[i]]
        else:
            if e >= len(extra):
                raise SimError("the control run has too few reads to fill channel %d" % unc.chodr[i])
            while len(reads) < tgt[i] and e < len(extra):
                need = tgt[i] - len(reads)
                if len(extra[e]) > need:
                    reads += extra[e][:need]
                    extra[e] = extra[e][need:]
                else:
                    reads += extra[e]
                    e += 1
            if len(reads) < tgt[i]:
                raise SimError("the control run has too few reads to fill channel %d" % unc.chodr[i])
        sim_reads[unc.chodr[i] - 1] = reads

    for ch in range(1, n + 1):
        for rd, tm in sim_reads[ch - 1]:
            client.add_read(ch, str(rd), samp(tm))


# ---------------------------------------------------------------------------------------------------------------------
# the client (reference src/client_sim.{hpp,cpp})

class _ScanIntv:
    """The activity of one channel between two mux scans: switch times relative to the interval's start, and the
    gaps and eject delays it takes round-robin."""
    __slots__ = ("channel", "intv", "start_time", "active", "bounds", "gaps", "delays", "g", "d")

    def __init__(self, channel, intv):
        self.channel, self.intv = channel, intv
        self.start_time, self.active = U32, False
        self.bounds = collections.deque()
        self.gaps, self.delays, self.g, self.d = [], [], 0, 0

    def set_active(self, st, en):
        if st == 0:
            self.active = True
        else:
            self.bounds.append(st)
        self.bounds.append(en)

    def get_end(self):
        return self.bounds[-1] if self.bounds else 0

    def is_active(self, t, log):
        while self.bounds and ((t - self.start_time) & U32) >= self.bounds[0]:
            self.bounds.popleft()
            self.active = not self.active
            log.write("switch %d %d %d %d\n" % (self.active, self.channel, self.intv, t))
        return self.active

    def next_gap(self):
        if not self.gaps:
            if self.active:                 # an interval with no gaps ends at its first read
                self.active = False
                if self.bounds:
                    self.bounds.popleft()
            return 0
        gap = self.gaps[self.g]
        self.g = (self.g + 1) % len(self.gaps)
        return gap

    def next_delay(self):
        if not self.delays:
            return 0
        dl = self.delays[self.d]
        self.d = (self.d + 1) % len(self.delays)
        return dl


class _SimRead:
    """One control read on its channel: `n_chunks` full chunks from the template start, stored as int16 samples.
    A read named in the pattern but absent from the fast5 files stays empty: no duration, no chunks."""
    __slots__ = ("id", "channel", "number", "sig", "cal", "chunk_len", "n_chunks", "c", "start", "end", "duration")

    def __init__(self):
        self.id, self.channel, self.number, self.sig, self.cal = "", 0, 0, None, None
        self.chunk_len = self.n_chunks = self.c = self.start = self.end = self.duration = 0

    def load(self, read_id, channel, number, signal, calibration, offs, chunk_len, max_chunks):
        n = min(len(signal), max_chunks * chunk_len)        # ReadBuffer keeps at most max_chunks chunks of signal
        self.id, self.channel, self.number, self.cal = read_id, channel, int(number), calibration
        self.duration, self.chunk_len = n, chunk_len
        self.n_chunks = min((n - offs) // chunk_len, max_chunks) if n >= offs else 0
        self.sig = np.array(signal[offs:offs + self.n_chunks * chunk_len], dtype=np.int16)

    def begin(self, t):
        self.start, self.end, self.c = t, (t + self.duration) & U32, 0

    def started(self, t):
        return self.start != 0 and self.start <= t

    def chunk_ready(self, t):
        return self.started(t) and self.c < self.n_chunks and t >= self.start + (self.c + 1) * self.chunk_len

    def pop_chunk(self):
        from .api import Chunk
        L, c = self.chunk_len, self.c
        self.c += 1
        return Chunk(self.id, self.channel, self.number, self.start + c * L, self.sig, c * L, L, calibration=self.cal)

    def stop_receiving(self):
        self.c = self.n_chunks

    def unblock(self, t, delay):
        self.end = min((t + delay) & U32, (self.start + self.duration) & U32)


class _SimChannel:
    """One channel: its scan intervals and its reads, which follow each other round-robin while it is active."""
    __slots__ = ("channel", "intvs", "reads", "r", "extra_gap", "was_active")

    def __init__(self, channel):
        self.channel, self.intvs, self.reads = channel, collections.deque(), []
        self.r, self.extra_gap, self.was_active = 0, 0, False

    def is_dead(self):
        return not self.intvs

    def _intv(self, i):
        while i >= len(self.intvs):
            self.intvs.append(_ScanIntv(self.channel, len(self.intvs)))
        return self.intvs[i]

    def is_active(self, t, log):
        if self.is_dead():
            return False
        if self.intvs[0].is_active(t, log):
            if not self.was_active:
                self.reads[self.r].begin((t + self.intvs[0].next_gap()) & U32)
                self.was_active = True
        elif self.was_active:
            self.r = (self.r + 1) % len(self.reads)
            self.was_active = False
        return self.was_active

    def start(self, t, log):
        if not self.reads:          # a channel given intervals but no reads cannot produce any signal
            self.intvs.clear()
        if not self.is_dead():
            self.extra_gap = 0
            self.intvs[0].start_time = t
        return self.is_active(t, log)

    def chunk_ready(self, t, log):
        if not self.intvs[0].is_active(t, log):
            return False
        end, idle = self.reads[self.r].end, 0
        while t >= end:
            self.r = (self.r + 1) % len(self.reads)
            self.reads[self.r].begin((end + self.intvs[0].next_gap() + self.extra_gap) & U32)
            self.extra_gap = 0
            nxt = self.reads[self.r].end
            idle = idle + 1 if nxt == end else 0
            if idle > len(self.reads):  # only empty reads and no gaps: time cannot advance on this channel
                return False
            end = nxt
        return self.reads[self.r].chunk_ready(t)

    def read_number(self):
        return self.reads[self.r].number if self.reads else 0

    def intv_ended(self, t):
        return self.is_dead() or self.intvs[0].get_end() <= t

    def next_intv(self, t):
        self.intvs.popleft()
        if not self.is_dead():
            self.intvs[0].start_time = t

    def unblock(self, t, ej_time):
        delay = self.intvs[0].next_delay() if self.intvs else 0
        self.reads[self.r].unblock(t, delay)
        self.extra_gap = ej_time
        return delay


class ClientSim:
    """reference src/client_sim.hpp:35-390: a flow cell replaying control reads.  `clock` returns milliseconds since
    run() (default: the monotonic wall clock); it exists so that tests can drive the simulation with a fake clock."""

    def __init__(self, conf, clock=None, log=sys.stderr):
        self.conf, self.log = conf, log
        self.n_channels = int(conf.num_channels)
        sr = np.float32(conf.sample_rate)
        self._time_coef = float(sr / np.float32(1000))
        self.ej_time = int(np.float32(conf.ej_time) * sr)
        self.scan_time = int(np.float32(conf.scan_time) * sr)
        self.chunk_len = int(np.float32(conf.chunk_time) * sr) & 0xFFFF     # u16 chunk_len(), as RealtimePool
        self.max_chunks = int(conf.max_chunks)
        self.channels = [_SimChannel(c) for c in range(1, self.n_channels + 1)]
        self.read_locs, self.fast5s = {}, []
        self._running = self.in_scan = False
        self.scan_start = 0
        self._t0 = None
        self._clock = clock if clock is not None else \
            (lambda: (time.monotonic() - self._t0) * 1000.0 if self._t0 is not None else 0.0)

    def _ch(self, ch):
        if not 1 <= ch <= self.n_channels:
            raise ValueError("channel %d is outside 1..%d" % (ch, self.n_channels))
        return self.channels[ch - 1]

    @staticmethod
    def _u32(*vals):
        for v in vals:
            if not 0 <= v <= U32:
                raise ValueError("%r is not a sample count" % (v,))

    # -- the pattern -----------------------------------------------------------------------------------------------
    def add_intv(self, ch, i, st, en):
        self._u32(i, st, en)
        self._ch(ch)._intv(i).set_active(int(st), int(en))

    def add_gap(self, ch, i, length):
        self._u32(i, length)
        self._ch(ch)._intv(i).gaps.append(int(length))

    def add_delay(self, ch, i, length):
        self._u32(i, length)
        self._ch(ch)._intv(i).delays.append(int(length))

    def add_read(self, ch, read_id, offs):
        self._u32(offs)
        c = self._ch(ch)
        c.reads.append(_SimRead())
        self.read_locs[read_id] = (ch, len(c.reads) - 1, int(offs))

    # -- the reads -------------------------------------------------------------------------------------------------
    def add_fast5(self, fname):
        self.fast5s.append(fname)

    def load_read(self, read_id, number, signal, calibration):
        """Puts one read (int16 DAC values and their (range, offset, digitisation)) in its place; False if the pattern
        does not name it."""
        loc = self.read_locs.get(read_id)
        if loc is None:
            return False
        ch, i, offs = loc
        self.channels[ch - 1].reads[i].load(read_id, ch, number, signal, calibration, offs, self.chunk_len,
                                            self.max_chunks)
        return True

    def load_fast5s(self, threads=0, batch=256):
        """Reads the named reads from the fast5 files, `batch` reads at a time, keeping only the samples of their
        chunks.  Stops once as many reads as the pattern names have been loaded, as the reference's reader does."""
        from .fast5 import Fast5File
        want, n = len(self.read_locs), 0
        max_len = self.max_chunks * self.chunk_len
        for path in self.fast5s:
            if n >= want:
                break
            with Fast5File(path) as f:
                keep = [i for i in range(f.n_reads) if f.info(i).read_id in self.read_locs]
                k = 0
                while k < len(keep) and n < want:
                    first = keep[k]
                    last = first
                    while k + 1 < len(keep) and keep[k + 1] == last + 1 and last - first + 1 < batch:
                        k += 1
                        last = keep[k]
                    k += 1
                    for r in f.load(first, last - first + 1, max_samples_per_read=max_len, threads=threads):
                        if n >= want:
                            break
                        self.load_read(r.read_id, r.number, r.signal, r.calibration)
                        n += 1
                        if n % 1000 == 0:
                            self.log.write("%d loaded\n" % n)
        return n

    # -- the run ---------------------------------------------------------------------------------------------------
    def clock(self):
        """Milliseconds since run()."""
        return self._clock()

    def get_time(self):
        """Sim time in samples, rounded to float32 as ClientSim::get_time."""
        return _f32(self._clock() * self._time_coef)

    def get_runtime(self):
        """Seconds since run()."""
        return _f32(self._clock() / 1000.0)

    @property
    def is_running(self):
        """A read-only property, as the reference binds it."""
        return self._running

    def run(self):
        self._running, self.in_scan = True, False
        self._t0 = time.monotonic()
        for ch in self.channels:
            ch.start(0, self.log)
        return True

    def get_read_chunks(self):
        """[(channel, Chunk)]: every chunk that is complete at the current time."""
        ret = []
        if not self._running:
            return ret
        t = int(self.get_time())
        ended, next_intv = True, False
        if self.in_scan:
            if t - self.scan_start >= self.scan_time:
                ended = self.in_scan = False
                next_intv = True
                self.log.write("%d ending mux scan\n" % t)
            else:
                return ret
        self._running = False
        for c, ch in enumerate(self.channels):
            if ch.is_dead():
                continue
            if next_intv:
                ch.next_intv(t)
                if ch.is_dead():
                    continue
            self._running = True
            if not ch.is_active(t, self.log):
                ended = ch.intv_ended(t) and ended
                continue
            ended = False
            while ch.chunk_ready(t, self.log):
                ret.append((c + 1, ch.reads[ch.r].pop_chunk()))
        if ended and not self.in_scan:
            self.log.write("%d starting mux scan\n" % t)
            self.scan_start = t & U32
        self.in_scan = ended
        return ret

    def stop_receiving_read(self, ch, number):
        c = self._ch(ch)
        if c.read_number() == number and c.reads:
            c.reads[c.r].stop_receiving()

    def unblock_read(self, ch, number):
        """Ends the read `delay` samples from now and adds the eject time to the gap after it; returns the delay."""
        c = self._ch(ch)
        if c.read_number() != number or not c.reads:
            return 0
        return c.unblock(int(self.get_time()) & U32, self.ej_time)


# ---------------------------------------------------------------------------------------------------------------------
# the decision loop (reference scripts/uncalled:169-300, sim branch)

def run_sim(conf, fast5s, out=None, clock=None, log=sys.stderr, backend=None, index=None, reads=()):
    """Simulates a read-until run: PAF lines to `out`, one per read the mapper decided on, with the decision tag
    (en: the read ended, ej + dl: ejected and its delay in samples, kp: kept) and its time in seconds since the
    channel's last chunk.  `clock` (ms since the start) replaces the wall clock for the client and the tag times;
    `backend`/`index` replace the GPU stream mapper as in RealtimePool; `reads`, (read_id, number, int16 signal,
    calibration) tuples, are loaded besides the fast5 files.  Returns the ClientSim."""
    from .api import Paf, RealtimePool
    out = out if out is not None else sys.stdout
    client = ClientSim(conf, clock, log=log)
    load_sim(client, conf, log=log)
    for f in fast5s:
        client.add_fast5(f)
    pool = RealtimePool(conf, backend=backend, index=index)
    try:
        log.write("Loading reads\n")
        client.load_fast5s(threads=conf.threads)
        for r in reads:
            client.load_read(*r)
        client.run()
        now = client.clock
        deplete = conf.realtime_mode == RealtimePool.DEPLETE
        skip_parity = {RealtimePool.EVEN: 1, RealtimePool.ODD: 0}.get(conf.active_chs)
        n = conf.num_channels
        chunk_times = [now() / 1000.0] * n
        unblocked = [None] * n
        end_time = conf.duration * 3600 if conf.duration else float("inf")
        while client.is_running:
            t0 = now()
            for ch, nm, paf in pool.update():
                t = now() / 1000.0 - chunk_times[ch - 1]
                if paf.is_ended():
                    paf.set_float(Paf.ENDED, t)
                    client.stop_receiving_read(ch, nm)
                elif paf.is_mapped() == deplete:
                    paf.set_float(Paf.EJECT, t)
                    paf.set_int(Paf.DELAY, client.unblock_read(ch, nm))
                    unblocked[ch - 1] = nm
                else:
                    paf.set_float(Paf.KEEP, t)
                    client.stop_receiving_read(ch, nm)
                paf.print_paf(out)
            for channel, chunk in client.get_read_chunks():
                if skip_parity is not None and channel % 2 == skip_parity:
                    client.stop_receiving_read(channel, chunk.number)
                elif unblocked[channel - 1] == chunk.number:
                    out.write("# recieved chunk from %s after unblocking\n" % chunk.id)
                else:
                    chunk_times[channel - 1] = now() / 1000.0
                    pool.add_chunk(chunk)
            if client.get_runtime() >= end_time:
                break
            if clock is None:       # a substituted clock does not advance while the loop sleeps
                dt = (now() - t0) / 1000.0
                if dt < MAX_SLEEP:
                    time.sleep(MAX_SLEEP - dt)
    except KeyboardInterrupt:
        log.write("Keyboard interrupt\n")
    finally:
        pool.stop_all()
    return client
