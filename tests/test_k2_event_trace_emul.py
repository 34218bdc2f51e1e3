"""CPU tier: the mapper's path buffer after EVERY event, device source (under the warp emulator) against the oracle.

The other mapper tests compare a read's PAF record and four counters.  Those stay right when the flat placement loop
(phase D1 of uncalled_b200/csrc/unc_k2v2.cuh) puts a source, an order entry, an sa_checked bit or a seed row in the wrong
place, unless the damage changes which cluster wins.  Here both sides report every committed event: the path buffer in
buffer order (one row per position, dups marked invalid), the event's seeds in the order the tracker takes them and the
sources_added_ flags, and the first difference fails the test with the read, the event, the position and both rows.

The inputs reach the edges of the bucket phases: max_paths on both sides of 32 (one pack, one warp pass), 160 (one
chunk's children) and up to 32 767 (the largest value unc_check_params accepts, which the verdict's 16-bit counts and the
key's 18-bit record index are sized for); 2-, 5- and 14-warp CTAs; the exact-ties kernel; the streaming path; and a
low-complexity genome whose k-mer buckets hold thousands of keys with one fm_start.  test_every_bucket_shape_is_reached
checks that they do, from counters the emulator build keeps (emulib.k2_shape_stats).
"""
import collections
import ctypes as C
import hashlib

import numpy as np
import pytest

import emulib
import orclib
import synth
import synthdata


def _arr(ptr, n, dtype):
    dtype = np.dtype(dtype)
    if n == 0:
        return np.zeros(0, dtype)
    return np.frombuffer((C.c_char * (n * dtype.itemsize)).from_address(ptr), dtype=dtype).copy()


def _digest(a):
    return hashlib.blake2b(a.tobytes(), digest_size=16).hexdigest()


class _Recorder:
    """Per item (read, or channel when streaming): one entry per reported event,
    (event_i, nn, digest of the rows, digest of the seeds, flags, overflow).  keep = (item, k): also keep the full rows,
    seeds and flags of the item's k-th event."""

    def __init__(self, keep=None):
        self.ev = collections.defaultdict(list)
        self.keep, self.kept = keep, None

    def add(self, item, event_i, nn, rows_p, n_seeds, seeds_p, flags_p, overflow):
        rows = _arr(rows_p, nn, orclib.TRACE_ROW)
        seeds = _arr(seeds_p, n_seeds, orclib.TRACE_SEED)
        flags = _arr(flags_p, 32, np.uint32)
        k = len(self.ev[item])
        self.ev[item].append((int(event_i), int(nn), _digest(rows), _digest(seeds), flags.tobytes(), int(overflow)))
        if self.keep == (item, k):
            self.kept = (int(event_i), rows, seeds, flags, int(overflow))


class Pair:
    """One configuration mapped by the emulated device and by the oracle, both tracing every event."""

    def __init__(self, prefix, exact=False):
        self.E, self.O = emulib.Emu(prefix), orclib.Oracle(prefix)
        self.exact = exact
        self.shapes = collections.Counter()     # emulib.k2_shape_stats of every run so far

    def set(self, **kw):
        for k, v in kw.items():
            setattr(self.E.params, k, v)
            setattr(self.O.params, k, v)

    def _device(self, run, keep=None):
        rec = _Recorder(keep)
        cb = emulib.PATH_TRACE_FN(lambda ud, it, ev, nn, r, ns, s, f, ov: rec.add(it, ev, nn, r, ns, s, f, ov))
        self.E.L.emu_set_path_trace(cb, None)
        self.E.set_tie_order(1 if self.exact else 0)
        try:
            out = run()
        finally:
            self.E.L.emu_set_path_trace(emulib.PATH_TRACE_FN(), None)
            self.E.set_tie_order(0)
        return rec, out

    def _oracle(self, items, keep=None):
        """items: [(item, fn)]: fn() maps through the oracle; its events are recorded under `item`."""
        rec = _Recorder(keep)
        cur = [None]
        cb = orclib.PATH_TRACE_FN(lambda ud, ev, nn, r, ns, s, f: rec.add(cur[0], ev, nn, r, ns, s, f, 0))
        self.O.lib.orc_set_path_trace(cb, None)
        self.O.lib.orc_set_child_sort(1 if self.exact else 0)
        outs = []
        try:
            for it, fn in items:
                cur[0] = it
                outs.append(fn())
        finally:
            self.O.lib.orc_set_path_trace(orclib.PATH_TRACE_FN(), None)
            self.O.lib.orc_set_child_sort(0)
        return rec, outs

    def batch(self, sigs, n_warps=8, max_blocks=4096):
        """Maps the reads as one batch (max_blocks: the device's seed-cluster store per read, in blocks of 32);
        returns (device records, oracle records, {read: [nn of every event]})."""
        run_dev = lambda keep=None: self._device(lambda: self.E.map_batch(sigs, n_warps=n_warps, max_blocks=max_blocks)[0], keep)
        run_orc = lambda keep=None: self._oracle([(i, (lambda s=s: self.O.map_read(s))) for i, s in enumerate(sigs)], keep)
        emulib.k2_shape_stats(reset=True)
        dev, recs = run_dev()
        self.shapes.update(emulib.k2_shape_stats(reset=True))
        orc, want = run_orc()
        _compare(dev, orc, run_dev, run_orc, "max_paths %d, %d warps" % (self.E.params.max_paths, n_warps))
        for i in range(len(sigs)):
            _check_record(recs[i], want[i], i)
        return recs, want, {it: [e[1] for e in ev] for it, ev in dev.ev.items()}

    def stream(self, sigs, n_channels, chunk_len, n_warps=8):
        """Streams the reads over n_channels (the product's chunk feeding), each channel against the oracle's streaming
        Mapper over the channel's reads in order; the trace of a channel runs through its reads."""
        def run_dev(keep=None):
            def go():
                ES = emulib.EmuStream(self.E, n_channels, chunk_len, n_warps=n_warps)
                try:
                    return ES.map_reads(sigs, chunk_len)
                finally:
                    ES.close()
            return self._device(go, keep)

        chans = [list(range(c, len(sigs), n_channels)) for c in range(n_channels)]
        run_orc = lambda keep=None: self._oracle(
            [(c, (lambda ids=ids: self.O.stream_channel([sigs[i] for i in ids], chunk_len))) for c, ids in enumerate(chans)],
            keep)
        emulib.k2_shape_stats(reset=True)
        dev, res = run_dev()
        self.shapes.update(emulib.k2_shape_stats(reset=True))
        orc, want = run_orc()
        _compare(dev, orc, run_dev, run_orc, "streaming, %d-sample chunks, max_paths %d" % (chunk_len, self.E.params.max_paths))
        for c, ids in enumerate(chans):
            for i, (rec, nu, en) in zip(ids, want[c]):
                if nu == 0:
                    assert res[i] is None, i
                    continue
                assert (emulib.paf_tuple(res[i][3]), res[i][2], res[i][1]) == (orclib.paf_tuple(rec), nu, en), i
                assert _counts(res[i][3])[:3] == _counts(rec)[:3], i
                assert res[i][3].status == 0, i
        return res, want, {it: [e[1] for e in ev] for it, ev in dev.ev.items()}


def _counts(r):
    return (int(r.n_children), int(r.n_sources), int(r.n_seeds), int(r.n_clusters))


def _check_record(got, want, i):
    assert (emulib.paf_tuple(got), _counts(got)) == (orclib.paf_tuple(want), _counts(want)), i
    assert got.status == 0, (i, got.status)


def _row_str(r):
    if not r["valid"]:
        return "dup"
    sp, c = np.array([r["seed_prob"], r["prob_sum"]], np.uint32).view(np.float32)
    return ("fm [%d, %d] kmer %d len %d stays %d sa_checked %d moves %#x seed_prob %r C %r"
            % (r["fm_start"], r["fm_end"], r["kmer"], r["length"], r["consec_stays"], r["sa_checked"], r["event_moves"],
               float(sp), float(c)))


def _explain(item, k, run_dev, run_orc):
    """Both sides again, keeping the item's k-th event whole: where do they first differ?"""
    d, o = run_dev((item, k))[0].kept, run_orc((item, k))[0].kept
    if d is None or o is None:
        return "only the %s reports event #%d" % ("device" if o is None else "oracle", k)
    (ev, dr, ds, df, dov), (_, orw, osd, of, _) = d, o
    msg = ["event %d (#%d of item %d): nn %d / %d" % (ev, k, item, len(dr), len(orw))]
    for i in range(min(len(dr), len(orw))):
        if dr[i] != orw[i]:
            msg.append("first differing position %d:\n  device %s\n  oracle %s" % (i, _row_str(dr[i]), _row_str(orw[i])))
            break
    if len(ds) != len(osd) or not np.array_equal(ds, osd):
        j = next((j for j in range(min(len(ds), len(osd))) if ds[j] != osd[j]), min(len(ds), len(osd)))
        msg.append("seeds %d / %d, first differing %d: device %s oracle %s"
                   % (len(ds), len(osd), j, ds[j] if j < len(ds) else None, osd[j] if j < len(osd) else None))
    if not np.array_equal(df, of):
        w = int(np.nonzero(df != of)[0][0])
        msg.append("sources_added_ word %d: device %#010x oracle %#010x" % (w, df[w], of[w]))
    if dov:
        msg.append("device overflow flag set")
    return "\n".join(msg)


def _compare(dev, orc, run_dev, run_orc, label):
    """Every item's events, in order."""
    assert set(dev.ev) == set(orc.ev), (label, sorted(dev.ev), sorted(orc.ev))
    for item in sorted(orc.ev):
        d, o = dev.ev[item], orc.ev[item]
        for k in range(max(len(d), len(o))):
            if k >= len(d) or k >= len(o) or d[k] != o[k]:
                pytest.fail("%s, item %d: %s" % (label, item, _explain(item, k, run_dev, run_orc)))


# ---------------------------------------------------------------------------------------------------- inputs

GENOMES = ("g200k", "g4m7")
# max_paths -> worker CTA shape (warps, the tracker included): 14 is the product's (unc_abi.cu K2_WARPS)
EDGES = {1: 8, 2: 2, 31: 8, 32: 5, 33: 2, 159: 8, 160: 14, 161: 5, 300: 8, 10000: 14}
MAPS, NEVER = (1, 2), (4, 0)            # of synth.reads(g, 8, 4000, seed=11, frac_random=0.4): map early / never map


def _reads(name, ids):
    prefix, g = synthdata.get_index(name)
    sig, truth = synth.reads(g, 8, 4000, seed=11, frac_random=0.4)
    assert all(truth["random"][i] for i in NEVER) and not any(truth["random"][i] for i in MAPS)
    return prefix, [np.ascontiguousarray(sig[i], np.float32) for i in ids]


_TAB = np.fromfile(synth.MODEL_TABLE, np.float32).reshape(1024, 2)


def _homopolymer_read(g, i, base, n=3000):
    """1500 samples of a read of the genome (so that the read normalises to the model), then n samples of one
    homopolymer's level in blocks of 8 samples alternating by +-0.3 level stdv, with 0.1 stdv noise."""
    sig, _ = synth.reads(g, 4, 2500, seed=5, frac_random=0.0)
    rng = np.random.default_rng(1 + i)
    m, sd = _TAB[sum(base << (2 * j) for j in range(5))]
    lv = m + np.where(np.arange(n // 8) % 2, 0.3, -0.3) * sd
    tail = np.repeat(lv, 8) + rng.standard_normal(n // 8 * 8) * sd * 0.1
    return np.ascontiguousarray(np.concatenate([sig[i][:1500], tail]), np.float32)


def _low_complexity_reads():
    prefix, g = synthdata.get_low_complexity_index()
    return prefix, [_homopolymer_read(g, 0, 0), _homopolymer_read(g, 1, 3)]


# ---------------------------------------------------------------------------------------------------- tests

@pytest.mark.parametrize("max_paths", sorted(EDGES))
@pytest.mark.parametrize("name", GENOMES)
def test_default_kernel_every_event_at_the_max_paths_edges(name, max_paths):
    """Two reads that map early and one that never maps, on both sides of the pack (32), chunk (160) and walk-window
    sizes, at 200 events."""
    prefix, sigs = _reads(name, MAPS + NEVER[:1])
    P = Pair(prefix)
    P.set(max_paths=max_paths, max_events=200)
    recs, want, nn = P.batch(sigs, n_warps=EDGES[max_paths])
    assert max(max(v) for v in nn.values()) == max_paths or max_paths == 10000, nn
    if name == "g200k" and max_paths >= 160:
        assert sum(r.mapped for r in want) >= 1


def test_max_paths_32767_at_the_cap():
    """The largest max_paths unc_check_params accepts, on reads that never map: the buffer sits at the cap, and the cap
    cuts the children inside a 160-slot chunk."""
    prefix, sigs = _reads("g4m7", NEVER)
    P = Pair(prefix)
    P.set(max_paths=32767, max_events=240)
    recs, want, nn = P.batch(sigs, n_warps=14)
    assert max(nn[0]) == 32767, {k: max(v) for k, v in nn.items()}     # from event 226 on
    assert P.shapes["cut_in_chunk"] + P.shapes["cut_at_chunk"] > 0, P.shapes


def test_exact_ties_kernel_every_event():
    """The exact-ties kernel (the reference's pdqsort on the event's keys) against the oracle's pdqsort, on reads whose
    events contain ties (read 36 of this set: the tie order decides a seed) and on small buffers and CTAs."""
    prefix, g = synthdata.get_index("g4m7")
    sig, _ = synth.reads(g, 600, 4000, seed=7, frac_random=0.15)
    P = Pair(prefix, exact=True)
    stats = (C.c_ulong * 2)()
    P.E.L.emu_tie_stats(stats, 1)
    for max_paths, n_warps, ids in ((10000, 8, (36, 3)), (300, 5, (36,)), (33, 2, (36,))):
        P.set(max_paths=max_paths, max_events=150)
        P.batch([np.ascontiguousarray(sig[i], np.float32) for i in ids], n_warps=n_warps)
    P.E.L.emu_tie_stats(stats, 1)
    assert 0 < stats[1] < stats[0], tuple(stats)
    assert P.shapes["recount"] == stats[1], (P.shapes["recount"], tuple(stats))


@pytest.mark.parametrize("chunk_len", [450, 4000])
def test_streaming_every_event(chunk_len):
    """The streaming kernel: events continue across chunks (and across the reads of a channel); 2 channels."""
    prefix, g = synthdata.get_index("g200k")
    sig, _ = synth.reads(g, 4, 5000, seed=5, frac_random=0.3)
    P = Pair(prefix)
    P.set(max_events=300)
    res, want, nn = P.stream([sig[i][:5000 - 37 * i] for i in range(4)], 2, chunk_len, n_warps=5)
    assert len(nn) == 2 and any(r is not None and r[3].mapped for r in res)


def test_streaming_at_max_paths_32767():
    """The streaming kernel's per-channel slots at the largest buffer, on reads that never map."""
    prefix, sigs = _reads("g4m7", NEVER)
    P = Pair(prefix)
    P.set(max_paths=32767, max_events=240)
    res, want, nn = P.stream(sigs, 2, 450, n_warps=14)
    assert max(max(v) for v in nn.values()) > 32000, {k: max(v) for k, v in nn.items()}   # 32 689: the buffer near its cap


def test_low_complexity_genome():
    """Homopolymer and tandem-repeat stretches (synthdata.low_complexity_genome): huge buckets, buckets whose keys all
    share one fm_start (no radix pass), buckets spanning more than 2^16 rows (three passes) and long equal-fm_start
    runs across 32-key chunks."""
    prefix, sigs = _low_complexity_reads()
    P = Pair(prefix)
    P.set(max_paths=300, max_events=500)
    P.batch(sigs, n_warps=8)
    for k in ("huge", "pass0", "pass3", "eq_run_cross"):
        assert P.shapes[k] > 0, (k, P.shapes)


def test_cluster_store_reuses_emptied_blocks():
    """Regression: the seed tracker's store of 32-cluster blocks never reused a block that an erase had emptied, so a read
    whose clusters churn for long ran out of blocks with few clusters alive and failed with status -7 (found on the GPU:
    the low-complexity genome's second read at max_paths 10 000, 875 live clusters, 6 032 blocks gone by event 639).
    With 16 blocks, the same read at max_paths 1 000 ran out at event 353 with 103 clusters alive; it now maps on to the
    event limit exactly as the oracle does, with 121 clusters alive at the end."""
    prefix, sigs = _low_complexity_reads()
    P = Pair(prefix)
    P.set(max_paths=1000, max_events=360)
    recs, want, nn = P.batch(sigs[1:], max_blocks=16)
    assert len(nn[0]) == 360 and want[0].n_clusters > 103


def test_every_bucket_shape_is_reached():
    """A compact set of the inputs above, traced like the rest, reaches every edge the emulator build counts (all but a
    fourth radix pass, which needs a k-mer range of 2^24 rows)."""
    shapes = collections.Counter()
    for name, max_paths, n_warps, ids, events in (("g200k", 1, 8, MAPS, 60), ("g200k", 2, 2, MAPS, 60),
                                                  ("g200k", 33, 2, MAPS, 100), ("g4m7", 10000, 14, MAPS, 120)):
        prefix, sigs = _reads(name, ids)
        P = Pair(prefix)
        P.set(max_paths=max_paths, max_events=events)
        P.batch(sigs, n_warps=n_warps)
        shapes.update(P.shapes)
    prefix, sigs = _low_complexity_reads()
    P = Pair(prefix)
    P.set(max_paths=300, max_events=500)
    P.batch(sigs)
    shapes.update(P.shapes)
    prefix, g = synthdata.get_index("g4m7")
    sig, _ = synth.reads(g, 600, 4000, seed=7, frac_random=0.15)
    P = Pair(prefix, exact=True)
    P.set(max_events=120)
    P.batch([np.ascontiguousarray(sig[36], np.float32)])
    shapes.update(P.shapes)
    missing = [k for k in emulib.K2_SHAPES if k != "pass4" and shapes[k] == 0]
    assert not missing, (missing, dict(shapes))
