"""The streaming path on long-lived channels: the streaming normaliser (Normalizer, length 6000) past its first pass
around the ring, where Normalizer::push switches from Welford updates to the rolling update and its cursor wr_ wraps.

On a flow cell every channel keeps one Mapper, and so one normaliser, for the whole run; after about 30 000 samples
every chunk's scale and shift come from the rolling branch.  Here channels run through two or more passes around the
ring, and after every read both the records and the normaliser state (mean_, varsum_, n_, wr_) are compared, bit for bit:

1. the oracle's channel mode against the reference's own Mapper (oracle/_ref, live where it is built, else the stored
   digest of its results);
2. the device source under the warp emulator against the oracle, its ring against the event means it pushed, and both
   statistics against an exact computation over the window that does not use the recurrence;
3. on the GPU, unc_stream_step over 64 channels against the oracle: float32 and int16 DAC chunks, 450- and
   4000-sample chunks, and the exact-ties kernel against the oracle's pdqsort mode.
"""
import json
import os
from fractions import Fraction

import numpy as np
import pytest

import orclib
import synth
import synthdata

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NORM_LEN = 6000                  # Normalizer::PRMS_DEF.len
MAPPING = 1                      # UNC_STREAM_MAPPING
CAL = (1467.61, 10.0, 8192.0)    # (range, offset, digitisation) of the int16 runs


def _chunk_len(chunk_time):
    return int(np.float32(chunk_time) * np.float32(4000.0))      # ReadBuffer::PRMS.chunk_len()


def _mixed(g, n_random, n_genome, n_samples, seed, chunk_len):
    """n_random reads that never map (they keep the channel pushing events) and n_genome reads from the genome, in a
    seeded order, each cut short by up to one chunk so that it ends inside a chunk."""
    a, _ = synth.reads(g, n_random, n_samples, seed=seed, frac_random=1.0)
    b, _ = synth.reads(g, n_genome, n_samples, seed=seed + 1, frac_random=0.0)
    rng = np.random.default_rng(seed)
    reads = [a[i] for i in range(n_random)] + [b[i] for i in range(n_genome)]
    reads = [reads[i] for i in rng.permutation(len(reads))]
    return [np.ascontiguousarray(s[:n_samples - int(rng.integers(0, chunk_len))]) for s in reads]


def _boundary_channel(g, O):
    """A 450-sample-chunk channel one of whose reads ends exactly with the normaliser's 6000th push (n_ reaches the ring
    length on the last event of a chunk, wr_ wraps to 0), followed by more reads.  The first read is cut to the number of
    chunks that puts 6000 on a chunk boundary, and the read holding that boundary is cut there."""
    rnd, _ = synth.reads(g, 12, 9000, seed=109, frac_random=1.0)
    q = [O.chunk_pushes(s, 450) for s in rnd]
    for j in range(len(q[0]), 0, -1):
        tot = 0
        for i, qi in enumerate(q):
            qq = qi[:j] if i == 0 else qi
            hit = np.nonzero(tot + qq.astype(np.int64) == NORM_LEN)[0]
            if hit.size:
                reads = [rnd[0][:450 * j]] + [rnd[r] for r in range(1, i)] + [rnd[i][:450 * (int(hit[0]) + 1)]]
                reads = [np.ascontiguousarray(s) for s in reads]
                if i == 0:
                    reads = reads[1:]
                return reads + _mixed(g, 4, 4, 9000, 111, 450)
            tot += int(qq[-1])
            if tot >= NORM_LEN:
                break
    raise AssertionError("no chunk boundary at push 6000")


def _channels():
    """The channels of the reference pin: (name, chunk_time, max_chunks, reads)."""
    prefix, g = synthdata.get_index("g200k")
    O = orclib.Oracle(prefix)
    boundary = _boundary_channel(g, O)
    a, _ = synth.reads(g, 20, 9000, seed=101, frac_random=0.5)
    b, _ = synth.reads(g, 6, 30000, seed=102, frac_random=0.5)
    c, _ = synth.reads(g, 64, 4000, seed=103, frac_random=0.5)
    return prefix, [("chunks450", 0.1125, 1000000, [np.ascontiguousarray(s) for s in a]),
                    ("chunks4000", 1.0, 1000000, [np.ascontiguousarray(s) for s in b]),
                    ("chunks450_max7", 0.1125, 7, [np.ascontiguousarray(s) for s in c]),
                    ("boundary450", 0.1125, 1000000, boundary)]


def _state_key(state):
    return [[float(v).hex() for v in row] for row in state]


def _oracle_channel_results(O, reads, chunk_len, max_chunks):
    res, state, pushed = O.stream_channel_norm(reads, chunk_len, max_chunks)
    return [[list(orclib.paf_tuple(r)), int(nu), int(en)] for r, nu, en in res], state, pushed


def _ref_results():
    """The reference's own Mapper (oracle/_ref) over the channels of _channels(): per channel, per read, the records and
    the normaliser state.  Runs in the process that loaded oracle/_ref."""
    import ctypes as C
    R = orclib.ref()
    prefix, chans = _channels()
    assert R.ref_load(prefix.encode(), b"default") == 0
    out = {}
    for name, ct, mc, reads in chans:
        flat = np.ascontiguousarray(np.concatenate(reads), np.float32)
        lens = np.array([len(s) for s in reads], np.uint32)
        offs = np.concatenate([[0], np.cumsum(lens[:-1], dtype=np.uint64)]).astype(np.uint64)
        n = len(reads)
        recs, nu, en = (orclib.RefPaf * n)(), (C.c_uint32 * n)(), (C.c_int32 * n)()
        state = np.zeros((n, 4), np.float64)
        R.ref_stream_channel_norm(orclib.fp(flat), offs.ctypes.data_as(orclib.u64p), lens.ctypes.data_as(orclib.u32p), n,
                                  ct, mc, recs, nu, en, state.ctypes.data)
        out[name] = {"recs": [[list(orclib.paf_tuple(recs[i])), int(nu[i]), int(en[i])] for i in range(n)],
                     "state": _state_key(state)}
    return out


LIVE = r"""
import json, sys
sys.path[:0] = [%r, %r]
import test_stream_long_channels as T
print("REF-JSON " + json.dumps(T._ref_results()))
"""


def _chunk_boundaries(O, reads, results, chunk_len):
    """The channel's normaliser push counts at the end of every chunk it consumed."""
    out, tot = [], 0
    for s, (_, nu, _) in zip(reads, results):
        cp = O.chunk_pushes(s, chunk_len, nu).astype(np.int64)
        out += list(tot + cp)
        tot += int(cp[-1]) if nu else 0
    return out


def test_oracle_channel_mode_and_normaliser_match_reference():
    """orc_stream_map_channel against ref_stream_channel_norm: the records, chunks used, `ended` and the normaliser's
    (mean_, varsum_, n_, wr_) after every read, bit for bit.  450- and 4000-sample chunks, max_chunks 7 (reads end
    before their signal does), half the reads never mapping, and channels whose 6000th push falls inside a chunk and
    exactly on the last event of one."""
    prefix, chans = _channels()
    O = orclib.Oracle(prefix)
    got = {}
    for name, ct, mc, reads in chans:
        recs, state, pushed = _oracle_channel_results(O, reads, _chunk_len(ct), mc)
        got[name] = {"recs": recs, "state": _state_key(state)}
        assert pushed[-1] >= 2 * NORM_LEN, (name, pushed[-1])                       # at least two passes around the ring
        assert all(s[2] == NORM_LEN for s, p in zip(state, pushed) if p >= NORM_LEN), name
        assert all(s[3] == p % NORM_LEN for s, p in zip(state, pushed)), name            # wr_ = pushes mod 6000
        bnd = _chunk_boundaries(O, reads, [(None, r[1], None) for r in recs], _chunk_len(ct))
        assert bnd[-1] == pushed[-1], name
        if name == "chunks450":
            assert NORM_LEN not in bnd                                                   # the 6000th push is mid-chunk
        if name == "boundary450":
            i = list(pushed).index(NORM_LEN)                                              # a read ends on push 6000
            assert state[i][2] == NORM_LEN and state[i][3] == 0
        if name == "chunks450_max7":
            assert any(r[1] == 7 and not r[0][0] for r in recs)                          # given up at max_chunks
    live = orclib.ref_available("ref_stream_channel_norm")
    if live:
        out = orclib.run_in_subprocess(LIVE % (os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")))
        want = json.loads(out.split("REF-JSON ", 1)[1])
        for name in got:
            for i, (a, b) in enumerate(zip(got[name]["recs"], want[name]["recs"])):
                assert a == b, (name, i, a, b)
            for i, (a, b) in enumerate(zip(got[name]["state"], want[name]["state"])):
                assert a == b, (name, i, a, b)
            assert len(got[name]["recs"]) == len(want[name]["recs"])
    orclib.expect_reference("stream/long_channels_norm", json.dumps(got, sort_keys=True), live=live)


# ---------------------------------------------------------------------------------------------- emulated device source
class _StateRecorder:
    """Wraps a stream's step: after a step in which a channel's read finishes, reads that channel's normaliser through
    `norm_state(channel)`, so that the state after every read can be compared.  With `cal`, the float32 chunks (integer
    DAC values) are handed on as int16 chunks to be calibrated on the device."""

    def __init__(self, step, norm_state, cal=None):
        self.inner, self.norm_state, self.cal = step, norm_state, cal
        self.after = {}

    def __call__(self, descs, n, flat, res):
        if self.cal is not None:
            flat = flat.astype(np.int16)
            for i in range(n):
                descs[i].dtype = 1
                descs[i].cal_range, descs[i].cal_offset, descs[i].cal_digit = self.cal
        self.inner(descs, n, flat, res)
        for i in range(n):
            if res[i].state != MAPPING:
                c = descs[i].channel
                self.after.setdefault(c, []).append(self.norm_state(c))


def _exact_window(pushed):
    """mean and sum of squared deviations of the last min(len(pushed), 6000) pushed means, in exact arithmetic."""
    w = [Fraction(float(x)) for x in pushed[-NORM_LEN:]]
    mean = sum(w, Fraction(0)) / len(w)
    return mean, sum(((x - mean) ** 2 for x in w), Fraction(0))


# the exact check's relative tolerance on mean_ and varsum_ (see test_emulated_long_channel_normaliser_state)
EXACT_RTOL = 1e-9


def test_emulated_long_channel_normaliser_state():
    """One channel of 20 reads in 4000-sample chunks (about 15 000 pushes, 2.5 passes around the ring), the device
    source under the warp emulator; max_paths 300 and max_events 300 keep the mapping short.  After every read:

    - records, chunks used and `ended` equal the oracle's, and so does (mean, varsum, n, wr), bit for bit;
    - the ring holds the last 6000 event means the channel pushed, wr pointing past the newest;
    - mean and varsum agree with the exact mean and sum of squared deviations of the window (fractions.Fraction over
      the last min(pushes, 6000) pushed means) to a relative EXACT_RTOL = 1e-9.  Measured on this channel: the
      recurrence drifts from the exact values by at most 3.7e-15 (mean) and 3.7e-15 (varsum), relative; a window that
      holds one stale event in place of the newest one is off by 6.4e-6 to 6.8e-5 (mean) and 3.4e-6 to 4.1e-4
      (varsum), after every read past the first 6000 pushes.
    """
    import emulib
    prefix, g = synthdata.get_index("g200k")
    E, O = emulib.Emu(prefix), orclib.Oracle(prefix)
    E.params.max_paths = O.params.max_paths = 300
    E.params.max_events = O.params.max_events = 300
    reads = _mixed(g, 12, 8, 12000, 121, 4000)
    ES = emulib.EmuStream(E, 1, 4000)
    rec = _StateRecorder(ES.step, lambda c: ES.norm_state(c, ring=True, pushed=True))
    res = emulib.stream_reads(rec, 1, reads, 4000)
    ES.close()
    want, ostate, opushed = O.stream_channel_norm(reads, 4000)
    assert opushed[-1] >= 2 * NORM_LEN
    bad_rec = [i for i, (r, (w, nu, en)) in enumerate(zip(res, want))
               if (emulib.paf_tuple(r[3]), r[2], r[1]) != (orclib.paf_tuple(w), nu, en)]
    after = rec.after[0]
    assert len(after) == len(reads)
    bad_state = [i for i, (a, b) in enumerate(zip(after, ostate)) if a[0].view(np.uint64).tolist() != b.view(np.uint64).tolist()]
    assert not bad_rec and not bad_state, ("records differ after reads %s, normaliser state after reads %s" % (bad_rec, bad_state))
    worst = [0.0, 0.0]
    for i, (st, ring, pushed) in enumerate(after):
        P = len(pushed)
        assert P == opushed[i], i
        k = min(P, NORM_LEN)
        assert (st[2], st[3]) == (k, P % NORM_LEN), i
        assert np.array_equal(np.roll(ring, -int(st[3]))[NORM_LEN - k:], pushed[P - k:]), i
        mean, varsum = _exact_window(pushed)
        em = abs(Fraction(float(st[0])) - mean) / abs(mean)
        ev = abs(Fraction(float(st[1])) - varsum) / varsum
        assert em < EXACT_RTOL and ev < EXACT_RTOL, (i, float(em), float(ev))
        worst = [max(worst[0], float(em)), max(worst[1], float(ev))]
    print("normaliser pushes %d, worst relative drift from the exact window: mean %.2g, varsum %.2g"
          % (opushed[-1], worst[0], worst[1]))


# ---------------------------------------------------------------------------------------------- the GPU
N_CHANNELS = 64


def _gpu_reads(chunk_len):
    """Per channel, 7 reads that never map and 6 from the genome, 12000 samples each; read i on channel i % 64."""
    _, g = synthdata.get_index("g200k")
    per = [_mixed(g, 7, 6, 12000, 1000 + 2 * c, chunk_len) for c in range(N_CHANNELS)]
    return [per[i % N_CHANNELS][i // N_CHANNELS] for i in range(13 * N_CHANNELS)]


def _to_dac(s):
    raw = np.clip(np.round(s.astype(np.float64) * CAL[2] / CAL[0] - CAL[1]), -50, 32000).astype(np.int16)
    return raw


def _calibrate(raw):
    """pA as the device calibrates an int16 chunk (read_buffer.cpp: u16 reinterpretation), in float32."""
    return ((np.float32(CAL[0]) * (raw.astype(np.uint16).astype(np.float32) + np.float32(CAL[1]))) /
            np.float32(CAL[2])).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("chunk_len,dtype,tie_order", [(450, 0, 0), (4000, 0, 0), (450, 1, 0), (4000, 1, 0), (450, 0, 1)],
                         ids=["f32-450", "f32-4000", "i16-450", "i16-4000", "exact-ties-450"])
def test_device_long_channels_match_oracle(chunk_len, dtype, tie_order):
    """unc_stream_step on 64 channels of 13 reads each, every channel at least two passes around the normaliser's ring,
    against the oracle's channel mode (run on a process pool): records, chunks used and `ended` of every read, and the
    channel's normaliser state after every read through unc_stream_channel_norm, bit for bit.  dtype 1: the reads as
    int16 DAC chunks calibrated on the device, the oracle given the same calibration in float32.  tie_order 1: the
    exact-ties kernel against the oracle with the reference's pdqsort child sort."""
    import multiprocessing

    import uncalled_b200 as U
    prefix, _ = synthdata.get_index("g200k")
    reads = _gpu_reads(chunk_len)
    if dtype == 1:
        dac = [_to_dac(s) for s in reads]
        for r in dac[:N_CHANNELS]:
            r[50:53] = -7                           # negative DAC values: u16 wrap, rejected by max_mean
        fed, orc_reads = [r.astype(np.float32) for r in dac], [_calibrate(r) for r in dac]
    else:
        fed, orc_reads = reads, reads
    jobs = [(prefix, [orc_reads[i] for i in range(c, len(reads), N_CHANNELS)], chunk_len, tie_order) for c in range(N_CHANNELS)]
    ctx = multiprocessing.get_context("spawn")
    with ctx.Pool(min(os.cpu_count() or 1, N_CHANNELS)) as pool:
        pending = pool.map_async(orclib.stream_channel_job, jobs)
        idx = U.Index(prefix, device=0)
        sm = U.StreamMapper(idx, N_CHANNELS, chunk_len)
        if tie_order:
            sm.set_tie_order(tie_order)
        rec = _StateRecorder(sm.step, sm.norm_state, CAL if dtype == 1 else None)
        res = U.feed_reads(rec, N_CHANNELS, fed, chunk_len)
        sm.close()
        want = pending.get(timeout=1800)
    pushes = []
    for c, (owant, ostate, opushed) in enumerate(want):
        idxs = list(range(c, len(reads), N_CHANNELS))
        for k, (i, (paf, nu, en, ns)) in enumerate(zip(idxs, owant)):
            r = res[i]
            assert r is not None and (U.paf_key(r[3]), r[2], r[1]) == (tuple(paf), nu, en), (c, k)
            assert (r[3].n_children, r[3].n_sources, r[3].n_seeds) == ns, (c, k)
            assert r[3].status == 0
        got = np.array(rec.after[c], np.float64)
        assert got.shape == ostate.shape, c
        bad = [k for k in range(len(idxs)) if got[k].view(np.uint64).tolist() != ostate[k].view(np.uint64).tolist()]
        assert not bad, ("normaliser state differs", c, bad[0], got[bad[0]].tolist(), ostate[bad[0]].tolist())
        pushes.append(int(opushed[-1]))
    print("normaliser pushes per channel (%s, chunk %d, tie_order %d): min %d, median %d, max %d"
          % ("int16" if dtype else "float32", chunk_len, tie_order, min(pushes), int(np.median(pushes)), max(pushes)))
    assert min(pushes) >= 2 * NORM_LEN
