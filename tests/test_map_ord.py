"""`map-ord` on the CPU: the ordering logic of MapPoolOrd (reference src/map_pool_ord.cpp:48-121) on in-memory reads,
the device replay source (unc_replay.cuh) under the warp emulator against the oracle's channel mode and against the
host-stepped loop over the emulated unc_stream_step, windows, and the command line."""
import ctypes as C
import io
import os
import shutil
import sys

import numpy as np
import pytest

import orclib
import replaylib as RL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F5 = os.path.join(ROOT, "tests", "golden", "fast5")
MAPPING, FAILURE = 1, 3


def _conf(**kw):
    from uncalled_b200 import api
    c = api.Conf()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


# ------------------------------------------------------------------------------------------------ ordering logic
class _FakeReplay:
    """Stands in for the device: every read takes ceil(n / L) chunk steps and then the "no more signal" step (the
    lockstep loop's step count for a read that never maps); records the windows it is given."""

    def __init__(self, n_channels, L):
        self.L, self.steps, self.windows = L, [0] * n_channels, []

    def replay(self, reads, n, flat, out):
        self.windows.append([(reads[i].channel, reads[i].number, reads[i].n_samples, reads[i].offset) for i in range(n)])
        res = []
        for i in range(n):
            r = reads[i]
            k = -(-int(r.n_samples) // self.L)
            step = self.steps[r.channel] + k
            self.steps[r.channel] = step + 1
            res.append((step, 0, r.channel, i, k))
        for o, (step, kind, ch, i, k) in zip(out, sorted(res)):
            o.read, o.number, o.step, o.kind = i, reads[i].number, step, kind
            o.res.state, o.res.ended, o.res.chunks = FAILURE, 1, k
            o.res.rec.rd_len = int(reads[i].n_samples)
        return 0


class _Seqs:
    seqs = [("chr", 1000)]


def _pool(conf, reads, window_samples=1 << 28):
    from uncalled_b200 import api
    L = int(np.float32(conf.chunk_time) * np.float32(conf.sample_rate)) & 0xFFFF
    fake = _FakeReplay(conf.num_channels, L)
    pool = api.MapPoolOrd(conf, backend=fake, index=_Seqs(), window_samples=window_samples)
    for rid, ch, nm, st, n in reads:
        pool.queue_read(rid, np.zeros(n, np.int16), ch, nm, st, calibration=(1.0, 0.0, 1.0))
    return pool, fake


def _drain(pool):
    """update() until running() is false; nothing may come after that."""
    out = []
    while pool.running():
        out += pool.update()
    assert pool.update() == [] and not pool.running()
    return out


def test_reads_are_grouped_by_channel_and_sorted_by_start_with_ties_in_input_order():
    conf = _conf(num_channels=4, chunk_time=0.1125)
    reads = [("a", 2, 1, 900, 900), ("b", 2, 2, 100, 900), ("c", 1, 3, 500, 900), ("d", 2, 3, 100, 450),
             ("e", 4, 4, -5, 450), ("f", 4, 5, 7, 450)]
    pool, fake = _pool(conf, reads, window_samples=1)
    _drain(pool)
    per_ch = {}
    for w in fake.windows:
        for ch, nm, n, _ in w:
            per_ch.setdefault(ch, []).append(nm)
    # channel 2: b and d share start 100 (input order), a starts later; channel 4: start -5 is 2^64 - 5 as the
    # reference's u64 start_sample_, so it sorts after 7
    assert per_ch == {0: [3], 1: [2, 3, 1], 3: [5, 4]}
    assert all(len(w) == 1 for w in fake.windows)        # a window holds at least one read, even over its budget


def test_signals_are_cut_to_max_chunks_and_reads_without_samples_are_skipped():
    conf = _conf(num_channels=2, chunk_time=0.1125, max_chunks=3)
    pool, fake = _pool(conf, [("a", 1, 1, 0, 5000), ("b", 1, 2, 10, 0), ("c", 2, 3, 0, 1000)])
    out = _drain(pool)
    assert sorted((ch, n) for w in fake.windows for ch, _, n, _ in w) == [(0, 1350), (1, 1000)]
    assert sorted(p.rd_name for p in out) == ["a", "c"]
    assert {p.rd_name: p.chunks for p in out} == {"a": 3, "c": 3}


def test_min_active_reads_stops_the_run_after_the_first_step_below_it():
    """Channel 1: reads of 2 and 1 chunks (steps 0-2 and 3-4, each ending with the "no more signal" step); channel 2:
    one read of 5 chunks (steps 0-5).  After step 2 only channel 2 has a read in progress: with min_active_reads 2 the
    run stops there and the reads finished later are not reported.  Windows of one read hold results back until every
    channel's activity up to their step is known."""
    L = 450
    reads = [("a", 1, 1, 0, 2 * L), ("b", 1, 2, 1, L), ("c", 2, 3, 0, 5 * L)]
    for m, want in ((0, {"a", "b", "c"}), (1, {"a", "b", "c"}), (2, {"a"}), (3, set())):
        conf = _conf(num_channels=2, chunk_time=0.1125, min_active_reads=m)
        pool, _ = _pool(conf, reads, window_samples=L)
        assert {p.rd_name for p in _drain(pool)} == want, m
        assert not pool.running()


def test_host_loop_chunks_partial_last_chunk_and_empty_chunk_reset():
    """The host-stepped loop hands a read its chunks from get_chunk: full ones, the partial last one, then the empty
    chunk (request_reset) until the read is finished; the next read starts at the following update."""
    from uncalled_b200 import api
    seen = []

    class Step:
        def step(self, descs, n, flat, res):
            for i in range(n):
                d = descs[i]
                seen.append((d.channel, d.new_read, d.n_samples))
                res[i].state = FAILURE if d.n_samples == 0 else MAPPING
                res[i].ended = 1 if d.n_samples == 0 else 0

    conf = _conf(num_channels=2, chunk_time=0.1125)
    pool = api.RealtimePool(conf, backend=Step(), index=_Seqs())
    reads = [RL.Read("a", 1, 1, 0, np.zeros(1000, np.float32)), RL.Read("b", 1, 2, 5, np.zeros(450, np.float32)),
             RL.Read("c", 2, 3, 0, np.zeros(500, np.float32))]
    out = RL.host_map_ord(pool, RL.order_channels(reads, 2), 450)
    assert [(u, p.rd_name) for u, p in out] == [(2, "c"), (3, "a"), (5, "b")]
    assert [s for s in seen if s[0] == 0] == [(0, 1, 450), (0, 0, 450), (0, 0, 100), (0, 0, 0), (0, 1, 450), (0, 0, 0)]
    assert [s for s in seen if s[0] == 1] == [(1, 1, 450), (1, 0, 50), (1, 0, 0)]


def test_channel_outside_num_channels_is_an_error_before_the_device():
    conf = _conf(num_channels=2)
    pool, fake = _pool(conf, [("a", 3, 1, 0, 900)])
    with pytest.raises(ValueError, match="channel 3"):
        pool.update()
    assert fake.windows == []


# ------------------------------------------------------------------------------------------------ emulated device
@pytest.fixture(scope="module")
def emu():
    import synthdata
    prefix, g = synthdata.get_index("g200k")
    return prefix, g, RL.EmuReplay(prefix), orclib.Oracle(prefix)


def _emu_map_ord(E, seqs, conf, reads, window_samples=1 << 28, tie_order=0):
    from uncalled_b200 import api
    L = int(np.float32(conf.chunk_time) * np.float32(conf.sample_rate)) & 0xFFFF
    E.L.emu_set_tie_order(tie_order)
    pool = api.MapPoolOrd(conf, backend=RL.EmuReplayStream(E, conf.num_channels, L, max_chunks=conf.max_chunks),
                          index=RL.SeqIndex(seqs), window_samples=window_samples)
    for r in reads:
        pool.queue_read(r.id, r.signal, r.channel, r.number, r.start, r.cal)
    out, calls = [], 0
    while pool.running():
        out += pool.update()
        calls += 1
    pool.stop()
    E.L.emu_set_tie_order(0)
    return out, calls


def _emu_host(E, seqs, conf, reads, tie_order=0):
    from uncalled_b200 import api
    L = int(np.float32(conf.chunk_time) * np.float32(conf.sample_rate)) & 0xFFFF
    E.L.emu_set_tie_order(tie_order)
    pool = api.RealtimePool(conf, backend=RL.EmuReplayStream(E, conf.num_channels, L, max_chunks=conf.max_chunks),
                            index=RL.SeqIndex(seqs))
    out = RL.host_map_ord(pool, RL.order_channels(reads, conf.num_channels, conf.max_chunks * L), L)
    E.L.emu_set_tie_order(0)
    return [p for _, p in out]


@pytest.mark.parametrize("chunk_time,max_chunks,tie_order", [(0.1125, 1000000, 0), (1.0, 1000000, 0), (0.1125, 7, 0),
                                                             (0.1125, 1000000, 1)])
def test_emulated_replay_matches_oracle_channel_mode(emu, chunk_time, max_chunks, tie_order):
    """Two channels x three int16 reads of whole chunks: records, chunks used and `ended` equal the oracle's channel
    mode (child_sort 1 for the exact-ties kernel)."""
    prefix, g, E, O = emu
    L = int(np.float32(chunk_time) * np.float32(4000.0))
    reads = RL.synthetic_run(g, 2, 3, 9000, seed=7 + tie_order, int16=True, whole_chunks=L)
    conf = _conf(num_channels=2, chunk_time=chunk_time, max_chunks=max_chunks)
    out, _ = _emu_map_ord(E, RL.seqs_of(O), conf, reads, tie_order=tie_order)
    by_id = {p.rd_name: p for p in out}
    O.lib.orc_set_child_sort(tie_order)
    try:
        for q in RL.order_channels(reads, 2):
            want = O.stream_channel([RL.pcal(r.signal, r.cal) for r in q], L, max_chunks)
            for r, (rec, nu, en) in zip(q, want):
                p = by_id[r.id]
                assert (orclib.paf_tuple(p.rec), p.chunks, int(p.is_ended())) == (orclib.paf_tuple(rec), nu, en), r.id
    finally:
        O.lib.orc_set_child_sort(0)
    if max_chunks == 7:
        assert any(p.chunks == 7 for p in out)


def test_emulated_replay_passes_the_normaliser_ring_like_the_oracle(emu):
    """One channel whose reads push more than 6000 events into its normaliser (the ring wraps mid-run)."""
    prefix, g, E, O = emu
    L = 450
    import synth
    sigs, _ = synth.reads(g, 8, 9000, seed=101, frac_random=0.75)     # unmapped reads push every event of their signal
    reads = [RL.Read("r%d" % i, 1, i, 10 * i, np.round(np.asarray(s) * RL.CAL[2] / RL.CAL[0] - RL.CAL[1]).astype(np.int16),
                     RL.CAL) for i, s in enumerate(sigs)]
    conf = _conf(num_channels=1, chunk_time=0.1125)
    out, _ = _emu_map_ord(E, RL.seqs_of(O), conf, reads)
    q = RL.order_channels(reads, 1)[0]
    want, _, pushed = O.stream_channel_norm([RL.pcal(r.signal, r.cal) for r in q], L)
    assert pushed[-1] > 6000
    by_id = {p.rd_name: p for p in out}
    for r, (rec, nu, en) in zip(q, want):
        p = by_id[r.id]
        assert (orclib.paf_tuple(p.rec), p.chunks, int(p.is_ended())) == (orclib.paf_tuple(rec), nu, en), r.id


def test_emulated_replay_matches_host_loop_and_windows(emu):
    """Partial last chunks: the replay gives the emulated host-stepped loop's lines in its order, and the same records
    with windows of one read each (every channel's reads spread over several calls) as with one window."""
    prefix, g, E, O = emu
    seqs = RL.seqs_of(O)
    reads = RL.synthetic_run(g, 3, 2, 5000, seed=13, int16=True)
    conf = _conf(num_channels=3, chunk_time=0.1125)
    one, calls1 = _emu_map_ord(E, seqs, conf, reads)
    many, calls2 = _emu_map_ord(E, seqs, conf, reads, window_samples=1)
    host = _emu_host(E, seqs, conf, reads)
    assert calls1 == 1 and calls2 == len(reads)
    assert [RL.paf_fields(p) for p in one] == [RL.paf_fields(p) for p in host]
    assert sorted(RL.paf_fields(p) for p in many) == sorted(RL.paf_fields(p) for p in one)
    assert {p.rd_name: (orclib.paf_tuple(p.rec), p.chunks) for p in many} == \
        {p.rd_name: (orclib.paf_tuple(p.rec), p.chunks) for p in one}


def test_emulated_golden_fast5s_match_the_host_loop(tmp_path):
    """The GPU test's fast5 case through the emulated device: multi_gzip, multi_latest and multi_many_reads given
    together (shared channels and start times) through `map-ord`, against the emulated host-stepped loop."""
    from uncalled_b200 import cli
    from uncalled_b200.fast5 import Fast5File
    prefix = orclib.materialise_example_index(str(tmp_path))
    E, O = RL.EmuReplay(prefix), orclib.Oracle(prefix)
    seqs = RL.seqs_of(O)
    paths = [os.path.join(F5, n) for n in ("multi_gzip.fast5", "multi_latest.fast5", "multi_many_reads.fast5")]
    _, conf, args = cli.load_conf(["map-ord", prefix] + paths)
    L = int(np.float32(conf.chunk_time) * np.float32(conf.sample_rate)) & 0xFFFF
    out = io.StringIO()
    cli.map_ord_cmd(conf, args, out=out, backend=RL.EmuReplayStream(E, conf.num_channels, L), index=RL.SeqIndex(seqs))
    reads = []
    for path in paths:
        with Fast5File(path) as f:
            for r in f.load():
                reads.append(RL.Read(r.read_id, r.channel, r.number, r.start_sample, r.signal, r.calibration))
    host = _emu_host(E, seqs, conf, reads)
    assert sorted(out.getvalue().splitlines()) == sorted(p.line() for p in host)
    assert len(host) == len(reads)


# ------------------------------------------------------------------------------------------------ command line
def test_cli_options_map_onto_conf():
    from uncalled_b200 import cli
    _, conf, args = cli.load_conf(["map-ord", "idx", "a.fast5", "b.fast5", "-r", "-l", "ids.txt", "-n", "9", "-p", "fast",
                                   "-e", "500", "-c", "7", "--chunk-time", "0.1125", "--num-channels", "128",
                                   "--exact-ties", "--device", "1", "--min-active-reads", "12", "-t", "2"])
    assert args.subcmd == "map-ord" and args.fast5s == ["a.fast5", "b.fast5"] and args.recursive
    assert (conf.bwa_prefix, conf.read_list, conf.max_reads, conf.idx_preset, conf.max_events, conf.max_chunks) == \
        ("idx", "ids.txt", 9, "fast", 500, 7)
    assert (conf.chunk_time, conf.num_channels, conf.exact_ties, conf.device, conf.min_active_reads, conf.threads) == \
        (0.1125, 128, 1, 1, 12, 2)
    _, c2, _ = cli.load_conf(["map-ord", "idx", "a.fast5"])
    assert c2.min_active_reads == 0 and c2.chunk_time == 1.0


def test_cli_missing_index_exits_1(tmp_path, capsys):
    from uncalled_b200 import cli
    with pytest.raises(SystemExit) as e:
        cli.main(["map-ord", str(tmp_path / "none"), os.path.join(F5, "multi_latest.fast5")])
    assert e.value.code == 1 and "does not exist" in capsys.readouterr().err


def test_cli_channel_above_num_channels_exits_1_before_the_gpu(tmp_path, capsys):
    """multi_latest puts reads up to channel 186: with --num-channels 100 the command stops while loading, before the
    index is loaded onto the device (on a machine without one the error would otherwise be a device error)."""
    from uncalled_b200 import cli
    prefix = orclib.materialise_example_index(str(tmp_path))
    with pytest.raises(SystemExit) as e:
        cli.main(["map-ord", prefix, os.path.join(F5, "multi_latest.fast5"), "--num-channels", "100"])
    err = capsys.readouterr().err
    assert e.value.code == 1 and "outside 1..100" in err, err


def test_replay_structs_match_the_c_abi():
    from uncalled_b200 import stream as S
    assert C.sizeof(S.ReplayRead) == 40 and C.sizeof(S.ReplayResult) == 24 + C.sizeof(S.StreamResult)


# ------------------------------------------------------------------------------------------------ register budget
REPLAY_SPILL_STORE_BUDGET = 400     # bytes per kernel; DESIGN.md section 4 records the counts


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_replay_kernels_keep_two_ctas_of_14_warps(tmp_path):
    """k2_map_replay and k2_map_replay_exact stay at the mapper's 72 registers (2 CTAs x 14 warps per SM); the replay's
    outer loop adds its spill stores to the streaming kernel's, within the budget."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import spill_report
    _, text = spill_report.compile_cubin(str(tmp_path))
    st = spill_report.ptxas_stats(text)
    for k in ("k2_map_replay", "k2_map_replay_exact"):
        assert st[k]["regs"] <= 72 and st[k]["regs"] * 14 * 32 * 2 <= 65536, (k, st[k])
        assert st[k]["spill_st"] <= REPLAY_SPILL_STORE_BUDGET, (k, st[k])
