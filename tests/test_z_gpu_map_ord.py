"""`map-ord` on the H100: the device replay (unc_stream_replay behind api.MapPoolOrd) against the oracle's channel mode,
against the host-stepped MapPoolOrd loop over unc_stream_step (replaylib.host_map_ord), against itself cut into small
windows, on the example read (SURVEY 8(c)) and on the golden fast5 fixtures."""
import multiprocessing
import os

import numpy as np
import pytest

import orclib
import replaylib as RL
import synthdata

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F5 = os.path.join(ROOT, "tests", "golden", "fast5")
N_CHANNELS = 64


def _conf(**kw):
    from uncalled_b200 import api
    c = api.Conf()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _chunk_len(ct):
    return int(np.float32(ct) * np.float32(4000.0)) & 0xFFFF


def _map_ord(conf, reads, window_samples=1 << 28):
    from uncalled_b200 import api
    pool = api.MapPoolOrd(conf, window_samples=window_samples)
    for r in reads:
        pool.queue_read(r.id, r.signal, r.channel, r.number, r.start, r.cal)
    out, calls = [], 0
    while pool.running():
        out += pool.update()
        calls += 1
    pool.stop()
    return out, calls


def _host_loop(conf, reads):
    from uncalled_b200 import api
    pool = api.RealtimePool(conf)
    L = pool.chunk_len
    res = RL.host_map_ord(pool, RL.order_channels(reads, conf.num_channels, conf.max_chunks * L), L)
    pool.stop_all()
    return [p for _, p in res]


def test_map_ord_prints_the_reference_line_for_the_example_read(tmp_path, capsys):
    """SURVEY 8(c): `uncalled_map_ord` on the example read prints ... 67 41 67 - ... 10000 6948 6977 29 30 255."""
    from uncalled_b200 import cli
    prefix = orclib.materialise_example_index(str(tmp_path))
    cli.main(["map-ord", prefix, os.path.join(F5, "example_single.fast5")])
    cap = capsys.readouterr()
    lines = [l.split("\t") for l in cap.out.splitlines()]
    assert len(lines) == 1, cap.out
    f = lines[0]
    assert f[1:5] == ["67", "41", "67", "-"] and f[6:12] == ["10000", "6948", "6977", "29", "30", "255"], f
    assert "Loading fast5s" in cap.err and "Mapping" in cap.err and "Finishing" in cap.err


@pytest.mark.parametrize("chunk_time", [0.1125, 1.0])
@pytest.mark.parametrize("tie_order", [0, 1])
def test_synthetic_run_matches_oracle_host_loop_and_small_windows(chunk_time, tie_order):
    """64 channels x 3 int16 reads of whole chunks: every record, chunks used and `ended` equal the oracle's channel mode
    (child_sort = tie order), and the Paf lines equal the host-stepped loop's and those of a run cut into many windows."""
    prefix, g = synthdata.get_index("g200k")
    L = _chunk_len(chunk_time)
    reads = RL.synthetic_run(g, N_CHANNELS, 3, 12000, seed=31 + tie_order, int16=True, whole_chunks=L)
    chans = RL.order_channels(reads, N_CHANNELS)
    jobs = [(prefix, [RL.pcal(r.signal, r.cal) for r in q], L, tie_order) for q in chans]
    ctx = multiprocessing.get_context("spawn")
    with ctx.Pool(min(os.cpu_count() or 1, 16)) as mp:
        pending = mp.map_async(orclib.stream_channel_job, jobs)
        conf = _conf(bwa_prefix=prefix, num_channels=N_CHANNELS, chunk_time=chunk_time, exact_ties=tie_order)
        dev, calls1 = _map_ord(conf, reads)
        small, calls2 = _map_ord(conf, reads, window_samples=60000)
        host = _host_loop(conf, reads)
        want = pending.get(timeout=1800)
    assert calls1 == 1 and calls2 > 3, (calls1, calls2)
    by_id = {p.rd_name: p for p in dev}
    assert len(by_id) == len(reads)
    n_mapped = 0
    for q, (owant, _, _) in zip(chans, want):
        for r, (paf, nu, en, _) in zip(q, owant):
            p = by_id[r.id]
            assert (orclib.paf_tuple(p.rec), p.chunks, int(p.is_ended())) == (tuple(paf), nu, en), (r.id, paf, nu, en)
            n_mapped += int(p.is_mapped())
    assert 0 < n_mapped < len(reads)
    assert [RL.paf_fields(p) for p in dev] == [RL.paf_fields(p) for p in host]
    assert sorted(RL.paf_fields(p) for p in small) == sorted(RL.paf_fields(p) for p in dev)


def test_partial_chunks_and_max_chunks_match_the_host_loop():
    """Reads ending inside a chunk, and max_chunks 7 (reads cut to 7 chunks, then the "no more signal" chunk): the device
    replay gives the host-stepped loop's lines, in its order."""
    prefix, g = synthdata.get_index("g200k")
    reads = RL.synthetic_run(g, N_CHANNELS, 3, 9000, seed=44, int16=True)
    for mc in (1000000, 7):
        conf = _conf(bwa_prefix=prefix, num_channels=N_CHANNELS, chunk_time=0.1125, max_chunks=mc)
        dev, _ = _map_ord(conf, reads)
        host = _host_loop(conf, reads)
        assert [RL.paf_fields(p) for p in dev] == [RL.paf_fields(p) for p in host], mc
        if mc == 7:
            assert any(p.chunks == 7 and p.is_ended() for p in dev)


def _fast5_lines(args, capsys):
    from uncalled_b200 import cli
    cli.main(args)
    return sorted(capsys.readouterr().out.splitlines())


def test_golden_fast5s_match_the_host_loop(tmp_path, capsys):
    """multi_gzip, multi_latest and multi_many_reads given together share channels and start times (read idx on channel
    1 + 37 idx mod 512 at 1000 + 4001 idx): map-ord gives the host-stepped path's lines, keyed by read id; the same for
    multi_deep_chunks, whose start times are above 2^32."""
    from uncalled_b200 import api
    from uncalled_b200.fast5 import Fast5File
    prefix = orclib.materialise_example_index(str(tmp_path))
    for names in (["multi_gzip.fast5", "multi_latest.fast5", "multi_many_reads.fast5"], ["multi_deep_chunks.fast5"]):
        paths = [os.path.join(F5, n) for n in names]
        got = _fast5_lines(["map-ord", prefix] + paths, capsys)
        reads = []
        for path in paths:
            with Fast5File(path) as f:
                for r in f.load():
                    reads.append(RL.Read(r.read_id, r.channel, r.number, r.start_sample, r.signal, r.calibration))
        conf = _conf(bwa_prefix=prefix)
        host = sorted(p.line() for p in _host_loop(conf, reads))
        assert got == host, names
        assert len(got) == sum(1 for r in reads if len(r.signal))


def test_map_ord_releases_what_it_holds(tmp_path):
    """unc_debug_held returns to its starting value once the pool's stream is freed."""
    import ctypes as C
    from uncalled_b200 import _native as N
    from uncalled_b200 import api

    def held():
        d, p, h = C.c_uint64(), C.c_uint64(), C.c_uint32()
        N.check(N.lib().unc_debug_held(C.byref(d), C.byref(p), C.byref(h)))
        return d.value, p.value, h.value

    prefix, g = synthdata.get_index("g200k")
    reads = RL.synthetic_run(g, 8, 2, 8000, seed=5, int16=True)
    conf = _conf(bwa_prefix=prefix, num_channels=8, chunk_time=0.1125)
    index = api.Index(prefix, device=0)
    before = held()
    pool = api.MapPoolOrd(conf, window_samples=20000)
    pool.index = index
    from uncalled_b200.stream import StreamMapper
    p = N.default_params()
    pool.backend = StreamMapper(index, 8, pool.chunk_len, params=p)
    for r in reads:
        pool.queue_read(r.id, r.signal, r.channel, r.number, r.start, r.cal)
    n = 0
    while pool.running():
        n += len(pool.update())
    pool.stop()
    assert n == len(reads)
    assert held() == before
