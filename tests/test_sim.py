"""The read-until simulator (uncalled_b200/sim.py, `python -m uncalled_b200 sim`) without a GPU:
  * load_sim against the call sequence of the reference's own sim_utils.load_sim (tests/golden/sim/load_sim_golden.json);
  * ClientSim against the reference's own src/client_sim.cpp on a scripted scenario with a controlled clock
    (tests/golden/sim/client_golden.json);
  * run_sim end to end on the emulated device code with a fake clock;
  * bad input, the CLI parser and the Conf defaults.
The goldens under tests/golden/sim/ come from tools/make_sim_golden.py."""
import io
import json
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "golden", "sim")
CAL = (1400.0, 0.0, 8192.0)          # (range, offset, digitisation) of the synthetic int16 reads
TIMING_TAGS = ("mt", "ej", "kp", "en")


def _conf(**kw):
    from uncalled_b200.api import Conf
    c = Conf()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


class FakeClock:
    """Milliseconds that advance by `step` on every reading."""

    def __init__(self, step=5.0):
        self.t, self.step = 0.0, step

    def __call__(self):
        self.t += self.step
        return self.t


# ---------------------------------------------------------------------------------------------------------------------
# 1. load_sim: the reference's call sequence

class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("add_"):
            raise AttributeError(name)
        return lambda *a: self.calls.append([name] + [x if isinstance(x, str) else int(x) for x in a])


@pytest.mark.parametrize("case", ["defaults", "short_intervals"])
def test_load_sim_makes_the_reference_calls(case):
    from uncalled_b200 import sim
    gold = json.load(open(os.path.join(SIM, "load_sim_golden.json")))[case]
    conf = _conf(unc_seqsum=os.path.join(SIM, "unc_seqsum.txt"), unc_paf=os.path.join(SIM, "unc.paf"),
                 ctl_seqsum=os.path.join(SIM, "ctl_seqsum.txt"), **gold["conf"])
    rec = _Recorder()
    sim.load_sim(rec, conf, log=io.StringIO())
    assert rec.calls == gold["calls"]


def test_find_scans_finds_both_scans_of_the_fixture():
    from uncalled_b200 import sim
    p = sim.SeqsumProfile(os.path.join(SIM, "unc_seqsum.txt"))
    scans = sim.find_scans(p.sts, p.ens, p.mxs)
    assert len(scans) == 2 and scans[0][0] == 0
    bounds = p.rm_scans()
    assert len(bounds) == 3 and not np.any(p.ids == "")


# ---------------------------------------------------------------------------------------------------------------------
# 2. ClientSim: the reference's state machine, chunk for chunk

def replay_client_script(script, log=None):
    """Runs the script of tools/make_sim_golden.py through sim.ClientSim; output lines as the reference driver's."""
    from uncalled_b200 import sim
    clock = {"ms": 0.0}
    out, client = [], None
    for line in script:
        a = line.split()
        if a[0] == "conf":
            conf = _conf(num_channels=int(a[1]), sample_rate=float(a[2]), chunk_time=float(a[3]), max_chunks=int(a[4]),
                         scan_time=float(a[5]), ej_time=float(a[6]))
            client = sim.ClientSim(conf, clock=lambda: clock["ms"], log=log or io.StringIO())
        elif a[0] == "intv":
            client.add_intv(*map(int, a[1:]))
        elif a[0] == "gap":
            client.add_gap(*map(int, a[1:]))
        elif a[0] == "delay":
            client.add_delay(*map(int, a[1:]))
        elif a[0] == "read":
            client.add_read(int(a[1]), a[2], int(a[3]))
        elif a[0] == "load":
            n = int(a[3])
            client.load_read(a[1], int(a[2]), np.arange(n, dtype=np.int16), CAL)
        elif a[0] == "run":
            client.run()
        elif a[0] == "tick":
            clock["ms"] = float(a[1])
            for ch, c in client.get_read_chunks():
                first = int(c._raw[0]) if c.size() else -1
                out.append("chunk %s %d %d %s %d %d %d" % (a[1], ch, c.number, c.id, c.start, c.size(), first))
            out.append("running %s %d" % (a[1], 1 if client.is_running else 0))
        elif a[0] == "stop":
            client.stop_receiving_read(int(a[1]), int(a[2]))
        elif a[0] == "unblock":
            out.append("unblock %s %s %d" % (a[1], a[2], client.unblock_read(int(a[1]), int(a[2]))))
    return out


def test_client_sim_matches_the_reference_chunk_for_chunk():
    gold = json.load(open(os.path.join(SIM, "client_golden.json")))
    log = io.StringIO()
    got = replay_client_script(gold["script"], log)
    assert got == gold["out"]
    kinds = {l.split()[0] for l in got}
    assert kinds == {"chunk", "running", "unblock"}
    assert "starting mux scan" in log.getvalue() and "ending mux scan" in log.getvalue()
    assert any(l.startswith("unblock") and not l.endswith(" 0") for l in got)        # a delay was taken
    assert got[-1].endswith(" 0")                                                       # every interval ran out


def test_client_sim_keeps_only_the_int16_samples_of_its_chunks():
    from uncalled_b200 import sim
    conf = _conf(num_channels=2, chunk_time=0.25, max_chunks=3)
    c = sim.ClientSim(conf, clock=lambda: 0.0)
    c.add_intv(1, 0, 0, 100000)
    c.add_gap(1, 0, 10)
    c.add_read(1, "a", 300)
    c.add_read(1, "b", 0)
    c.add_read(1, "gone", 0)
    sig = (np.arange(10000) % 3000).astype(np.int16)
    assert c.load_read("a", 5, sig, CAL) and c.load_read("b", 6, sig[:2500], CAL)
    assert not c.load_read("not-in-the-pattern", 7, sig, CAL)
    a, b, gone = c.channels[0].reads
    assert a.duration == 3000                              # the signal is cut to max_chunks chunks, as ReadBuffer does
    assert a.n_chunks == 2 and a.sig.dtype == np.int16 and a.sig.nbytes == 2 * 1000 * 2 and a.sig[0] == 300
    assert b.n_chunks == 2 and b.duration == 2500 and a.cal == CAL
    assert gone.duration == 0 and gone.n_chunks == 0 and gone.sig is None


# ---------------------------------------------------------------------------------------------------------------------
# 3. run_sim end to end on the emulated device

def write_run_fixture(d, read_ids, n_channels, seq_time=6.0, read_time=2.0, seed=3):
    """A control and an UNCALLED sequencing summary (one mux scan, then `seq_time` s of reads on every channel), and an
    UNCALLED PAF ejecting every third read.  The control summary holds `read_ids`, spread over the channels; their
    template starts with the read, so every sample reaches the mapper."""
    rng = np.random.default_rng(seed)
    head = "read_id\tchannel\tmux\tstart_time\tduration\ttemplate_start\ttemplate_duration\tsequence_length_template\n"
    paths = {k: os.path.join(d, k) for k in ("unc_seqsum.txt", "ctl_seqsum.txt", "unc.paf")}

    def scan_rows(prefix):
        rows = []
        for mux in (1, 2, 3, 4):
            for ch in range(1, n_channels + 1):
                rows.append(("%s_scan%d_%d" % (prefix, mux, ch), ch, mux, 4.0 * (mux - 1), 2.5))
        return rows

    unc = scan_rows("u")
    for ch in range(1, n_channels + 1):
        t, k = 16.0 + 0.3 * ch, 0
        while t < 16.0 + seq_time:
            unc.append(("u_%d_%d" % (ch, k), ch, 1 + ch % 4, t, read_time))
            t += read_time + rng.uniform(0.2, 0.6)
            k += 1
    ctl = scan_rows("c")
    for i, rid in enumerate(read_ids):
        ch = 1 + i % n_channels
        ctl.append((rid, ch, 1 + ch % 4, 16.0 + 3.0 * (i // n_channels) + 0.1 * ch, read_time))
    for name, rows in (("unc_seqsum.txt", unc), ("ctl_seqsum.txt", ctl)):
        with open(paths[name], "w") as f:
            f.write(head)
            for rid, ch, mux, st, ln in rows:
                f.write("%s\t%d\t%d\t%.4f\t%.4f\t%.4f\t%.4f\t%d\n" % (rid, ch, mux, st, ln, st, ln, 900))
    with open(paths["unc.paf"], "w") as f:
        for k, (rid, ch, *_r) in enumerate(unc):
            tag = "ej:f:0.150000" if k % 3 == 0 else "kp:f:0.100000"
            f.write("%s\t%d\t*\t*\t*\t*\t*\t*\t*\t*\t*\t255\tch:i:%d\t%s\n" % (rid, 400, ch, tag))
    return paths


def synthetic_reads(n_reads=8, seed=11):
    """Half drawn from the g200k test genome, half random sequence; int16 DAC values with calibration CAL."""
    import synth
    import synthdata
    prefix, g = synthdata.get_index("g200k")
    sig, truth = synth.reads(g, n_reads, 4000, seed=seed, frac_random=0.0)
    rnd, _ = synth.reads(g, n_reads, 4000, seed=seed + 1, frac_random=1.0)
    on = np.arange(n_reads) % 2 == 0
    sig = np.where(on[:, None], sig, rnd)
    dac = np.round(sig * CAL[2] / CAL[0] - CAL[1]).astype(np.int16)
    ids = ["%s%d" % ("on" if on[i] else "off", i) for i in range(n_reads)]
    return prefix, [(ids[i], 100 + i, dac[i], CAL) for i in range(n_reads)], on


def scenario_run(tmp, mode, active=0, n_channels=8, gpu=False):
    """run_sim with the fake clock on the emulated device code (or, with gpu=True, on the GPU stream kernels);
    returns the output text."""
    from uncalled_b200 import sim
    prefix, reads, _ = synthetic_reads()
    paths = write_run_fixture(str(tmp), [r[0] for r in reads], n_channels)
    # One read per channel.  A read ends before ClientSim hands out its last full chunk, so a pass delivers 3 chunks;
    # when the read comes round again with the same number, its chunks go on to the same mapper, which gives up
    # on an unmapped read at max_chunks (the eject decision) -- as the reference's RealtimePool does.
    conf = _conf(num_channels=n_channels, chunk_time=0.25, max_chunks=4, min_ch_reads=1, realtime_mode=mode,
                 active_chs=active, unc_seqsum=paths["unc_seqsum.txt"], ctl_seqsum=paths["ctl_seqsum.txt"],
                 unc_paf=paths["unc.paf"], bwa_prefix=prefix)
    backend = index = None
    if not gpu:
        import emulib
        import orclib
        E, O = emulib.Emu(prefix), orclib.Oracle(prefix)
        backend = emulib.EmuStream(E, n_channels, 1000, max_chunks=conf.max_chunks)

        class index:
            seqs = [(O.lib.orc_seq_name(O.idx, i).decode(), int(O.lib.orc_seq_len(O.idx, i))) for i in range(O.lib.orc_n_seqs(O.idx))]
    out = io.StringIO()
    sim.run_sim(conf, [], out, clock=FakeClock(), log=io.StringIO(), backend=backend, index=index, reads=reads)
    return out.getvalue()


def paf_records(text):
    """{read id: [tag names]} of the PAF lines; comment lines are skipped."""
    recs = {}
    for l in text.splitlines():
        if l.startswith("#"):
            continue
        t = l.split("\t")
        recs.setdefault(t[0], []).append([x.split(":")[0] for x in t[12:]])
    return recs


def strip_timing(text):
    """PAF lines without the values of the time-valued tags (the tag names stay)."""
    out = []
    for l in text.splitlines():
        if l.startswith("#"):
            out.append(l)
            continue
        t = l.split("\t")
        out.append("\t".join(t[:12] + [x.split(":")[0] if x.split(":")[0] in TIMING_TAGS else x for x in t[12:]]))
    return out


_RUNS = {}


def _run(tmp_path_factory, mode, active=0):
    if (mode, active) not in _RUNS:
        _RUNS[(mode, active)] = scenario_run(tmp_path_factory.mktemp("sim"), mode, active)
    return _RUNS[(mode, active)]


def write_run_golden(path):
    import tempfile
    from uncalled_b200.api import RealtimePool
    with tempfile.TemporaryDirectory() as d:
        text = scenario_run(d, RealtimePool.ENRICH)
    json.dump({"mode": "enrich", "lines": strip_timing(text)}, open(path, "w"), indent=0)


def test_run_sim_enrich_ejects_off_target_reads(tmp_path_factory):
    from uncalled_b200.api import RealtimePool
    recs = paf_records(_run(tmp_path_factory, RealtimePool.ENRICH))
    assert any(r.startswith("on") for r in recs) and any(r.startswith("off") for r in recs)
    for rid, lines in recs.items():
        for tags in lines:
            assert sum(t in ("ej", "kp", "en") for t in tags) == 1, (rid, tags)
            assert ("ej" in tags) == ("dl" in tags)
            if rid.startswith("off"):
                assert "kp" not in tags, (rid, tags)
            else:
                assert "ej" not in tags, (rid, tags)
    assert any("ej" in t for r, ls in recs.items() for t in ls if r.startswith("off"))
    assert any("kp" in t for r, ls in recs.items() for t in ls if r.startswith("on"))


def test_run_sim_deplete_is_the_reverse(tmp_path_factory):
    from uncalled_b200.api import RealtimePool
    recs = paf_records(_run(tmp_path_factory, RealtimePool.DEPLETE))
    for rid, lines in recs.items():
        for tags in lines:
            if rid.startswith("on"):
                assert "kp" not in tags, (rid, tags)
            else:
                assert "ej" not in tags, (rid, tags)
    assert any("ej" in t for r, ls in recs.items() for t in ls if r.startswith("on"))


@pytest.mark.parametrize("active,parity", [(1, 0), (2, 1)])
def test_run_sim_even_and_odd_leave_the_other_channels_unprinted(tmp_path_factory, active, parity):
    from uncalled_b200.api import RealtimePool
    text = _run(tmp_path_factory, RealtimePool.ENRICH, active)
    chans = [int(x[5:]) for l in text.splitlines() if not l.startswith("#") for x in l.split("\t") if x.startswith("ch:i:")]
    assert chans and all(c % 2 == parity for c in chans)


def test_run_sim_is_deterministic_and_matches_the_golden(tmp_path_factory, tmp_path):
    from uncalled_b200.api import RealtimePool
    first = _run(tmp_path_factory, RealtimePool.ENRICH)
    assert scenario_run(tmp_path, RealtimePool.ENRICH) == first
    gold = json.load(open(os.path.join(SIM, "run_golden.json")))
    assert strip_timing(first) == gold["lines"]


# ---------------------------------------------------------------------------------------------------------------------
# 4. bad input, parser, defaults

def _sim_argv(tmp, **over):
    a = {"--ctl-seqsum": os.path.join(SIM, "ctl_seqsum.txt"), "--unc-seqsum": os.path.join(SIM, "unc_seqsum.txt"),
         "--unc-paf": os.path.join(SIM, "unc.paf")}
    a.update(over)
    prefix = str(tmp / "idx")
    for ext in (".bwt", ".uncl"):
        open(prefix + ext, "w").close()
    argv = ["sim", prefix, os.path.join(ROOT, "tests", "golden", "fast5", "multi_gzip.fast5"), "-E"]
    for k, v in a.items():
        argv += [k, v]
    return argv


@pytest.mark.parametrize("which", ["--ctl-seqsum", "--unc-seqsum", "--unc-paf"])
def test_missing_input_is_reported_before_any_device_call(tmp_path, capsys, monkeypatch, which):
    from uncalled_b200 import cli
    import uncalled_b200._native as N
    monkeypatch.setattr(N, "lib", lambda: pytest.fail("a device call was made"))
    gone = str(tmp_path / "gone.txt")
    with pytest.raises(SystemExit) as e:
        cli.main(_sim_argv(tmp_path, **{which: gone}))
    assert e.value.code == 1 and gone in capsys.readouterr().err


@pytest.mark.parametrize("column", ["channel", "start_time", "duration", "mux", "read_id", "template_start",
                                    "template_duration", "sequence_length_template"])
def test_missing_summary_column_is_named(tmp_path, capsys, monkeypatch, column):
    from uncalled_b200 import cli
    import uncalled_b200._native as N
    monkeypatch.setattr(N, "lib", lambda: pytest.fail("a device call was made"))
    lines = open(os.path.join(SIM, "ctl_seqsum.txt")).read().splitlines()
    head = lines[0].split("\t")
    k = head.index(column)
    bad = tmp_path / "ctl.txt"
    bad.write_text("\n".join("\t".join(x for i, x in enumerate(l.split("\t")) if i != k) for l in lines) + "\n")
    with pytest.raises(SystemExit) as e:
        cli.main(_sim_argv(tmp_path, **{"--ctl-seqsum": str(bad)}))
    err = capsys.readouterr().err
    assert e.value.code == 1 and str(bad) in err and '"%s"' % column in err


def test_sim_parser_options(tmp_path, capsys):
    from uncalled_b200 import cli
    from uncalled_b200.api import RealtimePool
    _, conf, args = cli.load_conf(["sim", "idx/ecoli", "a.fast5", "b.fast5", "-D", "--even", "--ctl-seqsum", "c.txt",
                                   "--unc-seqsum", "u.txt", "--unc-paf", "u.paf", "--sim-speed", "2.5", "-t", "3",
                                   "-c", "7", "-e", "900", "--chunk-time", "0.5", "--num-channels", "128", "-p", "fast",
                                   "-r", "--device", "1"])
    assert (conf.bwa_prefix, conf.idx_preset, conf.ctl_seqsum, conf.unc_seqsum, conf.unc_paf, conf.sim_speed) == \
        ("idx/ecoli", "fast", "c.txt", "u.txt", "u.paf", 2.5)
    assert (conf.threads, conf.max_chunks, conf.max_events, conf.chunk_time, conf.num_channels, conf.device) == \
        (3, 7, 900, 0.5, 128, 1)
    assert (conf.realtime_mode, conf.active_chs, args.fast5s, args.recursive) == \
        (RealtimePool.DEPLETE, RealtimePool.EVEN, ["a.fast5", "b.fast5"], True)
    _, conf, _ = cli.load_conf(["sim", "x", "a.fast5", "-E", "--odd", "--ctl-seqsum", "c", "--unc-seqsum", "u",
                                "--unc-paf", "p"])
    assert (conf.realtime_mode, conf.active_chs, conf.sim_speed) == (RealtimePool.ENRICH, RealtimePool.ODD, 1.0)
    base = ["sim", "x", "a.fast5", "--ctl-seqsum", "c", "--unc-seqsum", "u", "--unc-paf", "p"]
    for extra in ([], ["-D", "-E"], ["-E", "--even", "--odd"]):
        with pytest.raises(SystemExit) as e:
            cli.load_conf(base + extra)
        assert e.value.code == 2
    with pytest.raises(SystemExit):
        cli.load_conf(["sim", "x", "a.fast5", "-E", "--ctl-seqsum", "c", "--unc-seqsum", "u"])   # --unc-paf is required
    capsys.readouterr()


def test_sim_without_a_gpu_fails_with_no_device(tmp_path, capsys):
    import uncalled_b200._native as N
    from uncalled_b200 import cli
    if N.lib().unc_device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(N.UncError, match="NO_DEVICE|no CUDA device"):
        cli.main(_sim_argv(tmp_path))


def test_conf_simulator_defaults():
    """The [simulator] section of the reference's uncalled/conf/defaults.toml."""
    c = _conf()
    assert (c.ctl_seqsum, c.unc_seqsum, c.unc_paf) == ("", "", "")
    assert (c.sim_speed, c.min_ch_reads, c.scan_time, c.scan_intv_time, c.ej_time) == (1.0, 10, 10.0, 5400.0, 0.1)
    for name in ("ctl_seqsum", "unc_seqsum", "unc_paf", "sim_speed", "scan_time", "scan_intv_time", "ej_time", "min_ch_reads"):
        assert type(c).__dict__[name].__doc__


def test_chunks_carry_int16_with_calibration():
    from uncalled_b200.api import Chunk
    c = Chunk("r", 2, 5, 100, np.arange(10, dtype=np.int16), 2, 4, calibration=CAL)
    assert (c.dtype, c.cal, c.size()) == (1, CAL, 4)
    assert c.pop().dtype == np.int16 and c.empty()
    with pytest.raises(TypeError):
        Chunk("r", 2, 5, 100, np.arange(10, dtype=np.float32), calibration=CAL)
    assert Chunk("r", 1, 1, 0, [1.5, 2.5]).dtype == 0
