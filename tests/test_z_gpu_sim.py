"""The read-until simulator on the GPU: the emulated end-to-end scenario of tests/test_sim.py through the sm_90a stream
kernels with the same fake clock, and `python -m uncalled_b200 sim` on the wall clock."""
import json
import os
import subprocess
import sys

import pytest

import test_sim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F5 = os.path.join(ROOT, "tests", "golden", "fast5")


@pytest.mark.gpu
def test_gpu_run_matches_the_emulator_golden(tmp_path):
    from uncalled_b200.api import RealtimePool
    text = test_sim.scenario_run(tmp_path, RealtimePool.ENRICH, gpu=True)
    gold = json.load(open(os.path.join(test_sim.SIM, "run_golden.json")))
    assert test_sim.strip_timing(text) == gold["lines"]


@pytest.mark.gpu
def test_gpu_sim_cli_on_the_wall_clock(tmp_path):
    import orclib
    from uncalled_b200.fast5 import Fast5File
    prefix = orclib.materialise_example_index(str(tmp_path))
    files = [os.path.join(F5, f) for f in ("multi_gzip.fast5", "multi_latest.fast5", "multi_contig.fast5")]
    ids = []
    for f in files:
        with Fast5File(f) as h:
            ids += [h.info(i).read_id for i in range(h.n_reads)]
    # two channels, so that the 23 control reads cover the default 10 reads per active channel
    paths = test_sim.write_run_fixture(str(tmp_path), ids, 2, seq_time=10.0)
    cmd = [sys.executable, "-m", "uncalled_b200", "sim", prefix] + files + [
        "-E", "--num-channels", "4", "--chunk-time", "0.25", "--ctl-seqsum", paths["ctl_seqsum.txt"],
        "--unc-seqsum", paths["unc_seqsum.txt"], "--unc-paf", paths["unc.paf"]]
    env = dict(os.environ, PYTHONPATH=ROOT)
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env, cwd=str(tmp_path))
    assert res.returncode == 0, res.stderr[-3000:]
    lines = [l for l in res.stdout.splitlines() if not l.startswith("#")]
    assert lines, res.stderr[-3000:]
    for l in lines:
        t = l.split("\t")
        assert t[0] in ids
        tags = [x.split(":")[0] for x in t[12:]]
        assert sum(k in ("kp", "ej", "en") for k in tags) == 1, l
        assert ("ej" not in tags) or ("dl" in tags), l
