"""The device FM-index builder (unc_index_build_device) writes the same five files, byte for byte, as the host builder
(unc_index_build) and bwa.

CPU tier: the device source under the warp emulator (tests/emul/emul_index_build.cpp, driven by the library's own launch
sequence) against the host builder on seeded inputs with long repeats, palindromes, IUPAC runs and tiny lengths, also
with the sort workspace forced small so the doubling rounds run in many batches; the size limit and the device check
come before anything is written; the bindings keep the host builder without a device.

GPU tier: the same inputs and seeded genomes of 1 Mb and 60 Mb (above bwa's `bwtsw` switch) against the host builder,
`uncalled index` end to end, and a 1.1 Gbp genome (2.2e9 FM rows, above 2^31) against the digests of bwa's own files,
loaded and searched and mapped against."""
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import indexlib as I

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

UNC_E_IO, UNC_E_NO_DEVICE, UNC_E_TOO_LARGE = -2, -4, -5
LIMIT_BASES = 0xFFFFFF00 // 2          # seq_len = 2 x bases must stay below 0xFFFFFF00


def _lib():
    from uncalled_b200 import _native as N
    return N.lib()


def _host(fa, prefix):
    assert _lib().unc_index_build(fa.encode(), prefix.encode()) == 0
    return I.read_files(prefix)


def _fixture_fa(tmp_path, name):
    fa = str(tmp_path / (name + ".fa"))
    with open(fa, "wb") as f:
        f.write(I.fixture(name))
    return fa


def _no_device():
    return _lib().unc_device_count() == 0


# ---------------------------------------------------------------- CPU tier: the device source under the emulator

def test_example_emul(tmp_path):
    fasta, files = I.example()
    fa = str(tmp_path / "example.fa")
    open(fa, "wb").write(fasta)
    rc, _ = I.emu_index_build(fa, str(tmp_path / "emu"))
    assert rc == 0
    assert I.read_files(str(tmp_path / "emu")) == files


@pytest.mark.parametrize("name", sorted(I.FIXTURES))
def test_fixture_emul(tmp_path, name):
    fa = _fixture_fa(tmp_path, name)
    want = _host(fa, str(tmp_path / "host"))
    rc, info = I.emu_index_build(fa, str(tmp_path / "emu"))
    assert rc == 0
    got = I.read_files(str(tmp_path / "emu"))
    for e in I.EXTS:
        assert got[e] == want[e], e
    if name in ("polya", "block_repeats", "palindrome", "tandem"):      # long repeats force many rounds
        assert len(info["active"]) >= 8, info
    assert info["peak_bytes"] <= info["model_bytes"], info              # the memory check bounds the allocations


# (fixture, workspace rows): small enough that the first rounds take several batches
SMALL_WS = [("multi_iupac", 2000), ("tandem", 1000), ("polya", 1000), ("palindrome", 4000), ("synth1", 600),
            ("len129", 16), ("tiny_ACAC", 8)]


@pytest.mark.parametrize("name,ws", SMALL_WS, ids=["%s-%d" % c for c in SMALL_WS])
def test_small_workspace_emul(tmp_path, name, ws):
    fa = _fixture_fa(tmp_path, name)
    want = _host(fa, str(tmp_path / "host"))
    rc, info = I.emu_index_build(fa, str(tmp_path / "emu"), ws)
    assert rc == 0
    assert I.read_files(str(tmp_path / "emu")) == want
    if name not in ("len129", "tiny_ACAC"):
        assert max(info["batches"]) > 1, info       # the workspace did split a round


def _sparse_fasta(path, bases):
    """a header, then `bases` zero bytes (each an ambiguous base), without writing them"""
    with open(path, "wb") as f:
        f.write(b">big\n")
        f.truncate(5 + bases)


def _files_of(prefix):
    return [e for e in I.EXTS if os.path.exists(prefix + "." + e)]


def test_too_large_writes_nothing(tmp_path):
    fa = str(tmp_path / "big.fa")
    _sparse_fasta(fa, LIMIT_BASES)
    prefix = str(tmp_path / "out")
    assert _lib().unc_index_build_device(fa.encode(), prefix.encode()) == UNC_E_TOO_LARGE
    assert I.emu_index_build(fa, prefix)[0] == UNC_E_TOO_LARGE
    assert _files_of(prefix) == []


@pytest.mark.skipif(not _no_device(), reason="a CUDA device is visible")
def test_no_device_writes_nothing(tmp_path):
    fa = _fixture_fa(tmp_path, "synth1")
    prefix = str(tmp_path / "out")
    assert _lib().unc_index_build_device(fa.encode(), prefix.encode()) == UNC_E_NO_DEVICE
    assert _files_of(prefix) == []
    # one base below the limit passes the size check and stops at the device check, still before any file
    _sparse_fasta(fa, LIMIT_BASES - 1)
    assert _lib().unc_index_build_device(fa.encode(), prefix.encode()) == UNC_E_NO_DEVICE
    assert _files_of(prefix) == []


def test_empty_or_missing_input(tmp_path):
    fa = str(tmp_path / "e.fa")
    open(fa, "wb").write(b">empty\n\n")
    prefix = str(tmp_path / "out")
    assert _lib().unc_index_build_device(fa.encode(), prefix.encode()) == UNC_E_IO
    assert _lib().unc_index_build_device(str(tmp_path / "missing.fa").encode(), prefix.encode()) == UNC_E_IO
    assert _files_of(prefix) == []


@pytest.mark.skipif(not _no_device(), reason="a CUDA device is visible")
def test_bindings_use_the_host_builder_without_a_device(tmp_path):
    """unc_index_build_device would fail here (no device): the files appear, so both bindings took the host builder"""
    fa = _fixture_fa(tmp_path, "synth2")
    want = _host(fa, str(tmp_path / "host"))
    from uncalled_b200.index import BwaIndex
    BwaIndex.create(fa, str(tmp_path / "py"))
    assert I.read_files(str(tmp_path / "py")) == want
    import uncalled_b200._native as N
    N.build_pymodule()
    code = ("import sys; sys.path[:0] = [%r]; import _uncalled; _uncalled.BwaIndex.create(%r, %r)"
            % (os.path.join(ROOT, "uncalled_b200"), fa, str(tmp_path / "ext")))
    subprocess.run([sys.executable, "-c", code], check=True)
    assert I.read_files(str(tmp_path / "ext")) == want


# ---------------------------------------------------------------- GPU tier

def _device(fa, prefix):
    L = _lib()
    assert L.unc_init(0) == 0
    rc = L.unc_index_build_device(fa.encode(), prefix.encode())
    assert rc == 0, L.unc_last_error().decode()
    return I.read_files(prefix)


def _last_times():
    import ctypes as C
    ms, rounds, peak = (C.c_float * 3)(), C.c_uint32(), C.c_uint64()
    _lib().unc_index_build_device_last_times(ms, C.byref(rounds), C.byref(peak))
    return list(ms), rounds.value, peak.value


@pytest.mark.gpu
def test_gpu_example(tmp_path):
    fasta, files = I.example()
    fa = str(tmp_path / "example.fa")
    open(fa, "wb").write(fasta)
    assert _device(fa, str(tmp_path / "dev")) == files


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(I.FIXTURES))
def test_gpu_fixture(tmp_path, name):
    fa = _fixture_fa(tmp_path, name)
    want = _host(fa, str(tmp_path / "host"))
    got = _device(fa, str(tmp_path / "dev"))
    for e in I.EXTS:
        assert got[e] == want[e], e
    ms, rounds, peak = _last_times()
    assert all(t >= 0 for t in ms) and peak > 0


@pytest.mark.gpu
@pytest.mark.parametrize("mb", [1, 60])
def test_gpu_seeded_genome(tmp_path, mb):
    import masklib
    fa = str(tmp_path / "g.fa")
    open(fa, "wb").write(masklib.big_genome(mb * 1000000, seed=40 + mb, n_records=3))
    want = _host(fa, str(tmp_path / "host"))
    got = _device(fa, str(tmp_path / "dev"))
    for e in I.EXTS:
        assert got[e] == want[e], e
    ms, rounds, peak = _last_times()
    assert rounds >= 5, rounds                  # the planted 6 kb elements need rounds up to h > 3000


@pytest.mark.gpu
def test_gpu_uncalled_index(tmp_path):
    """`uncalled index` end to end on the device builder: the example reference's files and .uncl as shipped"""
    from uncalled_b200 import cli
    fasta, files = I.example()
    z = np.load(os.path.join(ROOT, "tests", "golden", "example_index_files.npz"))
    fa = str(tmp_path / "example_ref.fa")
    open(fa, "wb").write(fasta)
    assert cli.main(["index", fa, "-o", str(tmp_path / "example_ref")]) == 0
    assert I.read_files(str(tmp_path / "example_ref")) == files
    assert open(str(tmp_path / "example_ref.uncl"), "rb").read() == z["uncl"].tobytes()


def _sha256_file(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 24), b""):
            h.update(blk)
    return h.hexdigest()


def _pac_codes(prefix, l_pac):
    """the forward codes from the .pac file (ambiguous bases as replaced), one per byte"""
    pac = np.fromfile(prefix + ".pac", np.uint8)[:(l_pac + 3) // 4]
    codes = np.empty(pac.size * 4, np.uint8)
    for k in range(4):
        codes[k::4] = (pac >> (6 - 2 * k)) & 3
    return codes[:l_pac]


@pytest.mark.gpu
def test_gpu_above_2_31_rows_against_bwa(tmp_path):
    """1.1 Gbp: the five files against the digests of bwa's own (tools/make_index_device_golden.py); then the index
    loads (k_sa_expand / k_occ2_build above 2^31 rows), its SA orders suffixes, its ranges count occurrences, and
    seeded reads map to where they were drawn from"""
    gold = json.load(open(I.BIG_GOLDEN))
    work = tempfile.mkdtemp(dir=str(tmp_path))
    try:
        fa, prefix = os.path.join(work, "big.fa"), os.path.join(work, "big")
        data = I.big_fasta()
        assert hashlib.sha256(data).hexdigest() == gold["fasta_sha256"]
        with open(fa, "wb") as f:
            f.write(data)
        del data
        L = _lib()
        assert L.unc_init(0) == 0
        rc = L.unc_index_build_device(fa.encode(), prefix.encode())
        assert rc == 0, L.unc_last_error().decode()
        os.remove(fa)
        for e in I.EXTS:
            assert _sha256_file(prefix + "." + e) == gold["files"][e], e
        ms, rounds, peak = _last_times()
        print("1.1 Gbp device build: phases ms", ms, "rounds", rounds, "peak bytes", peak)

        uncl = json.load(open(os.path.join(ROOT, "tests", "golden", "synth_uncl.json")))["g20m"]["uncl"]
        open(prefix + ".uncl", "w").write(uncl)
        import uncalled_b200 as U
        idx = U.Index(prefix, device=0)
        l_pac = int(open(prefix + ".ann").readline().split()[0])
        n = 2 * l_pac
        assert idx.n_rows == n and n + 1 > 2 ** 31
        fwd = _pac_codes(prefix, l_pac)
        rng = np.random.default_rng(5)

        # suffix order of consecutive rows, read from the text (forward codes, then their reverse complement)
        def sym(pos):                          # text symbols at positions pos (array), 4 past the end
            pos = np.asarray(pos, np.int64)
            out = np.full(pos.shape, 4, np.int64)
            f = pos < l_pac
            out[f] = fwd[pos[f]]
            r = (pos >= l_pac) & (pos < n)
            out[r] = 3 - fwd[n - 1 - pos[r]].astype(np.int64)
            return out
        rows = rng.integers(1, n - 1, 3000).astype(np.uint64)
        a, b = idx.sa(rows).astype(np.int64), idx.sa(rows + 1).astype(np.int64)
        assert (a < n).all() and (b < n).all() and (a != b).all()
        todo, step = np.arange(len(rows)), np.arange(64)
        for d in range(0, 1 << 17, 64):          # 64 symbols at a time, the pairs not decided yet
            x, y = sym(a[todo, None] + d + step), sym(b[todo, None] + d + step)
            diff = x != y
            first = diff.argmax(axis=1)
            dec = diff.any(axis=1)
            k = np.arange(len(todo))[dec]
            assert (x[k, first[dec]] < y[k, first[dec]]).all(), d
            todo = todo[~dec]
            if not len(todo):
                break
        assert not len(todo)

        # backward-search range sizes against occurrence counts in the text
        text = fwd.tobytes() + (3 - fwd[::-1]).tobytes()
        del fwd
        L2 = np.concatenate([[0], np.frombuffer(open(prefix + ".bwt", "rb").read(40)[8:], np.uint64)]).astype(np.uint64)
        for q in range(12):
            k = 20 if q < 8 else 12
            p = int(rng.integers(0, n - k))
            sub = text[p:p + k]
            cnt, j = 0, text.find(sub)
            while j != -1:
                cnt += 1
                j = text.find(sub, j + 1)
            st = np.array([L2[sub[-1]] + 1], np.uint64)
            en = np.array([L2[sub[-1] + 1]], np.uint64)
            for c in sub[-2::-1]:
                st, en = idx.neighbors(st, en, np.array([c], np.uint8))
            assert int(en[0]) - int(st[0]) + 1 == cnt, (q, p, cnt)
        del text

        # seeded reads from known forward positions map there
        import synth
        fwd = _pac_codes(prefix, l_pac)
        ann = open(prefix + ".ann").read().split("\n")[1:]
        offs = [int(ann[2 * r + 1].split()[0]) for r in range(len(ann) // 2)]
        n_reads, n_samples = 300, 6000
        sig, truth = synth.reads(fwd, n_reads, n_samples, seed=11, frac_random=0.0)
        bm = U.BatchMapper(idx, max_reads=n_reads, max_samples=n_reads * n_samples)
        out = bm.map(sig.reshape(-1), U.make_descs([n_samples] * n_reads))
        mapped = right = 0
        for i in range(n_reads):
            st = int(truth["start"][i])
            rid = int(np.searchsorted(offs, st, side="right")) - 1
            if not out[i]["mapped"]:
                continue
            mapped += 1
            o = st - offs[rid]
            if int(out[i]["rid"]) == rid and int(out[i]["rf_st"]) < o + 2000 and int(out[i]["rf_en"]) > o:
                right += 1
        print("1.1 Gbp mapping: %d of %d reads mapped, %d of them to their origin" % (mapped, n_reads, right))
        assert mapped >= n_reads // 2 and right >= 0.95 * mapped
        idx.close()
    finally:
        shutil.rmtree(work, ignore_errors=True)
