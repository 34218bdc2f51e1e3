"""Helpers of the map-ord tests and tools/bench_map_ord.py.

  * host_map_ord: the host-stepped MapPoolOrd loop (reference src/map_pool_ord.cpp:61-121) over api.RealtimePool, one
    unc_stream_step per update: the reference path the device replay (api.MapPoolOrd) is checked and timed against.
  * EmuReplay / EmuReplayStream: an emulated index and stream of tests/emul/emul_replay.cpp, whose emu_stream_replay is
    the CPU counterpart of unc_stream_replay (and whose emu_stream_step serves the host-stepped loop).
  * synthetic_run: a seeded run of many channels, several reads per channel with increasing start times.
"""
import ctypes as C
import os
import subprocess

import numpy as np

import emulib
import synth

CAL = (1467.61, 10.0, 8192.0)    # (range, offset, digitisation) of the int16 runs


class Read:
    __slots__ = ("id", "channel", "number", "start", "signal", "cal")

    def __init__(self, rid, channel, number, start, signal, cal=None):
        self.id, self.channel, self.number, self.start, self.signal, self.cal = rid, channel, number, start, signal, cal


def order_channels(reads, n_channels, max_len=None):
    """MapPoolOrd::load_fast5s: reads grouped by channel (1-based in the reads), each channel sorted by start sample (ties
    in list order), signals cut to max_len; reads without samples dropped."""
    chans = [[] for _ in range(n_channels)]
    for i, r in enumerate(reads):
        sig = r.signal if max_len is None else r.signal[:max_len]
        if len(sig):
            chans[r.channel - 1].append((r.start % (1 << 64), i, Read(r.id, r.channel, r.number, r.start, sig, r.cal)))
    return [[t[2] for t in sorted(q, key=lambda t: t[:2])] for q in chans]


def host_map_ord(pool, chans, chunk_len, min_active_reads=0):
    """MapPoolOrd::update over `pool` (api.RealtimePool) until nothing runs: every update each channel offers its front
    read's next chunk (ReadBuffer::get_chunk: the last one partial, then empty) through try_add_chunk and advances only
    when it is accepted; each result pops the channel's front read.  RealtimePool.update returns a read in the update
    that finishes it, so is_read_finished is never true at the top of an update.  After each update, fewer than
    min_active_reads channels with a read in progress stop everything.  Returns [(update index, Paf)]."""
    from uncalled_b200.api import Chunk
    chans = [list(q) for q in chans]
    idx = [0] * len(chans)
    out, u = [], 0
    while True:
        empty = True
        for i, q in enumerate(chans):
            if not q:
                continue
            empty = False
            r = q[0]
            st = idx[i] * chunk_len
            c = Chunk(r.id, i + 1, r.number, r.start + st, r.signal, min(st, len(r.signal)), chunk_len, calibration=r.cal)
            if pool.try_add_chunk(c):
                idx[i] += 1
        for ch, nm, paf in pool.update():
            i = ch - 1
            if chans[i] and chans[i][0].number == nm:
                chans[i].pop(0)
                idx[i] = 0
            out.append((u, paf))
        active = sum(r is not None for r in pool._read)
        if active < min_active_reads:
            pool.stop_all()
            break
        if empty and pool.all_finished():
            break
        u += 1
    return out


_lib = None


def emu_lib():
    """tests/emul/emul_replay.cpp compiled for the host: the emulator harness of emul_main.cpp plus emu_stream_replay."""
    global _lib
    if _lib is None:
        src = os.path.join(emulib.EMUL_DIR, "emul_replay.cpp")
        out = os.path.join(emulib.EMUL_DIR, "libunc_emul_replay.so")
        csrc = os.path.join(emulib.ROOT, "uncalled_b200", "csrc")
        deps = [src, os.path.join(emulib.EMUL_DIR, "emul_main.cpp"), os.path.join(emulib.EMUL_DIR, "warp_emul.hpp"),
                os.path.join(emulib.ROOT, "include", "unc_b200.h")] + \
            [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
        if not (os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps)):
            tmp = os.path.join(emulib.EMUL_DIR, "libunc_emul_replay.%d.tmp.so" % os.getpid())
            subprocess.run(["g++", "-O2", "-g", "-std=c++17", "-ffp-contract=off", "-DUNC_EMUL", "-DK2_MAXSEG=16u", "-fPIC",
                            "-shared", "-I" + emulib.EMUL_DIR, "-I" + csrc, "-o", tmp, src], check=True, capture_output=True)
            os.replace(tmp, out)
        L = emulib._bind(C.CDLL(out))
        L.emu_stream_replay.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_int]
        L.emu_replay_stream_free.argtypes = [C.c_void_p]
        _lib = L
    return _lib


class EmuReplay(emulib.Emu):
    """An emulated index in the replay library (its streams serve both the step and the replay calls)."""

    def __init__(self, prefix, preset="default"):
        self.L = emu_lib()
        self.idx = self.L.emu_index_load(prefix.encode(), preset.encode(), emulib.MODEL_TABLE.encode())
        if not self.idx:
            raise RuntimeError("emu_index_load failed")
        self.params = emulib.default_params()


class EmuReplayStream(emulib.EmuStream):
    """An emulated stream of an EmuReplay index, with emu_stream_replay (tests/emul/emul_replay.cpp) besides step()."""

    def replay(self, reads, n, flat, out):
        flat = np.ascontiguousarray(flat)
        rc = self.emu.L.emu_stream_replay(self.h, reads, n, flat.ctypes.data, out, self.n_warps)
        if rc not in (0, -7):
            raise RuntimeError("emu_stream_replay rc=%d" % rc)
        return rc

    def close(self):
        if self.h:
            self.emu.L.emu_replay_stream_free(self.h)
            self.h = None


def seqs_of(oracle):
    return [(oracle.lib.orc_seq_name(oracle.idx, i).decode(), int(oracle.lib.orc_seq_len(oracle.idx, i)))
            for i in range(oracle.lib.orc_n_seqs(oracle.idx))]


class SeqIndex:
    def __init__(self, seqs):
        self.seqs = seqs


def synthetic_run(g, n_channels, reads_per_channel, n_samples, seed, int16=True, whole_chunks=None):
    """A seeded run: n_channels x reads_per_channel reads of up to n_samples samples, about half from the genome, spread
    round-robin over the channels with increasing start times.  With whole_chunks=L every signal is cut to a multiple of L
    (the oracle's channel mode takes whole chunks only); otherwise lengths vary by up to 1.5 chunks of 4000."""
    n = n_channels * reads_per_channel
    sigs, _ = synth.reads(g, n, n_samples, seed=seed, frac_random=0.5)
    rng = np.random.default_rng(seed)
    reads = []
    for i in range(n):
        s = np.asarray(sigs[i])[:n_samples - int(rng.integers(0, 6000))]
        if whole_chunks:
            s = s[:len(s) // whole_chunks * whole_chunks]
        cal = None
        if int16:
            s = np.round(s * CAL[2] / CAL[0] - CAL[1]).astype(np.int16)
            cal = CAL
        else:
            s = np.ascontiguousarray(s, np.float32)
        ch = 1 + i % n_channels
        reads.append(Read("r%05d" % i, ch, i, 1000 + 50000 * (i // n_channels) + int(rng.integers(0, 1000)), s, cal))
    return reads


def pcal(sig, cal):
    """The calibrated signal as the device computes it from int16 (u16 reinterpretation, src/read_buffer.cpp:239-242)."""
    if cal is None:
        return np.asarray(sig, np.float32)
    rng, off, dig = (np.float32(x) for x in cal)
    return (rng * (np.asarray(sig).view(np.uint16).astype(np.float32) + off) / dig).astype(np.float32)


def paf_fields(p):
    """The comparable part of a Paf line: the 12 columns, ch, st and whether it is ended."""
    return (tuple(p.fields()), tuple(p.int_tags), p.is_ended())

