"""fast5 input through the native reader (uncalled_b200/csrc/unc_fast5.cpp, no libhdf5 / h5py needed): what the
reference's Fast5Reader + ReadBuffer(hdf5_tools::File&, raw_path, ch_path) hand to the mapper
(src/fast5_reader.cpp:134-248, src/read_buffer.cpp:198-246).  Signals stay int16 DAC values; the calibration
(with the reference's u16 reinterpretation) happens on the GPU."""
import ctypes as C
import os

import numpy as np

from . import _native as N


class Fast5Error(RuntimeError):
    pass


class Fast5Read:
    __slots__ = ("read_id", "number", "start_sample", "channel", "calibration", "signal", "n_samples")

    def __init__(self, info, signal):
        self.read_id = (info.read_id or b"").decode("utf-8", "replace")
        self.number, self.start_sample, self.channel = info.number, info.start_sample, info.channel
        self.n_samples = int(info.n_samples)         # the signal's length in the file
        self.calibration = (info.cal_range, info.cal_offset, info.cal_digitisation)   # MapPool.add_read order
        self.signal = signal

    def pa(self):
        """The calibrated signal exactly as src/read_buffer.cpp:239-242 computes it (host copy, for tests)."""
        rng, off, dig = (np.float32(x) for x in self.calibration)
        return (rng * (self.signal.view(np.uint16).astype(np.float32) + off) / dig).astype(np.float32)


class Fast5File:
    """One single- or multi-read fast5 file."""

    def __init__(self, path):
        self._L = N.lib()
        self._h = C.c_void_p()
        if self._L.unc_fast5_open(os.fsencode(path), C.byref(self._h)) != 0:
            self._h = None
            raise Fast5Error(self._L.unc_fast5_last_error().decode("utf-8", "replace"))
        n, single = C.c_uint32(), C.c_int()
        self._L.unc_fast5_count(self._h, C.byref(n), C.byref(single))
        self.n_reads, self.single_read_format, self.path = n.value, bool(single.value), path

    def __len__(self):
        return self.n_reads

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def close(self):
        if getattr(self, "_h", None) is not None:
            self._L.unc_fast5_close(self._h)
            self._h = None

    __del__ = close

    def info(self, i):
        r = N.Fast5Read()
        if self._L.unc_fast5_info(self._h, i, C.byref(r)) != 0:
            raise Fast5Error(self._L.unc_fast5_last_error().decode("utf-8", "replace"))
        return Fast5Read(r, None)

    def load(self, first=0, n=None, max_samples_per_read=0, threads=0):
        """Reads [first, first+n): decoded by `threads` host threads (0 = all) into one int16 buffer."""
        n = self.n_reads - first if n is None else n
        infos = (N.Fast5Read * max(n, 1))()
        total = 0
        for i in range(n):
            if self._L.unc_fast5_info(self._h, first + i, C.byref(infos[i])) != 0:
                raise Fast5Error(self._L.unc_fast5_last_error().decode("utf-8", "replace"))
            ns = infos[i].n_samples
            total += min(ns, max_samples_per_read) if max_samples_per_read else ns
        buf = np.zeros(max(total, 1), np.int16)
        if self._L.unc_fast5_load(self._h, first, n, int(max_samples_per_read), buf.ctypes.data_as(C.c_void_p), total,
                                  infos, threads) != 0:
            raise Fast5Error(self._L.unc_fast5_last_error().decode("utf-8", "replace"))
        return [Fast5Read(infos[i], buf[infos[i].sample_offset:infos[i].sample_offset + infos[i].n_samples])
                for i in range(n)]
