"""ctypes binding of the C-ABI in include/unc_b200.h (uncalled_b200/libunc_b200.so).

The library holds ONLY the CUDA path.  Importing this module never falls back to a CPU
implementation: if the shared library is missing, or no CUDA device is usable, the calls
raise UncError.
"""
import ctypes as C
import os
import subprocess

import numpy as np

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG_DIR)
LIB_PATH = os.path.join(PKG_DIR, "libunc_b200.so")
MODEL_TABLE = os.path.join(PKG_DIR, "data", "r94_5mer_template.f32")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-fmad=false", "-std=c++17",
              "-Xcompiler", "-fPIC", "--shared", "-diag-suppress", "550"]


class UncError(RuntimeError):
    pass


class Params(C.Structure):
    """unc_params: mirror of Mapper::PRMS and sub-structs (reference src/mapper.cpp:29-52)."""
    _fields_ = [(n, C.c_uint32) for n in
                ("seed_len", "min_rep_len", "max_rep_copy", "max_paths", "max_consec_stay", "max_events")] + \
               [("max_stay_frac", C.c_float), ("min_seed_prob", C.c_float),
                ("min_map_len", C.c_uint32), ("min_mean_conf", C.c_float), ("min_top_conf", C.c_float),
                ("window_length1", C.c_uint32), ("window_length2", C.c_uint32),
                ("threshold1", C.c_float), ("threshold2", C.c_float), ("peak_height", C.c_float),
                ("min_mean", C.c_float), ("max_mean", C.c_float),
                ("bp_per_sec", C.c_float), ("sample_rate", C.c_float)]


class EventParams(C.Structure):
    """unc_event_params: EventDetector::Params and EventProfiler's win_len / win_stdv_min (reference
    src/event_detector.cpp:17-26, src/event_profiler.cpp:3-9)."""
    _fields_ = [("window_length1", C.c_uint32), ("window_length2", C.c_uint32), ("threshold1", C.c_float),
                ("threshold2", C.c_float), ("peak_height", C.c_float), ("min_mean", C.c_float), ("max_mean", C.c_float),
                ("win_len", C.c_uint32), ("win_stdv_min", C.c_float)]


class ReadDesc(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("n_samples", C.c_uint32), ("dtype", C.c_uint32),
                ("cal_range", C.c_float), ("cal_offset", C.c_float), ("cal_digit", C.c_float)]


class PafRec(C.Structure):
    _fields_ = [("mapped", C.c_int32), ("fwd", C.c_int32), ("rid", C.c_int32), ("status", C.c_int32),
                ("n_events", C.c_uint32), ("events_used", C.c_uint32), ("matches", C.c_uint32),
                ("n_clusters", C.c_uint32),
                ("rd_len", C.c_uint64), ("rd_st", C.c_uint64), ("rd_en", C.c_uint64),
                ("rf_st", C.c_uint64), ("rf_en", C.c_uint64), ("rf_len", C.c_uint64),
                ("n_children", C.c_uint64), ("n_sources", C.c_uint64), ("n_occ_blocks", C.c_uint64),
                ("n_sa_steps", C.c_uint64), ("n_seeds", C.c_uint64)]


PAF_DTYPE = np.dtype([("mapped", "<i4"), ("fwd", "<i4"), ("rid", "<i4"), ("status", "<i4"),
                      ("n_events", "<u4"), ("events_used", "<u4"), ("matches", "<u4"), ("n_clusters", "<u4"),
                      ("rd_len", "<u8"), ("rd_st", "<u8"), ("rd_en", "<u8"), ("rf_st", "<u8"), ("rf_en", "<u8"),
                      ("rf_len", "<u8"), ("n_children", "<u8"), ("n_sources", "<u8"), ("n_occ_blocks", "<u8"),
                      ("n_sa_steps", "<u8"), ("n_seeds", "<u8")])
DESC_DTYPE = np.dtype([("offset", "<u8"), ("n_samples", "<u4"), ("dtype", "<u4"), ("cal_range", "<f4"),
                       ("cal_offset", "<f4"), ("cal_digit", "<f4")], align=True)
assert PAF_DTYPE.itemsize == C.sizeof(PafRec) and DESC_DTYPE.itemsize == C.sizeof(ReadDesc)


class Timing(C.Structure):
    _fields_ = [("h2d_ms", C.c_float), ("k1_ms", C.c_float), ("k2_ms", C.c_float), ("d2h_ms", C.c_float),
                ("total_ms", C.c_float), ("kernel_launches", C.c_uint32),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("k1_events_ms", C.c_float), ("pad_", C.c_float)]


class IndexInfo(C.Structure):
    _fields_ = [("n_rows", C.c_uint64), ("n_seqs", C.c_int32), ("device", C.c_int32),
                ("device_bytes", C.c_uint64), ("n_kmer_groups", C.c_uint32)]


class Fast5Read(C.Structure):
    """unc_fast5_read (include/unc_b200.h)"""
    _fields_ = [("read_id", C.c_char_p), ("number", C.c_int32), ("start_sample", C.c_int32), ("channel", C.c_int32),
                ("cal_digitisation", C.c_float), ("cal_range", C.c_float), ("cal_offset", C.c_float),
                ("n_samples", C.c_uint64), ("sample_offset", C.c_uint64)]


EXPORTS = ["unc_strerror", "unc_last_error", "unc_device_count", "unc_init", "unc_shutdown", "unc_params_default",
           "unc_index_load", "unc_index_get_info", "unc_index_seq", "unc_index_kmer_range",
           "unc_index_thresholds", "unc_index_free", "unc_index_build", "unc_pool_create", "unc_pool_free",
           "unc_map_batch", "unc_map_batch_device", "unc_map_batch_ordered", "unc_pool_set_tie_order", "unc_map_batch_submit", "unc_map_batch_wait", "unc_pool_record", "unc_pool_elapsed", "unc_events_batch", "unc_match_probs", "unc_fm_step", "unc_fm_neighbors",
           "unc_fm_sa", "unc_pool_last_timing", "unc_pool_k1_stats", "unc_stream_create", "unc_stream_set_tie_order", "unc_stream_set_chunk_timeout", "unc_stream_last_step_ms", "unc_stream_channel_norm", "unc_stream_step", "unc_stream_replay",
           "unc_stream_free", "unc_self_align", "unc_free", "unc_fast5_open", "unc_fast5_count", "unc_fast5_info",
           "unc_fast5_load", "unc_fast5_close", "unc_fast5_last_error", "unc_dtw_batch", "unc_dtw_release", "unc_dtw_last_kernel_ms",
           "unc_mask_internal", "unc_mask_last_kernel_ms", "unc_mask_external", "unc_mask_external_last_kernel_ms",
           "unc_mask_external_last_times", "unc_index_build_device", "unc_index_build_device_last_times",
           "unc_index_build_device_last_active", "unc_dtw_aligner_create", "unc_dtw_aligner_free", "unc_dtw_aligner_contig",
           "unc_dtw_aligner_set_budget", "unc_dtw_align_batch", "unc_dtw_align_path", "unc_dtw_align_last_times",
           "unc_debug_held", "unc_dtw_batch_banded", "unc_dtw_aligner_set_band", "unc_event_params_default", "unc_events_create",
           "unc_events_free", "unc_events_run", "unc_events_fetch", "unc_events_annotate", "unc_match_probs_batch",
           "unc_events_last_times", "unc_repeats_create", "unc_repeats_lengths", "unc_repeats_last_kernel_ms",
           "unc_repeats_destroy", "unc_bwa_open", "unc_bwa_free", "unc_bwa_load_pac", "unc_bwa_info", "unc_bwa_seq",
           "unc_bwa_kmer_ranges", "unc_bwa_pos2rid", "unc_bwa_coord_to_pacseq", "unc_bwa_get_base", "unc_bwa_neighbor",
           "unc_bwa_sa", "unc_bwa_range_to_fms", "unc_bwa_get_kmers", "unc_bwa_last_kernel_ms"]


def build(force=False, verbose=False):
    """Compile uncalled_b200/libunc_b200.so for sm_90a (H100) with nvcc (cross-compiles without a GPU)."""
    src_dir = os.path.join(PKG_DIR, "csrc")
    srcs = [os.path.join(src_dir, f) for f in ("unc_abi.cu", "unc_index_build.cpp", "unc_fast5.cpp")]
    deps = srcs + [os.path.join(src_dir, f) for f in
                   ("unc_device.cuh", "unc_k2v2.cuh", "unc_dtw.cuh", "unc_dtw_band.cuh", "unc_dtw_plan.hpp", "unc_dtw_host.inl", "unc_dtw_align.cuh", "unc_dtw_align_host.inl", "unc_k1.cuh", "unc_stream.cuh", "unc_stream_host.inl", "unc_stream_logic.hpp", "unc_replay.cuh", "unc_replay_host.inl", "unc_events.cuh", "unc_events_host.inl", "unc_ordered_logic.hpp", "unc_pdqsort.cuh", "unc_warp.cuh",
                    "unc_selfalign.cuh", "unc_selfalign_host.hpp", "unc_selfalign_host.inl", "unc_repeats_host.inl", "unc_bwa.cuh", "unc_bwa_host.inl",
                    "unc_mask.cuh", "unc_mask_host.hpp", "unc_mask_host.inl",
                    "unc_mask_ext.cuh", "unc_mask_ext_host.hpp", "unc_mask_ext_host.inl",
                    "unc_fmb.cuh", "unc_fmb_run.hpp", "unc_fmb_host.inl", "unc_index_host.hpp",
                    "unc_host_index.hpp", "unc_host_params.hpp")] + \
        [os.path.join(ROOT, "include", "unc_b200.h")]
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(d) for d in deps):
        return LIB_PATH
    cmd = ["nvcc"] + NVCC_FLAGS + ["-o", LIB_PATH] + srcs + ["-lz"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise UncError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stdout + r.stderr)
    return LIB_PATH


def build_pymodule(force=False):
    """Compile the `_uncalled` extension module (csrc/pyuncalled.cpp, pybind11) next to libunc_b200.so: the reference's
    Python package imports its C++ core under that name (uncalled/__init__.py:1), so with this directory and the
    reference's `uncalled/` on PYTHONPATH its own `scripts/uncalled` runs on the GPU path."""
    import sysconfig
    import pybind11
    src = os.path.join(PKG_DIR, "csrc", "pyuncalled.cpp")
    out = os.path.join(PKG_DIR, "_uncalled" + sysconfig.get_config_var("EXT_SUFFIX"))
    deps = [src, os.path.join(ROOT, "include", "unc_b200.h")]
    if not force and os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    cmd = ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + pybind11.get_include(), "-I" + sysconfig.get_paths()["include"],
           src, "-o", out, "-L" + PKG_DIR, "-lunc_b200", "-Wl,-rpath,$ORIGIN"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise UncError("g++ failed on pyuncalled.cpp:\n" + r.stdout + r.stderr)
    return out


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise UncError("uncalled_b200/libunc_b200.so is missing: run `python -c 'import __graft_entry__ as g; "
                       "g.build()'` (there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    L.unc_strerror.restype = C.c_char_p
    L.unc_strerror.argtypes = [C.c_int]
    L.unc_last_error.restype = C.c_char_p
    L.unc_init.argtypes = [C.c_int]
    L.unc_params_default.argtypes = [C.POINTER(Params)]
    L.unc_index_load.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(vp)]
    L.unc_index_get_info.argtypes = [vp, C.POINTER(IndexInfo)]
    L.unc_index_seq.argtypes = [vp, C.c_int, C.POINTER(C.c_char_p), C.POINTER(u64)]
    L.unc_index_kmer_range.argtypes = [vp, u32, C.POINTER(u64), C.POINTER(u64)]
    L.unc_index_thresholds.argtypes = [vp, C.POINTER(C.c_float)]
    L.unc_index_free.argtypes = [vp]
    L.unc_index_free.restype = None
    L.unc_index_build.argtypes = [C.c_char_p, C.c_char_p]
    L.unc_index_build_device.argtypes = [C.c_char_p, C.c_char_p]
    L.unc_index_build_device_last_times.argtypes = [C.POINTER(C.c_float), C.POINTER(u32), C.POINTER(u64)]
    L.unc_index_build_device_last_times.restype = None
    L.unc_index_build_device_last_active.argtypes = [C.POINTER(u64), u32]
    L.unc_index_build_device_last_active.restype = u32
    L.unc_pool_create.argtypes = [vp, C.POINTER(Params), u32, u64, C.POINTER(vp)]
    L.unc_pool_free.argtypes = [vp]
    L.unc_pool_free.restype = None
    L.unc_map_batch.argtypes = [vp, vp, u32, vp, vp]
    L.unc_map_batch_device.argtypes = [vp, vp, u32, vp, vp]
    L.unc_map_batch_ordered.argtypes = [vp, vp, u32, vp, C.c_int, vp, vp, C.POINTER(u32), C.POINTER(u32)]
    L.unc_pool_set_tie_order.argtypes = [vp, C.c_int]
    L.unc_map_batch_submit.argtypes = [vp, vp, u32, vp, C.c_int]
    L.unc_map_batch_wait.argtypes = [vp, vp]
    L.unc_pool_record.argtypes = [vp, C.c_int]
    L.unc_pool_elapsed.argtypes = [vp, C.c_int, vp, C.c_int, C.POINTER(C.c_float)]
    L.unc_events_batch.argtypes = [vp, vp, u32, vp, u32, vp, vp, vp, vp]
    L.unc_match_probs.argtypes = [vp, C.c_float, vp]
    L.unc_fm_step.argtypes = [vp, u32, vp, vp, vp, vp, vp, vp]
    L.unc_fm_neighbors.argtypes = [vp, u32, vp, vp, vp, vp, vp]
    L.unc_fm_sa.argtypes = [vp, u32, vp, vp]
    L.unc_pool_last_timing.argtypes = [vp, C.POINTER(Timing)]
    L.unc_pool_k1_stats.argtypes = [vp, vp]
    L.unc_stream_create.argtypes = [vp, C.POINTER(Params), u32, u32, u32, C.POINTER(vp)]
    L.unc_stream_step.argtypes = [vp, vp, u32, vp, vp]
    L.unc_stream_set_tie_order.argtypes = [vp, C.c_int]
    L.unc_stream_set_chunk_timeout.argtypes = [vp, C.c_float]
    L.unc_stream_last_step_ms.argtypes = [vp]
    L.unc_stream_last_step_ms.restype = C.c_float
    L.unc_stream_channel_norm.argtypes = [vp, u32, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(u32), C.POINTER(u32)]
    L.unc_stream_replay.argtypes = [vp, vp, u32, vp, vp]
    L.unc_stream_free.argtypes = [vp]
    L.unc_stream_free.restype = None
    L.unc_self_align.argtypes = [C.c_char_p, u32, C.POINTER(C.c_uint64), C.POINTER(vp), C.POINTER(vp)]
    L.unc_free.argtypes = [vp]
    L.unc_free.restype = None
    L.unc_fast5_open.argtypes = [C.c_char_p, C.POINTER(vp)]
    L.unc_fast5_count.argtypes = [vp, C.POINTER(u32), C.POINTER(C.c_int)]
    L.unc_fast5_info.argtypes = [vp, u32, C.POINTER(Fast5Read)]
    L.unc_fast5_load.argtypes = [vp, u32, u32, C.c_uint64, vp, C.c_uint64, C.POINTER(Fast5Read), C.c_int]
    L.unc_fast5_close.argtypes = [vp]
    L.unc_fast5_close.restype = None
    L.unc_fast5_last_error.restype = C.c_char_p
    L.unc_mask_internal.argtypes = [C.c_char_p, C.c_char_p, u32, u32, vp, vp, C.POINTER(u32)]
    L.unc_mask_last_kernel_ms.argtypes = []
    L.unc_mask_last_kernel_ms.restype = C.c_float
    L.unc_mask_external.argtypes = [C.c_char_p, C.c_char_p, u32, u32, C.c_char_p, C.c_char_p, u64, vp, C.POINTER(u64),
                                    C.POINTER(u64)]
    L.unc_mask_external_last_kernel_ms.argtypes = []
    L.unc_mask_external_last_kernel_ms.restype = C.c_float
    L.unc_mask_external_last_times.argtypes = [vp, C.POINTER(u64)]
    L.unc_mask_external_last_times.restype = None
    L.unc_dtw_aligner_create.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(vp)]
    L.unc_dtw_aligner_free.argtypes = [vp]
    L.unc_dtw_aligner_free.restype = None
    L.unc_dtw_aligner_contig.argtypes = [vp, C.c_char_p, C.POINTER(C.c_int32), C.POINTER(u64)]
    L.unc_dtw_aligner_set_budget.argtypes = [vp, u64]
    L.unc_dtw_aligner_set_band.argtypes = [vp, u32]
    L.unc_dtw_align_batch.argtypes = [vp, u32, vp, vp, vp, C.c_int, vp]
    L.unc_dtw_align_path.argtypes = [vp, u32, vp, vp, vp]
    L.unc_dtw_align_last_times.argtypes = [vp, vp, C.POINTER(u64), C.POINTER(u64)]
    L.unc_debug_held.argtypes = [C.POINTER(u64), C.POINTER(u64), C.POINTER(u32)]
    L.unc_event_params_default.argtypes = [C.POINTER(EventParams)]
    L.unc_events_create.argtypes = [C.c_char_p, C.POINTER(EventParams), C.POINTER(vp)]
    L.unc_events_free.argtypes = [vp]
    L.unc_events_free.restype = None
    L.unc_events_run.argtypes = [vp, vp, u32, vp, C.c_int, vp]
    L.unc_events_fetch.argtypes = [vp, vp]
    L.unc_events_annotate.argtypes = [vp, u32, vp, vp, vp, vp, vp, vp, vp, vp]
    L.unc_match_probs_batch.argtypes = [vp, vp, u64, vp]
    L.unc_events_last_times.argtypes = [vp, C.POINTER(C.c_float)]
    L.unc_repeats_create.argtypes = [C.c_char_p, C.POINTER(vp)]
    L.unc_repeats_lengths.argtypes = [vp, u64, u32, vp]
    L.unc_repeats_last_kernel_ms.argtypes = [vp, C.POINTER(C.c_float)]
    L.unc_repeats_destroy.argtypes = [vp]
    L.unc_repeats_destroy.restype = None
    L.unc_bwa_open.argtypes = [C.c_char_p, C.c_int, C.c_int, C.POINTER(vp)]
    L.unc_bwa_free.argtypes = [vp]
    L.unc_bwa_free.restype = None
    L.unc_bwa_load_pac.argtypes = [vp]
    L.unc_bwa_info.argtypes = [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(C.c_int32), C.POINTER(C.c_int32), vp]
    L.unc_bwa_seq.argtypes = [vp, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(u64), C.POINTER(u64)]
    L.unc_bwa_kmer_ranges.argtypes = [vp, vp, vp]
    L.unc_bwa_pos2rid.argtypes = [vp, u64]
    L.unc_bwa_pos2rid.restype = C.c_int32
    L.unc_bwa_coord_to_pacseq.argtypes = [vp, C.c_char_p, u64, C.POINTER(u64)]
    L.unc_bwa_get_base.argtypes = [vp, u64, C.POINTER(C.c_uint8)]
    L.unc_bwa_neighbor.argtypes = [vp, u64, vp, vp, vp, vp, vp]
    L.unc_bwa_sa.argtypes = [vp, u64, vp, vp]
    L.unc_bwa_range_to_fms.argtypes = [vp, C.c_char_p, u64, u64, vp, vp]
    L.unc_bwa_get_kmers.argtypes = [vp, u64, u64, vp]
    L.unc_bwa_last_kernel_ms.argtypes = [vp, C.POINTER(C.c_float)]
    _lib = L
    return L


def check(rc):
    if rc != 0:
        L = lib()
        raise UncError("%s: %s" % (L.unc_strerror(rc).decode(), L.unc_last_error().decode()))


def default_params():
    p = Params()
    check(lib().unc_params_default(C.byref(p)))
    return p
