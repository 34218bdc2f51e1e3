// unc_events.cuh -- `events`: what the signal front end of the mapper computes for a read, made visible.  For every
// event of the whole signal (no max_events cap): the reference's full Event and the per-event annotations of its
// DEBUG_EVENTS build (src/mapper.cpp:894-905,968-989).
//
//   (a) detect     EventDetector::get_events (src/event_detector.cpp:114-127) with create_event (:296-319): mean, stdv,
//                  start, length of every event that passes the min_mean / max_mean filter (:104-108).  K1 itself in
//                  its FULL variant: the warp per read of k1_warp_read<true> (unc_k1.cuh), then the serial routine
//                  below (K1's detector step unc_evdt_add<true>, one thread per read) for the reads whose sums fail
//                  K1's exactness condition -- the same split as k1_events / k1_fallback.
//   (b) normalise  the offline Normalizer over the read's event means towards the model (set_signal + at,
//                  src/normalizer.cpp:31-44,114-118), as Mapper::map_read uses it (src/mapper.cpp:193): K1's
//                  unc_norm_scale_shift, then scale * mean + shift per event.
//   (c) annotate   EventProfiler::add_event / anno_event / get_full_mask (src/event_profiler.hpp:71-151, defaults
//                  src/event_profiler.cpp:3-9): the 25-event window's mean and stdv (the streaming Normalizer's double
//                  recurrences, unc_ring_push) and the stall mask, tail loop included.  An event's fields are those of
//                  the add_event call after which it is next_evt_, i.e. when anno_event() would hand it out; the last
//                  events, which never get there, have win_mean = win_stdv = NaN and the tail loop's mask.
//
// (b) and (c) are serial recurrences over a read's events: one thread per read.  (b)+(c) also run on means the caller
// supplies (EventProfiler::get_full_mask over given events).
//
// Row layout: read r's events occupy slots row[r] .. row[r] + n_events[r] of each per-event array (structure of arrays;
// the detection path gives each read as many slots as it has samples, an upper bound of its event count).
#pragma once
#include "unc_device.cuh"
#include "unc_k1.cuh"        // unc_norm_scale_shift
#include "unc_stream.cuh"    // DevRing, unc_ring_*

struct DevEvents {
    const void *samples;             // (a) only
    const DevReadDesc *reads;        // (a) only
    u32 n_reads;
    const u64 *row;                  // first slot of read r
    u32 *n_events;                   // (a) writes, (b)(c) read
    float *mean_event_len;           // (a): EventDetector::mean_event_len (may be null for (b)(c))
    u32 *start;                      // Event fields
    float *length, *mean, *stdv;
    float *norm_mean;                // (b)
    float *scale, *shift;            // (b): per read
    float *win_mean, *win_stdv;      // (c)
    u32 *win_mask;
};

// (a) one read
UNC_DEV void unc_events_detect_read(const DevEvents &E, const DevParams &p, u32 r) {
    const DevReadDesc rd = E.reads[r];
    const u64 o = E.row[r];
    DevEvdt e;
    unc_evdt_reset(e);
    u32 ne = 0;
    for (u32 i = 0; i < rd.n_samples; i++) {
        DevEvdtFull f;
        float mean;
        if (!unc_evdt_add<true>(e, p, unc_sample(E.samples, rd, i), &mean, &f)) continue;
        E.start[o + ne] = f.start;
        E.length[o + ne] = (float) f.length;
        E.mean[o + ne] = f.mean;
        E.stdv[o + ne] = f.stdv;
        ne++;
    }
    E.n_events[r] = ne;
    if (E.mean_event_len) E.mean_event_len[r] = f_div(e.len_sum, (float) e.total_events);
}

// (b) + (c) one read
UNC_DEV void unc_events_annotate_read(const DevEvents &E, const DevParams &p, float win_stdv_min, u32 r) {
    const u64 o = E.row[r];
    const u32 ne = E.n_events[r];
    const float *mean = E.mean + o;
    // (b)
    float scale = 0.0f, shift = 0.0f;
    if (ne > 0) {
        unc_norm_scale_shift(mean, ne, p.tgt_mean, p.tgt_stdv, &scale, &shift);
        for (u32 i = 0; i < ne; i++) E.norm_mean[o + i] = f_add(f_mul(scale, mean[i]), shift);
    }
    E.scale[r] = scale;
    E.shift[r] = shift;
    // (c) get_full_mask: entry m is decided by the add_event call that makes event m next_evt_
    DevRing win;
    float win_sig[UNC_EVP_WIN];
    unc_ring_reset(win, win_sig);
    u32 to_mask = 0, m = 0;
    bool is_full = false;
    for (u32 i = 0; i < ne; i++) {
        unc_ring_push(win, win_sig, UNC_EVP_WIN, mean[i]);
        if (unc_ring_unread(win) <= UNC_EVP_WIN / 2u) continue;
        const float wm = (float) win.mean;                                           // Normalizer::get_mean
        const float ws = (float) d_sqrt(d_div(win.varsum, (double) win.n));           // Normalizer::get_stdv
        if (ws < win_stdv_min) to_mask = UNC_EVP_WIN - 1u;
        else if (to_mask > 0) to_mask--;
        if (win.is_full) {                                                            // next_evt_ = events_.front(); pop
            win.rd = (win.rd + 1u) % UNC_EVP_WIN;
            win.is_full = 0;
            is_full = true;
        }
        if (is_full) {
            E.win_mean[o + m] = wm;
            E.win_stdv[o + m] = ws;
            E.win_mask[o + m] = to_mask == 0 ? 1u : 0u;
            m++;
        }
    }
    const float nan = u2f(0x7FC00000u);
    for (; m < ne; m++) {                                                             // the tail loop (:142-149)
        E.win_mean[o + m] = nan;
        E.win_stdv[o + m] = nan;
        if (to_mask == 0) E.win_mask[o + m] = 1u;
        else { E.win_mask[o + m] = 0u; to_mask--; }
    }
}
