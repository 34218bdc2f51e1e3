// tests/emul/emul_events.cpp -- the `events` device routines (unc_events.cuh, K1's warp routine in its FULL variant) on
// the CPU under the warp emulator, laid out and ordered as unc_events_run / unc_events_annotate launch them (a row of
// n_samples slots per read; k_events_warp, then the serial redo of the flagged reads, the annotation, then the records
// gathered read after read).  Test vehicle only.
#include "unc_device.cuh"   // UNC_EMUL is defined on the command line
#include "unc_events.cuh"
#include "../../include/unc_b200.h"
#include "unc_host_index.hpp"
#include "unc_host_params.hpp"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

thread_local WarpEmu *g_warp = nullptr;

namespace {

struct WarpArgs { const DevBatch *B; const DevParams *p; K1WarpSmem *sm; u32 *sql; const K1FullOut *fo; };
void warp_entry(void *a) {
    WarpArgs *w = (WarpArgs *) a;
    const int warp = c_tid() >> 5;
    unc_k1_warp_main<true>(*w->B, *w->p, w->sm + warp, w->fo, w->sql + (size_t) warp * K1_SQL_WORDS);
}

struct Rows {
    std::vector<u64> row;
    std::vector<u32> n, start, mask;
    std::vector<float> mel, scale, shift, len, mean, stdv, norm, wm, ws;
    DevEvents view(u32 nr, u64 slots) {
        row.resize(nr + 1); n.resize(nr + 1); mel.resize(nr + 1); scale.resize(nr + 1); shift.resize(nr + 1);
        for (auto *v : {&start, &mask}) v->assign(slots + 1, 0xEEEEEEEEu);
        for (auto *v : {&len, &mean, &stdv, &norm, &wm, &ws}) v->assign(slots + 1, -12345.0f);
        DevEvents E;
        E.samples = nullptr; E.reads = nullptr; E.n_reads = nr; E.row = row.data(); E.n_events = n.data();
        E.mean_event_len = mel.data(); E.start = start.data(); E.length = len.data(); E.mean = mean.data();
        E.stdv = stdv.data(); E.norm_mean = norm.data(); E.scale = scale.data(); E.shift = shift.data();
        E.win_mean = wm.data(); E.win_stdv = ws.data(); E.win_mask = mask.data();
        return E;
    }
};

bool make_params(const char *model_path, const unc_event_params *prm, DevParams *dp) {
    HostIndex hx;
    if (!hix_load_model(hx, model_path)) return false;
    unc_params m;
    unc_fill_default_params(&m);
    m.threshold1 = prm->threshold1; m.threshold2 = prm->threshold2; m.peak_height = prm->peak_height;
    m.min_mean = prm->min_mean; m.max_mean = prm->max_mean;
    *dp = unc_make_dev_params(m, hx);
    return true;
}

}  // namespace

extern "C" {

// unc_events_run + unc_events_fetch: out_reads[n], out_events[sum of n_events] (the caller sizes it by the samples)
// n_warps: warps of the emulated CTA; force_serial: every read through the serial routine; *n_redone (optional): reads
// the warp routine flagged for the serial routine
int emu_events_run(const char *model_path, const unc_event_params *prm, const unc_read_desc *reads, uint32_t n,
                   const void *samples, unc_event_read *out_reads, unc_event_full *out_events, int n_warps_arg,
                   int force_serial, uint32_t *n_redone) {
    DevParams dp;
    if (!make_params(model_path, prm, &dp)) return -1;
    std::vector<DevReadDesc> d(n + 1);
    u64 slots = 0;
    Rows R;
    R.row.resize(n + 1);
    for (u32 i = 0; i < n; i++) {
        d[i].offset = reads[i].offset; d[i].n_samples = reads[i].n_samples; d[i].dtype = reads[i].dtype;
        d[i].cal_range = reads[i].cal_range; d[i].cal_offset = reads[i].cal_offset; d[i].cal_digit = reads[i].cal_digit;
        d[i].pad = 0;
        slots += reads[i].n_samples;
    }
    std::vector<u64> row(n + 1);
    u64 s = 0;
    for (u32 i = 0; i < n; i++) { row[i] = s; s += reads[i].n_samples; }
    DevEvents E = R.view(n, slots);
    std::copy(row.begin(), row.end(), R.row.begin());
    E.samples = samples; E.reads = d.data();
    // k_events_warp: K1's warp per read (FULL), n_warps warps taking reads from the queue
    DevBatch B{};
    u64 bytes = 0;
    for (u32 i = 0; i < n; i++) bytes = std::max<u64>(bytes, (reads[i].offset + reads[i].n_samples) * (reads[i].dtype ? 2 : 4));
    std::vector<u32> flags(n + 1, 0);
    u32 queue = 0;
    B.samples = samples; B.samples_bytes = bytes; B.reads = d.data(); B.n_reads = n;
    B.k1_queue = &queue; B.k1_flags = flags.data(); B.k1_stats = nullptr;
    B.events = nullptr; B.normed = nullptr; B.ev_stride = 0; B.n_events = R.n.data(); B.mean_event_len = R.mel.data();
    K1FullOut fo = {R.row.data(), R.start.data(), R.len.data(), R.mean.data(), R.stdv.data()};
    const int n_warps = n_warps_arg > 0 ? n_warps_arg : 2;
    K1WarpSmem *ksm = (K1WarpSmem *) aligned_alloc(16, sizeof(K1WarpSmem) * n_warps);
    memset(ksm, 0, sizeof(K1WarpSmem) * n_warps);
    std::vector<u32> sql((size_t) K1_SQL_WORDS * n_warps, 0xEEEEEEEEu);
    WarpArgs wa = {&B, &dp, ksm, sql.data(), &fo};
    if (n) emu_run_cta(warp_entry, &wa, 32 * n_warps);
    free(ksm);
    u32 redo = 0;
    for (u32 r = 0; r < n; r++)                                             // k_events_detect: the flagged reads
        if (flags[r] || force_serial) { unc_events_detect_read(E, dp, r); redo++; }
    if (n_redone) *n_redone = redo;
    for (u32 r = 0; r < n; r++) unc_events_annotate_read(E, dp, prm->win_stdv_min, r);   // k_events_annotate
    u64 o = 0;
    for (u32 r = 0; r < n; r++) {                                          // k_events_gather
        out_reads[r].n_events = R.n[r]; out_reads[r].mean_event_len = R.mel[r];
        out_reads[r].norm_scale = R.scale[r]; out_reads[r].norm_shift = R.shift[r];
        for (u32 i = 0; i < R.n[r]; i++, o++) {
            const u64 k = R.row[r] + i;
            unc_event_full &x = out_events[o];
            x.start = R.start[k]; x.length = R.len[k]; x.mean = R.mean[k]; x.stdv = R.stdv[k]; x.norm_mean = R.norm[k];
            x.win_mean = R.wm[k]; x.win_stdv = R.ws[k]; x.win_mask = R.mask[k];
        }
    }
    return 0;
}

// unc_events_annotate on the caller's means: read i is means[off[i] .. off[i+1])
int emu_events_annotate(const char *model_path, const unc_event_params *prm, uint32_t n, const uint64_t *off,
                        const float *means, float *norm_mean, float *win_mean, float *win_stdv, uint32_t *win_mask,
                        float *scale, float *shift) {
    DevParams dp;
    if (!make_params(model_path, prm, &dp)) return -1;
    const u64 total = off[n] - off[0];
    Rows R;
    DevEvents E = R.view(n, total);
    for (u32 i = 0; i < n; i++) { R.row[i] = off[i] - off[0]; R.n[i] = (u32) (off[i + 1] - off[i]); }
    std::copy(means + off[0], means + off[n], R.mean.begin());
    E.mean_event_len = nullptr;
    for (u32 r = 0; r < n; r++) unc_events_annotate_read(E, dp, prm->win_stdv_min, r);
    std::copy(R.norm.begin(), R.norm.begin() + total, norm_mean + off[0]);     // indexed like the means
    std::copy(R.wm.begin(), R.wm.begin() + total, win_mean + off[0]);
    std::copy(R.ws.begin(), R.ws.begin() + total, win_stdv + off[0]);
    std::copy(R.mask.begin(), R.mask.begin() + total, win_mask + off[0]);
    std::copy(R.scale.begin(), R.scale.begin() + n, scale);
    std::copy(R.shift.begin(), R.shift.begin() + n, shift);
    return 0;
}

}  // extern "C"
