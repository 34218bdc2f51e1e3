// tests/emul/emul_main.cpp -- runs the DEVICE source (uncalled_b200/csrc/unc_device.cuh,
// compiled with -DUNC_EMUL) on the CPU under the 32-fiber warp emulator.  Test vehicle only:
// it lets the CPU-only test tier compare the warp-cooperative kernel logic with the oracle.
#include "unc_device.cuh"   // UNC_EMUL is defined on the command line
#include "unc_k1.cuh"
#include "unc_stream.cuh"
#include "unc_stream_logic.hpp"
#include "unc_ordered_logic.hpp"
#include "unc_selfalign.cuh"
#include "unc_selfalign_host.hpp"
#include "../../include/unc_b200.h"
#include "unc_host_index.hpp"
#include "unc_host_params.hpp"

thread_local WarpEmu *g_warp = nullptr;

struct EmuIndex {
    HostIndex h;
    DevIndex ix;
    std::vector<uint2> kmer_range;
    std::vector<float> lv_mean, lv_var2, lognorm;
    std::vector<uint4> occ2;
    K2V2Tab kt;
};

extern "C" {

void *emu_index_load(const char *prefix, const char *preset, const char *model_table) {
    EmuIndex *e = new EmuIndex();
    if (!hix_load_model(e->h, model_table) || !hix_load(e->h, prefix, preset ? preset : "default")) {
        fprintf(stderr, "emu_index_load: %s\n", e->h.error.c_str());
        delete e;
        return nullptr;
    }
    HostIndex &h = e->h;
    DevIndex &ix = e->ix;
    ix.bwt = (const uint4 *) h.bwt.data();
    ix.sa = h.sa32.data();
    ix.sa_full = nullptr;
    ix.lv_mean = h.lv_mean.data(); ix.lv_var2 = h.lv_var2.data(); ix.lognorm = h.lognorm.data();
    ix.thresh = h.thresh;
    ix.primary = (u32) h.primary; ix.seq_len = (u32) h.seq_len;
    for (int i = 0; i < 5; i++) ix.L2[i] = (u32) h.L2[i];
    ix.start_bits = 64 - __builtin_clzll(h.seq_len);
    e->kmer_range.resize(1024);
    for (u32 k = 0; k < 1024; k++) e->kmer_range[k] = unc_kmer_range_compute(ix, k);
    ix.kmer_range = e->kmer_range.data();
    {   // the GPU-side Occ layout and the k-mer rank tables, as unc_index_load builds them
        const u32 n_blk = (u32) (h.bwt.size() / 16) * 2u;
        e->occ2.resize((size_t) n_blk * 2);
        for (u32 j = 0; j < n_blk; j++) unc_occ2_build_block(ix.bwt, j, e->occ2.data());
        ix.occ2 = e->occ2.data();
        if (!hix_k2v2_tab(e->kmer_range.data(), e->kt)) { fprintf(stderr, "emu_index_load: too many overlapping k-mer ranges\n"); delete e; return nullptr; }
        ix.kt = &e->kt;
    }
    return e;
}

void emu_index_free(void *p) { delete (EmuIndex *) p; }

void emu_kmer_range(void *p, uint32_t k, uint64_t *st, uint64_t *en) {
    EmuIndex *e = (EmuIndex *) p;
    *st = e->kmer_range[k].x; *en = e->kmer_range[k].y;
}

struct CtaArgs {
    const DevIndex *ix; const DevParams *p; const DevBatch *B; const DevWork *W; K2Shared *sh;
};
struct K1Args { const DevBatch *B; const DevParams *p; K1WarpSmem *sm; };
static void k1_entry(void *a) {
    K1Args *w = (K1Args *) a;
    unc_k1_warp_main(*w->B, *w->p, w->sm + (c_tid() >> 5));
}
static uint32_t g_k1_stats[4];
extern "C" void emu_k1_stats(uint32_t *out) { memcpy(out, g_k1_stats, sizeof(g_k1_stats)); }

static int g_tie_order = 0;       // emu_set_tie_order: 1 = the exact-ties kernel (k2_map_exact of unc_abi.cu)
// The device seed tracker alone under the emulator (one warp): the seeds one by one through trk_add_seed, after each the state
// the oracle's orc_tracker_run reports.  `dir_fast_cap` entries of the directory live in a separate ("shared memory") array
// first, so that a small value exercises its move to the workspace.
struct TrkArgs { DevParams p; const u32 *ref_en, *ref_len, *evt; u32 n; u32 *out; uint4 *clu, *dir, *dir_fast; u32 max_blocks, dir_fast_cap; u32 overflow; };
static void trk_entry(void *vp) {
    TrkArgs *a = (TrkArgs *) vp;
    Tracker t;
    t.blocks = a->clu; t.dir_glob = a->dir; t.max_blocks = a->max_blocks;
    t.dir = a->dir_fast_cap ? a->dir_fast : a->dir; t.dir_cap = a->dir_fast_cap;
    trk_reset(t);
    for (u32 i = 0; i < a->n; i++) {
        trk_add_seed(t, a->p, a->ref_en[i], a->ref_len[i], a->evt[i]);
        if (w_lane() == 0) {
            u32 *o = a->out + (size_t) 6 * i;
            o[0] = t.n_live; o[1] = t.max_map.total_len; o[2] = t.max_map.ren_start; o[3] = t.max_map.evt_en;
            o[4] = trk_get_final(t, a->p) ? t.max_map.total_len : 0u; o[5] = t.n_lens;
        }
        w_sync();
    }
    if (w_lane() == 0) a->overflow = t.overflow | ((t.dir == t.dir_glob ? 1u : 0u) << 1);
}
extern "C" int emu_tracker_run(uint32_t min_map_len, float min_mean_conf, float min_top_conf, const uint32_t *ref_en, const uint32_t *ref_len,
                               const uint32_t *evt, uint32_t n, uint32_t *out, uint32_t max_blocks, uint32_t dir_fast_cap) {
    TrkArgs a;
    memset(&a.p, 0, sizeof(a.p));
    a.p.min_map_len = min_map_len; a.p.min_mean_conf = min_mean_conf; a.p.min_top_conf = min_top_conf;
    a.ref_en = ref_en; a.ref_len = ref_len; a.evt = evt; a.n = n; a.out = out;
    std::vector<uint4> clu((size_t) max_blocks * 32 * 2), dir(max_blocks + 1), fast(dir_fast_cap + 1);
    a.clu = clu.data(); a.dir = dir.data(); a.dir_fast = fast.data(); a.max_blocks = max_blocks; a.dir_fast_cap = dir_fast_cap; a.overflow = 0;
    emu_run_warp(trk_entry, &a);
    return (int) a.overflow;      // bit 0: block store overflowed, bit 1: the directory ended in the workspace
}

// The mapper's per-event trace in the oracle's row layout (orc_trace_row / orc_trace_seed of oracle/unc_oracle.h), so
// that a test compares the path buffers of both sides byte for byte.  item = the batch index, or the channel when streaming.
struct EmuTraceRow {
    uint64_t fm_start, fm_end;
    uint32_t kmer, length, consec_stays, sa_checked, event_moves, seed_prob, prob_sum, valid;
};
struct EmuTraceSeed {
    uint64_t ref_end;
    uint32_t move_count, evt;
};
typedef void (*EmuPathTraceFn)(void *ud, uint32_t item, uint32_t event_i, uint32_t nn, const EmuTraceRow *rows, uint32_t n_seeds,
                               const EmuTraceSeed *seeds, const uint32_t *flags, uint32_t overflow);
static EmuPathTraceFn g_trace_fn = nullptr;
static void *g_trace_ud = nullptr;
static void emu_path_trace_decode(u32 item, u32 event_i, u32 nn, const uint4 *recs, const u32 *order, u32 n_rows,
                                  const uint2 *rl, const u32 *flags, u32 overflow) {
    std::vector<EmuTraceRow> rows(nn + 1);
    memset(rows.data(), 0, rows.size() * sizeof(EmuTraceRow));
    for (u32 i = 0; i < nn; i++) {
        if (order[i] & UNC_INVALID) continue;               // a dup: invalidated at its position
        const uint4 q0 = recs[(size_t) order[i] * 2], q1 = recs[(size_t) order[i] * 2 + 1];
        EmuTraceRow &o = rows[i];
        o.fm_start = q0.x; o.fm_end = q0.y;
        o.kmer = q0.z & UNC_KMASK; o.length = (q0.z >> 16) & 0xFFu; o.consec_stays = (q0.z >> 24) & 0xFFu;
        o.event_moves = q0.w & UNC_PATH_MASK; o.sa_checked = q0.w >> 31;
        o.seed_prob = q1.x; o.prob_sum = q1.y; o.valid = 1;
    }
    std::vector<EmuTraceSeed> seeds(n_rows + 1);
    for (u32 j = 0; j < n_rows; j++) {
        seeds[j].ref_end = rl[j].x; seeds[j].move_count = rl[j].y & 0xFFu;
        seeds[j].evt = (rl[j].y & 0x100u) ? event_i - 1u : event_i;
    }
    if (g_trace_fn) g_trace_fn(g_trace_ud, item, event_i, nn, rows.data(), n_rows, seeds.data(), flags, overflow);
}
extern "C" void emu_set_path_trace(EmuPathTraceFn fn, void *ud) {
    g_trace_fn = fn; g_trace_ud = ud;
    g_emu_path_trace = fn ? emu_path_trace_decode : nullptr;
}
// how often the bucket phases met each of their edges (K2S_* of unc_device.cuh), since the last reset
extern "C" uint32_t emu_k2_shape_stats(unsigned long *out, int reset) {
    if (out) memcpy(out, g_emu_k2_shape, sizeof(g_emu_k2_shape));
    if (reset) memset(g_emu_k2_shape, 0, sizeof(g_emu_k2_shape));
    return K2S_N;
}

extern "C" void emu_set_tie_order(int mode) { g_tie_order = mode; }
extern "C" void emu_tie_stats(unsigned long *out, int reset) {
    out[0] = g_emu_tie_stats[0]; out[1] = g_emu_tie_stats[1];
    if (reset) g_emu_tie_stats[0] = g_emu_tie_stats[1] = 0;
}
static void cta_entry(void *a) {
    CtaArgs *w = (CtaArgs *) a;
    if (g_tie_order) unc_k2_cta_main<true, true>(*w->ix, *w->p, *w->B, *w->W, w->sh);             // k2_map_exact
    else if (w->B->flags_in) unc_k2_cta_main<false, true>(*w->ix, *w->p, *w->B, *w->W, w->sh);      // k2_map_ord
    else unc_k2_cta_main<false, false>(*w->ix, *w->p, *w->B, *w->W, w->sh);                         // k2_map
}

// events (optional, n_reads x stride) / normed (optional) are filled like unc_events_batch.
static int emu_map_batch_impl(void *pidx, const unc_params *prm, const unc_read_desc *reads, uint32_t n_reads,
                  const void *samples, unc_paf_rec *out, uint32_t stride, float *events_out, float *normed_out,
                  uint32_t *n_events_out, float *mel_out, int run_k2, uint32_t max_blocks, int n_warps,
                  const uint32_t *flags_in, uint32_t *flags_out, uint32_t *cand_out = nullptr) {
    EmuIndex *e = (EmuIndex *) pidx;
    std::string err;
    if (unc_check_params(*prm, err)) { fprintf(stderr, "%s\n", err.c_str()); return UNC_E_ARG; }
    DevParams dp = unc_make_dev_params(*prm, e->h);
    u32 max_n = 0;
    for (u32 i = 0; i < n_reads; i++) if (reads[i].n_samples > max_n) max_n = reads[i].n_samples;
    if (stride < max_n) stride = max_n;
    std::vector<DevReadDesc> rd(n_reads);
    for (u32 i = 0; i < n_reads; i++) {
        rd[i].offset = reads[i].offset; rd[i].n_samples = reads[i].n_samples; rd[i].dtype = reads[i].dtype;
        rd[i].cal_range = reads[i].cal_range; rd[i].cal_offset = reads[i].cal_offset; rd[i].cal_digit = reads[i].cal_digit;
        rd[i].pad = 0;
    }
    std::vector<float> events((size_t) n_reads * stride + 1), normed((size_t) n_reads * stride + 1);
    std::vector<u32> n_events(n_reads);
    std::vector<float> scale(n_reads), shift(n_reads), mel(n_reads);
    std::vector<u64> seq_off(e->h.offsets.begin(), e->h.offsets.end());
    DevBatch B;
    B.samples = samples; B.reads = rd.data(); B.n_reads = n_reads;
    B.events = events.data(); B.normed = normed.data(); B.ev_stride = stride;
    B.n_events = n_events.data(); B.scale = scale.data(); B.shift = shift.data(); B.mean_event_len = mel.data();
    u32 queue = 0;
    B.queue = &queue; B.out = (DevRec *) out; B.dbg = nullptr;
    B.seq_offsets = seq_off.data(); B.seq_lens = e->h.lens.data(); B.n_seqs = (u32) e->h.names.size();
    B.l_pac = (u64) e->h.l_pac;
    B.flags_in = flags_in; B.flags_out = flags_out;
    u64 total_bytes = 0;
    for (u32 i = 0; i < n_reads; i++) {
        u64 e = (reads[i].offset + reads[i].n_samples) * (reads[i].dtype ? 2 : 4);
        if (e > total_bytes) total_bytes = e;
    }
    B.samples_bytes = total_bytes;
    u32 k1_queue = 0;
    std::vector<u32> k1_flags(n_reads);
    memset(g_k1_stats, 0, sizeof(g_k1_stats));
    B.k1_queue = &k1_queue; B.k1_flags = k1_flags.data(); B.k1_stats = g_k1_stats;
    if (getenv("UNC_EMU_K1_SERIAL")) {
        for (u32 r = 0; r < n_reads; r++) unc_k1_read(B, dp, r);
    } else {
        // the event-detection kernel (warp per read), then the serial redo of flagged reads and the
        // normaliser statistics, exactly as launch_k1() in unc_abi.cu orders them
        const int k1_warps = getenv("UNC_EMU_K1_WARPS") ? atoi(getenv("UNC_EMU_K1_WARPS")) : 2;
        K1WarpSmem *ksm = (K1WarpSmem *) aligned_alloc(16, sizeof(K1WarpSmem) * k1_warps);
        memset(ksm, 0, sizeof(K1WarpSmem) * k1_warps);
        K1Args ka = {&B, &dp, ksm};
        emu_run_cta(k1_entry, &ka, 32 * k1_warps);
        free(ksm);
        for (u32 r = 0; r < n_reads; r++) if (k1_flags[r]) unc_k1_read(B, dp, r);
        for (u32 r = 0; r < n_reads; r++) if (!k1_flags[r]) unc_k1_norm_read(B, dp, r);
    }
    if (events_out) memcpy(events_out, events.data(), (size_t) n_reads * stride * 4);
    if (normed_out) memcpy(normed_out, normed.data(), (size_t) n_reads * stride * 4);
    if (n_events_out) memcpy(n_events_out, n_events.data(), n_reads * 4);
    if (mel_out) memcpy(mel_out, mel.data(), n_reads * 4);
    if (cand_out) {                                  // k_event0_cands of unc_abi.cu
        memset(cand_out, 0, (size_t) n_reads * 128);
        for (u32 r = 0; r < n_reads; r++)
            for (u32 k = 0; k < UNC_NKMER; k++)
                if (unc_event0_cand(e->ix, dp, B, r, k)) cand_out[(size_t) r * 32 + (k >> 5)] |= 1u << (k & 31u);
    }
    if (!run_k2) return 0;

    u32 maxp = dp.max_paths;
    const size_t nchmax = (maxp + 31) / 32;
    std::vector<uint4> paths((size_t) 2 * (nchmax * 160 + maxp) * 2), ckey((size_t) 2 * maxp), cks(nchmax * 160), elist(nchmax * 32), wlist(nchmax * 160);
    std::vector<uint2> hist((size_t) 24 * (nchmax * 160 + maxp));
    std::vector<u32> order((size_t) 2 * maxp);
    std::vector<uint4> clu((size_t) max_blocks * 32 * 2), dir(max_blocks + 1);
    const u32 rl_cap = UNC_RL_CAP;
    std::vector<uint2> rlist(2 * rl_cap);
    DevWork W;
    W.paths = paths.data(); W.hist = hist.data(); W.wlist = wlist.data(); W.ckey = ckey.data(); W.cks = cks.data(); W.elist = elist.data(); W.order = order.data(); W.rlist = rlist.data();
    W.clu = clu.data(); W.dir = dir.data();
    W.max_blocks = max_blocks; W.rl_cap = rl_cap;
    K2Shared *sh = (K2Shared *) calloc(1, K2_SMEM_BYTES(maxp));
    CtaArgs a = {&e->ix, &dp, &B, &W, sh};
    emu_run_cta(cta_entry, &a, 32 * (n_warps > 0 ? n_warps : 8));   // one persistent CTA maps the whole batch
    free(sh);
    return 0;
}

int emu_map_batch(void *pidx, const unc_params *prm, const unc_read_desc *reads, uint32_t n_reads,
                  const void *samples, unc_paf_rec *out, uint32_t stride, float *events_out, float *normed_out,
                  uint32_t *n_events_out, float *mel_out, int run_k2, uint32_t max_blocks, int n_warps) {
    return emu_map_batch_impl(pidx, prm, reads, n_reads, samples, out, stride, events_out, normed_out, n_events_out, mel_out,
                              run_k2, max_blocks, n_warps, nullptr, nullptr);
}

// unc_map_batch_ordered with the emulated kernels behind the product's own host logic (unc_ordered_logic.hpp)
int emu_map_batch_ordered(void *pidx, const unc_params *prm, const unc_read_desc *reads, uint32_t n_reads,
                          const void *samples, uint32_t *carry, unc_paf_rec *out, uint32_t *n_remapped, uint32_t *n_rounds,
                          uint32_t max_blocks, int n_warps) {
    std::vector<unc_read_desc> sub;
    auto map_subset = [&](const uint32_t *ids, uint32_t m, const uint32_t *fi, uint32_t *fo, unc_paf_rec *recs, uint32_t *cand) -> int {
        sub.resize(m);
        for (uint32_t j = 0; j < m; j++) sub[j] = reads[ids[j]];
        int rc = emu_map_batch_impl(pidx, prm, sub.data(), m, samples, recs, 0, nullptr, nullptr, nullptr, nullptr, 1, max_blocks,
                                    n_warps, fi, fo, cand);
        if (rc) return rc;
        for (uint32_t j = 0; j < m; j++) if (recs[j].status != 0) return UNC_E_OVERFLOW;
        return UNC_OK;
    };
    return unc_ordered_map(n_reads, prm->max_paths, carry, out, n_remapped, n_rounds, map_subset);
}

// unc_pdq_sort (unc_pdqsort.cuh) on its own: keys = n x (fm_start, fm_end, seed_prob bits, tag); returns 0 if the
// scratch stack sufficed
unsigned long emu_pdq_heapsorts(void) { return g_emu_pdq_heapsorts; }
void emu_pdq_heapsort(uint4 *keys, uint32_t n) { pq_heapsort(keys, 0, (int) n); }
int emu_pdq_min_bad(int reset) { int v = g_emu_pdq_min_bad; if (reset) g_emu_pdq_min_bad = 1 << 30; return v; }
int emu_pdq_sort(uint4 *keys, uint32_t n, uint32_t stack_cap) {
    std::vector<uint4> stack(stack_cap ? stack_cap : 1);
    return unc_pdq_sort(keys, n, stack.data(), stack_cap) ? 0 : 1;
}

void emu_match_probs(void *pidx, float event, float *out) {
    EmuIndex *e = (EmuIndex *) pidx;
    for (u32 k = 0; k < 1024; k++) out[k] = unc_match_prob(event, e->h.lv_mean[k], e->h.lv_var2[k], e->h.lognorm[k]);
}

uint64_t emu_sa(void *pidx, uint64_t row) {
    EmuIndex *e = (EmuIndex *) pidx;
    u32 a = 0, b = 0;
    return unc_sa(e->ix, (u32) row, &a, &b);
}

// unc_fm_step of unc_abi.cu on the emulator's occ2 blocks: ns / ne hold 4 entries per query
void emu_fm_step(void *pidx, uint32_t n, const uint64_t *st, const uint64_t *en, const uint8_t *want, uint64_t *ns,
                 uint64_t *ne, uint8_t *valid) {
    EmuIndex *e = (EmuIndex *) pidx;
    for (uint32_t i = 0; i < n; i++) {
        u32 s[4], t[4], nb = 0;
        valid[i] = (uint8_t) unc_occ2_neighbors(e->ix, (u32) st[i], (u32) en[i], want[i], s, t, &nb);
        for (u32 b = 0; b < 4; b++) { ns[(size_t) i * 4 + b] = s[b]; ne[(size_t) i * 4 + b] = t[b]; }
    }
}


// ---------------------------------------------------------------- streaming path under the emulator
struct EmuStream {
    EmuIndex *e;
    unc_params prm;
    DevParams dp;
    u32 n_channels, max_chunk_len, max_chunks, ev_stride, max_blocks;
    std::vector<HostChan> ch;
    std::vector<DevChanSig> sig;
    std::vector<float> norm_sig;
    std::vector<DevMapState> map;
    std::vector<uint4> paths, ckey, cks, elist, wlist, clu, dir;
    std::vector<uint2> hist, rlist;
    std::vector<u32> order;
    DevWork W;
    DevWorkStrides S;
    std::vector<std::vector<float>> pushed;   // per channel: every event mean unc_stream_chunk emitted, in order
};
struct StreamCtaArgs { const DevIndex *ix; const DevParams *p; const DevBatch *B; const DevWork *W; const DevWorkStrides *S; K2Shared *sh; };
static void stream_cta_entry(void *a) {
    StreamCtaArgs *w = (StreamCtaArgs *) a;
    if (g_tie_order) unc_k2_cta_main_stream<true>(*w->ix, *w->p, *w->B, *w->W, *w->S, w->sh);
    else unc_k2_cta_main_stream<false>(*w->ix, *w->p, *w->B, *w->W, *w->S, w->sh);
}

void *emu_stream_create(void *pidx, const unc_params *prm, uint32_t n_channels, uint32_t max_chunk_len,
                        uint32_t max_chunks, uint32_t max_blocks) {
    EmuStream *T = new EmuStream();
    T->e = (EmuIndex *) pidx; T->prm = *prm; T->dp = unc_make_dev_params(*prm, T->e->h);
    T->n_channels = n_channels; T->max_chunk_len = max_chunk_len; T->max_chunks = max_chunks;
    T->ev_stride = (max_chunk_len + 3u) & ~3u; T->max_blocks = max_blocks;
    T->ch.resize(n_channels);
    T->pushed.resize(n_channels);
    T->sig.resize(n_channels); memset(T->sig.data(), 0, n_channels * sizeof(DevChanSig));
    T->norm_sig.assign((size_t) n_channels * UNC_NORM_LEN, 0.0f);
    T->map.resize(n_channels); memset(T->map.data(), 0, n_channels * sizeof(DevMapState));
    const size_t maxp = prm->max_paths, nchmax = (maxp + 31) / 32, n = n_channels;
    DevWorkStrides &S = T->S;
    S.paths = 2 * (nchmax * 160 + maxp) * 2; S.hist = 24 * (nchmax * 160 + maxp); S.ckey = 2 * maxp;
    S.cks = nchmax * 160; S.elist = nchmax * 32; S.order = 2 * maxp;
    const u32 rl_cap = UNC_RL_CAP;
    S.rlist = 2 * rl_cap; S.clu = (size_t) max_blocks * 32 * 2; S.dir = (size_t) max_blocks + 1;
    T->paths.resize(n * S.paths); T->hist.resize(n * S.hist); T->ckey.resize(n * S.ckey); T->cks.resize(n * S.cks);
    T->wlist.resize(n * S.cks); T->elist.resize(n * S.elist); T->order.resize(n * S.order); T->rlist.resize(n * S.rlist);
    T->clu.resize(n * S.clu); T->dir.resize(n * S.dir);
    DevWork &W = T->W;
    W.paths = T->paths.data(); W.hist = T->hist.data(); W.wlist = T->wlist.data(); W.ckey = T->ckey.data(); W.cks = T->cks.data();
    W.elist = T->elist.data(); W.order = T->order.data(); W.rlist = T->rlist.data(); W.clu = T->clu.data(); W.dir = T->dir.data();
    W.max_blocks = max_blocks; W.rl_cap = rl_cap;
    return T;
}
void emu_stream_free(void *p) { delete (EmuStream *) p; }

// Mirrors unc_stream_step (unc_stream_host.inl): same bookkeeping (unc_stream_logic.hpp), the two device
// routines run on the CPU: unc_stream_chunk per item, then the mapper CTA under the emulator.
int emu_stream_step(void *pst, const unc_chunk_desc *chunks, uint32_t n, const void *samples, unc_stream_result *out,
                    int n_warps) {
    EmuStream *T = (EmuStream *) pst;
    const float bp_per_samp = T->prm.bp_per_sec / T->prm.sample_rate;
    std::vector<int> item_of(n, -1);
    std::vector<DevReadDesc> rd;
    std::vector<u32> chan, isnew;
    u64 total_bytes = 0;
    for (u32 i = 0; i < n; i++) {
        const unc_chunk_desc &c = chunks[i];
        if (c.channel >= T->n_channels || c.n_samples > T->max_chunk_len) return UNC_E_ARG;
        if (!stream_admit(T->ch[c.channel], c, T->max_chunks)) continue;
        DevReadDesc d;
        d.offset = c.offset; d.n_samples = c.n_samples; d.dtype = c.dtype;
        d.cal_range = c.cal_range; d.cal_offset = c.cal_offset; d.cal_digit = c.cal_digit; d.pad = 0;
        total_bytes = std::max<u64>(total_bytes, (c.offset + c.n_samples) * (c.dtype ? 2 : 4));
        item_of[i] = (int) rd.size();
        rd.push_back(d); chan.push_back(c.channel); isnew.push_back(c.new_read ? 1u : 0u);
    }
    const u32 m = (u32) rd.size();
    std::vector<DevRec> recs(m);
    std::vector<u32> tot(m);
    if (m) {
        std::vector<float> events((size_t) m * T->ev_stride + 1), scale(m), shift(m), mel(m);
        std::vector<u32> n_events(m), flags(m);
        std::vector<u64> seq_off(T->e->h.offsets.begin(), T->e->h.offsets.end());
        u32 queue = 0, k1q = 0;
        DevBatch B;
        memset(&B, 0, sizeof(B));
        B.samples = samples; B.samples_bytes = total_bytes; B.reads = rd.data(); B.n_reads = m;
        B.events = events.data(); B.normed = nullptr; B.ev_stride = T->ev_stride; B.n_events = n_events.data();
        B.scale = scale.data(); B.shift = shift.data(); B.mean_event_len = mel.data();
        B.queue = &queue; B.k1_queue = &k1q; B.k1_flags = flags.data(); B.k1_stats = nullptr;
        B.out = recs.data(); B.dbg = nullptr;
        B.seq_offsets = seq_off.data(); B.seq_lens = T->e->h.lens.data(); B.n_seqs = (u32) T->e->h.names.size();
        B.l_pac = (u64) T->e->h.l_pac;
        B.mstate = T->map.data(); B.chan = chan.data();
        DevStream S;
        S.sig = T->sig.data(); S.norm_sig = T->norm_sig.data(); S.map = T->map.data();
        for (u32 r = 0; r < m; r++) {
            unc_stream_chunk(B, T->dp, S, r, isnew[r]);
            tot[r] = T->sig[chan[r]].evdt.total_events;
            const float *ev = events.data() + (size_t) r * T->ev_stride;
            T->pushed[chan[r]].insert(T->pushed[chan[r]].end(), ev, ev + n_events[r]);
        }
        K2Shared *sh = (K2Shared *) calloc(1, K2_SMEM_BYTES(T->dp.max_paths));
        StreamCtaArgs a = {&T->e->ix, &T->dp, &B, &T->W, &T->S, sh};
        emu_run_cta(stream_cta_entry, &a, 32 * (n_warps > 0 ? n_warps : 8));
        free(sh);
    }
    for (u32 i = 0; i < n; i++) {
        HostChan &h = T->ch[chunks[i].channel];
        if (item_of[i] >= 0) {
            unc_paf_rec r;
            memcpy(&r, &recs[item_of[i]], sizeof(r));
            stream_settle(h, r, tot[item_of[i]], T->prm.max_events, T->max_chunks);
        }
        stream_result(h, bp_per_samp, &out[i]);
    }
    return 0;
}

// The channel's streaming normaliser as the device left it: state = (mean, varsum, n, wr) of DevChanSig.norm, ring (optional,
// UNC_NORM_LEN floats) = its slice of DevStream::norm_sig.  Returns the number of event means the channel has pushed so far;
// pushed (optional, cap floats) receives the first min(cap, that number) of them.
uint64_t emu_stream_norm_state(void *pst, uint32_t channel, double *state, float *ring, float *pushed, uint64_t cap) {
    EmuStream *T = (EmuStream *) pst;
    const DevRing &z = T->sig[channel].norm;
    state[0] = z.mean; state[1] = z.varsum; state[2] = z.n; state[3] = z.wr;
    if (ring) memcpy(ring, T->norm_sig.data() + (size_t) channel * UNC_NORM_LEN, UNC_NORM_LEN * sizeof(float));
    const std::vector<float> &p = T->pushed[channel];
    if (pushed) memcpy(pushed, p.data(), std::min<uint64_t>(cap, p.size()) * sizeof(float));
    return p.size();
}

// ---- self_align: the device functions of unc_selfalign.cuh, one "thread" after the other, around the same
// host steps as unc_self_align (uncalled_b200/csrc/unc_selfalign_host.inl)
int emu_glibc_rand(unsigned seed, uint32_t n, int32_t *out) {
    GlibcRand g(seed);
    for (uint32_t i = 0; i < n; i++) out[i] = g.next();
    return 0;
}

int emu_self_align(const char *prefix, uint32_t sample_dist, uint64_t *n_paths, uint64_t **offsets, uint64_t **values) {
    HostIndex h;
    std::vector<char> pac;
    if (!hix_load_fm(h, prefix) || !hix_read_file(std::string(prefix) + ".pac", pac)) return -1;
    pac.resize(pac.size() + 16, 0);
    std::vector<u32> pos, lim;
    unc_selfalign_sample(h.lens, sample_dist, pos, lim);
    const size_t n = pos.size();
    DevIndex ix{};
    ix.bwt = (const uint4 *) h.bwt.data();
    ix.primary = (u32) h.primary; ix.seq_len = (u32) h.seq_len;
    for (int i = 0; i < 5; i++) ix.L2[i] = (u32) h.L2[i];
    std::vector<u32> count(n), stage((size_t) UNC_SA_STAGE * n);
    DevSelfAlign A{};
    A.pac = (const u8 *) pac.data(); A.pos = pos.data(); A.lim = lim.data(); A.n = (u32) n;
    A.count = count.data(); A.stage = stage.data();
    for (size_t i = 0; i < n; i++) unc_selfalign_count(ix, A, (u32) i);
    uint64_t *off = (uint64_t *) malloc((n + 1) * 8);
    off[0] = 0;
    for (size_t i = 0; i < n; i++) off[i + 1] = off[i] + count[i];
    uint64_t *val = (uint64_t *) malloc((off[n] ? off[n] : 1) * 8);
    A.offsets = off; A.values = val;
    for (size_t i = 0; i < n; i++) unc_selfalign_write(ix, A, (u32) i);
    *n_paths = n; *offsets = off; *values = val;
    return 0;
}
void emu_free(void *p) { free(p); }

}  // extern "C"
