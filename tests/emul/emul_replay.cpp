// tests/emul/emul_replay.cpp -- the device replay of `map-ord` (uncalled_b200/csrc/unc_replay.cuh) on the CPU under the
// warp emulator, around the same host steps as unc_stream_replay (uncalled_b200/csrc/unc_replay_host.inl).  It is the
// emulator harness of emul_main.cpp (index, streams, unc_stream_step's counterpart) plus emu_stream_replay, built as
// a library of its own so that the host-stepped loop and the replay run on the same emulated streams.
#include <map>

#include "emul_main.cpp"
#include "unc_replay.cuh"

// per stream: the steps its replays have taken on each channel (unc_stream's `steps`)
static std::map<void *, std::vector<u64>> g_steps;

extern "C" void emu_replay_stream_free(void *p) {
    g_steps.erase(p);
    emu_stream_free(p);
}

struct ReplayCtaArgs { const DevIndex *ix; const DevParams *p; const DevBatch *B; const DevWork *W; const DevWorkStrides *S;
                       const DevStream *St; const DevReplay *R; K2Shared *sh; u32 *ctl; };
static void replay_cta_entry(void *a) {
    ReplayCtaArgs *w = (ReplayCtaArgs *) a;
    if (g_tie_order) unc_replay_cta_main<true>(*w->ix, *w->p, *w->B, *w->W, *w->S, *w->St, *w->R, w->sh, w->ctl);
    else unc_replay_cta_main<false>(*w->ix, *w->p, *w->B, *w->W, *w->S, *w->St, *w->R, w->sh, w->ctl);
}

// Mirrors unc_stream_replay (unc_replay_host.inl): the same grouping and channel order, and the replay CTA body of
// unc_replay.cuh run as ONE CTA under the emulator (it takes the channels one after the other).  Returns 0 or
// UNC_E_OVERFLOW; a bad descriptor returns UNC_E_ARG with nothing changed.
extern "C" int emu_stream_replay(void *pst, const unc_replay_read *reads, uint32_t n, const void *samples, unc_replay_result *out,
                      int n_warps) {
    EmuStream *T = (EmuStream *) pst;
    if (n == 0) return 0;
    const u32 nch = T->n_channels, dtype = reads[0].dtype;
    std::vector<u32> cnt(nch, 0);
    std::vector<u64> total(nch, 0);
    u64 hi = 0;
    for (u32 i = 0; i < n; i++) {
        const unc_replay_read &r = reads[i];
        if (r.channel >= nch || r.n_samples == 0 || r.dtype != dtype || r.dtype > 1) return UNC_E_ARG;
        hi = std::max<u64>(hi, r.offset + r.n_samples);
        cnt[r.channel]++; total[r.channel] += r.n_samples;
    }
    std::vector<u64> &steps = g_steps[T];
    if (steps.size() != nch) steps.assign(nch, 0);
    std::vector<u32> first(nch, 0);
    for (u32 c = 1; c < nch; c++) first[c] = first[c - 1] + cnt[c - 1];
    std::vector<unc_replay_read> grouped(n);
    std::vector<u32> idx(n), fill(first);
    for (u32 i = 0; i < n; i++) { const u32 j = fill[reads[i].channel]++; grouped[j] = reads[i]; idx[j] = i; }
    std::vector<u32> chans, ch_first, ch_count, iota(nch);
    for (u32 c = 0; c < nch; c++) { iota[c] = c; if (cnt[c]) chans.push_back(c); }
    std::stable_sort(chans.begin(), chans.end(), [&](u32 a, u32 b) { return total[a] > total[b]; });
    for (u32 c : chans) { ch_first.push_back(first[c]); ch_count.push_back(cnt[c]); }
    std::vector<float> events((size_t) nch * T->ev_stride + 1), scale(nch), shift(nch), mel(nch);
    std::vector<u32> n_events(nch), flags(nch);
    std::vector<DevReadDesc> desc(nch);
    std::vector<DevRec> recs(nch);
    std::vector<u64> seq_off(T->e->h.offsets.begin(), T->e->h.offsets.end());
    u32 queue = 0, k1q = 0, ctr[4] = {0, 0, 0, 0}, ctl[2] = {0, 0};
    DevBatch B;
    memset(&B, 0, sizeof(B));
    B.samples = samples; B.samples_bytes = hi * (dtype ? 2 : 4); B.reads = desc.data(); B.n_reads = nch;
    B.events = events.data(); B.normed = nullptr; B.ev_stride = T->ev_stride; B.n_events = n_events.data();
    B.scale = scale.data(); B.shift = shift.data(); B.mean_event_len = mel.data();
    B.queue = &queue; B.k1_queue = &k1q; B.k1_flags = flags.data(); B.k1_stats = nullptr;
    B.out = recs.data(); B.dbg = nullptr;
    B.seq_offsets = seq_off.data(); B.seq_lens = T->e->h.lens.data(); B.n_seqs = (u32) T->e->h.names.size();
    B.l_pac = (u64) T->e->h.l_pac;
    B.mstate = T->map.data(); B.chan = iota.data();
    DevStream St;
    St.sig = T->sig.data(); St.norm_sig = T->norm_sig.data(); St.map = T->map.data();
    DevReplay R;
    R.reads = grouped.data(); R.read_idx = idx.data(); R.chans = chans.data(); R.first = ch_first.data(); R.count = ch_count.data();
    R.n_chans = (u32) chans.size(); R.chunk_len = T->max_chunk_len; R.max_chunks = T->max_chunks; R.max_events = T->prm.max_events;
    R.bp_per_samp = T->prm.bp_per_sec / T->prm.sample_rate;
    R.hc = T->ch.data(); R.step = steps.data(); R.desc = desc.data(); R.out = out;
    R.n_out = &ctr[0]; R.queue = &ctr[1]; R.overflow = &ctr[2];
    K2Shared *sh = (K2Shared *) calloc(1, K2_SMEM_BYTES(T->dp.max_paths));
    ReplayCtaArgs a = {&T->e->ix, &T->dp, &B, &T->W, &T->S, &St, &R, sh, ctl};
    emu_run_cta(replay_cta_entry, &a, 32 * (n_warps > 0 ? n_warps : 8));
    free(sh);
    if (ctr[0] != n) return UNC_E_CUDA;
    std::sort(out, out + n, [&](const unc_replay_result &x, const unc_replay_result &y) {
        if (x.step != y.step) return x.step < y.step;
        if (x.kind != y.kind) return x.kind < y.kind;
        return reads[x.read].channel < reads[y.read].channel;
    });
    return ctr[2] ? UNC_E_OVERFLOW : 0;
}

