// tests/emul/emul_dtw_align.cpp -- the signal-to-span aligner's device stages (unc_k1.cuh for (a), unc_dtw_align.cuh for
// (b)-(e)) on the CPU under the warp emulator, in the order unc_dtw_align_batch launches them.  Test vehicle only.
#include "unc_device.cuh"   // UNC_EMUL is defined on the command line
#include "unc_k1.cuh"
#include "unc_stream.cuh"
#include "unc_dtw_align.cuh"
#include "../../include/unc_b200.h"
#include "unc_host_index.hpp"
#include "unc_host_params.hpp"

thread_local WarpEmu *g_warp = nullptr;

struct K1Args { const DevBatch *B; const DevParams *p; K1WarpSmem *sm; };
static void k1_entry(void *a) {
    K1Args *w = (K1Args *) a;
    unc_k1_warp_main(*w->B, *w->p, w->sm + (c_tid() >> 5));
}

extern "C" {

// n reads of f32 samples (reads[i]: offset, n_samples) against their spans q[i] (pac_st = .pac coordinate of the first
// base).  events_in != NULL: stage (a) is skipped and reads[i].n_samples event means are taken from events_in at
// reads[i].offset instead.  Out per read: n_events, n_kept, tgt (2 floats), the kept normalised means (row i of `means`,
// stride max n_samples) and the k-mers (at the k-mer offset, in query order), and the verdict.
int emu_dtw_align_stages(uint32_t n, const unc_read_desc *reads, const float *samples, const float *events_in,
                         const uint8_t *pac, const uint64_t *pac_st, const uint32_t *n_kmers, const uint32_t *fwd,
                         const float *model_means_stdvs, uint32_t stride, uint32_t *n_events, uint32_t *n_kept, float *tgt,
                         float *means, uint16_t *kmers, int32_t *verdict, int k1_warps) {
    unc_params prm;
    unc_fill_default_params(&prm);
    HostIndex h;
    DevParams dp = unc_make_dev_params(prm, h);
    std::vector<DevReadDesc> rd(n);
    u64 hi = 0;
    for (u32 i = 0; i < n; i++) {
        rd[i].offset = reads[i].offset; rd[i].n_samples = reads[i].n_samples; rd[i].dtype = 0;
        rd[i].cal_range = 1; rd[i].cal_offset = 0; rd[i].cal_digit = 1; rd[i].pad = 0;
        hi = std::max<u64>(hi, reads[i].offset + reads[i].n_samples);
    }
    std::vector<u32> mel(n), scale(n), shift(n), flags(n);
    if (events_in) {
        for (u32 i = 0; i < n; i++) {
            memcpy(means + (size_t) i * stride, events_in + reads[i].offset, (size_t) reads[i].n_samples * 4);
            n_events[i] = reads[i].n_samples;
        }
    } else {
        DevBatch B;
        memset(&B, 0, sizeof(B));
        B.samples = samples; B.samples_bytes = hi * 4; B.reads = rd.data(); B.n_reads = n;
        B.events = means; B.ev_stride = stride; B.n_events = n_events;
        B.mean_event_len = (float *) mel.data(); B.scale = (float *) scale.data(); B.shift = (float *) shift.data();
        u32 k1_queue = 0;
        B.k1_queue = &k1_queue; B.k1_flags = flags.data();
        K1WarpSmem *ksm = (K1WarpSmem *) aligned_alloc(16, sizeof(K1WarpSmem) * k1_warps);
        memset(ksm, 0, sizeof(K1WarpSmem) * k1_warps);
        K1Args ka = {&B, &dp, ksm};
        emu_run_cta(k1_entry, &ka, 32 * k1_warps);
        free(ksm);
        for (u32 r = 0; r < n; r++) if (flags[r]) unc_k1_read(B, dp, r);         // k1_fallback
    }
    std::vector<DevAlignRead> q(n);
    std::vector<float> lv(1024);
    for (u32 k = 0; k < 1024; k++) lv[k] = model_means_stdvs[2 * k];
    u64 koff = 0;
    for (u32 i = 0; i < n; i++) { q[i].kmer_off = koff; q[i].pac_st = pac_st[i]; q[i].n_kmers = n_kmers[i]; q[i].fwd = fwd[i]; koff += n_kmers[i]; }
    DevAlign A;
    A.events = means; A.ev_stride = stride; A.n_events = n_events; A.n_kept = n_kept; A.q = q.data(); A.n = n;
    A.pac = pac; A.lv_mean = lv.data(); A.kmers = kmers; A.tgt = tgt;
    for (u32 r = 0; r < n; r++) unc_align_mask(A, r);                                       // (b)
    for (u32 r = 0; r < n; r++) for (u32 i = 0; i < q[r].n_kmers; i++) kmers[q[r].kmer_off + i] = unc_align_kmer(A, q[r], i);   // (c)
    for (u32 r = 0; r < n; r++) unc_align_target(A, r);                                     // (d)
    for (u32 r = 0; r < n; r++) unc_align_norm(A, r);                                       // (e)
    for (u32 r = 0; r < n; r++) verdict[r] = unc_align_verdict(n_kept[r]);
    return 0;
}

}  // extern "C"
