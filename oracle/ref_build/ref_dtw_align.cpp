// oracle/_ref/libref_dtw_align.so: the loop body of the reference's dtw_test driver (src/dtw_test.cpp:94-175) for one
// signal and one query, through the reference's own EventDetector, EventProfiler::get_full_mask, BwaIndex::get_kmers after
// load_pacseq (+ kmers_revcomp), Normalizer and DTWr94d.
//
// TEST INFRASTRUCTURE ONLY.  Built by oracle/dtw_align.mk where the reference tree lies under /root/reference, against
// oracle/_ref/libuncalled_ref.so (which holds the reference's own compiled sources).  Nothing of the reference is copied
// here; this file only calls it, with dtw_test.cpp's own includes and arithmetic.  dtw_test.cpp itself is not compiled:
// its Fast5Reader needs libhdf5, so the signal is passed in.
#include <iostream>
#include <math.h>
#include <unordered_map>
#include <cstdint>
#include <string>

#include "event_profiler.hpp"
#include "normalizer.hpp"
#include "model_r94.inl"
#include "pore_model.hpp"
// the index's bns_ / pacseq_ are private; only the .ann/.amb/.pac are opened (bns_restore), not the FM index
#define private public
#include "bwa_index.hpp"
#undef private
#include "dtw.hpp"

static const KmerLen KLEN_DTW = KmerLen::k5;
static BwaIndex<KLEN_DTW> *g_idx = nullptr;
static std::string g_prefix;

extern "C" {

// means: room for n; kmers_out: rf_en - rf_st - 4; path: room for both.  Returns 0 aligned, 1 skipped (more than 50 000
// means), 2 no event left after the mask (the reference's behaviour is undefined there: Normalizer::set_signal divides
// by zero).
__attribute__((visibility("default"))) int ref_dtw_align(const char *bwa_prefix, const float *sig, uint32_t n, const char *rf_name, uint64_t rf_st, uint64_t rf_en,
                  int fwd, uint32_t *n_events, uint32_t *n_kept, float *tgt, float *means, uint16_t *kmers_out, float *score,
                  float *mean_score, uint64_t *path, uint64_t *path_len) {
    if (!g_idx || g_prefix != bwa_prefix) {
        if (g_idx) { bns_destroy(g_idx->bns_); free(g_idx->pacseq_); delete g_idx; }
        g_idx = new BwaIndex<KLEN_DTW>();
        g_idx->bns_ = bns_restore(bwa_prefix);
        g_idx->load_pacseq();
        g_prefix = bwa_prefix;
    }
    BwaIndex<KLEN_DTW> &idx = *g_idx;
    auto model = pmodel_r94_template;
    DTWParams dtwp = {DTWSubSeq::NONE, 1, 1, 1};
    EventDetector evdt;
    EventProfiler evpr;
    std::vector<u16> kmers = idx.get_kmers(rf_name, rf_st, rf_en);
    if (!fwd) kmers = kmers_revcomp<KLEN_DTW>(kmers);
    float read_mean = 0;
    for (u16 k : kmers) read_mean += model.get_mean(k);
    read_mean /= kmers.size();
    float read_stdv = 0;
    for (u16 k : kmers) read_stdv += pow(model.get_mean(k) - read_mean, 2);
    read_stdv = sqrt(read_stdv / kmers.size());
    Normalizer norm(read_mean, read_stdv);
    tgt[0] = read_mean; tgt[1] = read_stdv;
    std::copy(kmers.begin(), kmers.end(), kmers_out);
    std::vector<float> signal(sig, sig + n);
    auto events = evdt.get_events(signal);
    auto mask = evpr.get_full_mask(events);
    signal.clear();
    for (u32 i = 0; i < events.size(); i++) if (mask[i]) signal.push_back(events[i].mean);
    *n_events = (uint32_t) events.size();
    *n_kept = (uint32_t) signal.size();
    if (signal.empty()) return 2;
    norm.set_signal(signal);
    signal.clear();
    while (!norm.empty()) signal.push_back(norm.pop());
    std::copy(signal.begin(), signal.end(), means);
    if (signal.size() > 50000) return 1;
    DTWr94d dtw(signal, kmers, dtwp);
    auto p = dtw.get_path();
    for (size_t i = 0; i < p.size(); i++) { path[2 * i] = p[i].first; path[2 * i + 1] = p[i].second; }
    *path_len = p.size();
    *score = dtw.score();
    *mean_score = dtw.mean_score();
    return 0;
}

}  // extern "C"
