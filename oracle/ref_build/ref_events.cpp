// oracle/_ref/libref_events.so: the reference's own EventDetector::get_events, EventProfiler (add_event / anno_event /
// get_full_mask), offline Normalizer and PoreModel::match_prob, for the checkers of `events`.
//
// TEST INFRASTRUCTURE ONLY.  Built by oracle/events.mk where the reference tree lies under /root/reference, against
// oracle/_ref/libuncalled_ref.so (which holds the reference's own compiled sources).  Nothing of the reference is copied
// here; this file only calls it.  (ref_shim.cpp's ref_get_events drops each event's stdv.)
#include <cmath>
#include <cstdint>
#include <vector>

#include "event_profiler.hpp"
#include "normalizer.hpp"
#include "model_r94.inl"
#include "pore_model.hpp"

#define EXPORT __attribute__((visibility("default")))

extern "C" {

// EventDetector().get_events(raw): every output array needs room for n entries
EXPORT uint32_t ref_get_events_full(const float *raw, uint32_t n, float *means, float *stdvs, uint32_t *starts,
                                    uint32_t *lens, float *mean_event_len) {
    EventDetector ed;
    std::vector<float> sig(raw, raw + n);
    std::vector<Event> ev = ed.get_events(sig);
    for (size_t i = 0; i < ev.size(); i++) {
        means[i] = ev[i].mean; stdvs[i] = ev[i].stdv; starts[i] = ev[i].start; lens[i] = ev[i].length;
    }
    if (mean_event_len) *mean_event_len = ed.mean_event_len();
    return (uint32_t) ev.size();
}

// EventProfiler() over n events with these means: get_full_mask, and, from a second pass of add_event, anno_event()'s
// win_mean / win_stdv for every event that becomes next_evt_ (NaN for the others)
EXPORT void ref_profile_events(const float *means, uint32_t n, float *win_mean, float *win_stdv, uint8_t *mask) {
    std::vector<Event> ev(n);
    for (uint32_t i = 0; i < n; i++) { ev[i].mean = means[i]; ev[i].stdv = 0; ev[i].start = i; ev[i].length = 1; }
    EventProfiler ep;
    std::vector<bool> m = ep.get_full_mask(ev);
    for (uint32_t i = 0; i < n; i++) { mask[i] = m[i] ? 1 : 0; win_mean[i] = NAN; win_stdv[i] = NAN; }
    ep.reset();
    for (uint32_t i = 0; i < n; i++) {
        ep.add_event(ev[i]);
        if (!ep.is_full()) continue;
        AnnoEvent a = ep.anno_event();
        win_mean[a.evt.start] = a.win_mean;
        win_stdv[a.evt.start] = a.win_stdv;
    }
}

// Normalizer(model mean, model stdv) + set_signal + pop() for n > 0 means, as Mapper::map_read drives it, with the
// model the mapper holds (pmodel_r94_complement, src/mapper.cpp:57).  The scale and shift pop() applies
// (Normalizer::at, src/normalizer.cpp:114-118) are not reachable from outside the class; they are checked through
// the normalised means.
EXPORT void ref_normalize_full(const float *events, uint32_t n, float *out) {
    const PoreModel<KmerLen::k5> &model = pmodel_r94_complement;
    Normalizer norm(model.get_means_mean(), model.get_means_stdv());
    std::vector<float> ev(events, events + n);
    norm.set_signal(ev);
    for (uint32_t i = 0; i < n; i++) out[i] = norm.pop();
}

// PoreModel::match_prob of the mapper's model (pmodel_r94_complement)
EXPORT float ref_match_prob_c(float samp, uint16_t kmer) { return pmodel_r94_complement.match_prob(samp, kmer); }

}  // extern "C"
