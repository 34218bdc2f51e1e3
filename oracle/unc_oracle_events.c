/* oracle/unc_oracle_events.c -- the C restatement of `events` (test infrastructure only).
 *
 * unc_oracle.c is compiled into this library (included below), so that its event detector and Normalizer ring are
 * reused as they are, and unc_oracle.c itself stays unchanged; the library stands alone.  Plain C, -ffp-contract=off:
 * the reference's float / double operations in its order. */
#include "unc_oracle.c"
#include "unc_oracle_events.h"

uint32_t orc_detect_events_full(const orc_params *p, const float *raw, uint32_t n, float *means, float *stdvs,
                                uint32_t *starts, uint32_t *lens, float *mean_event_len) {
    evdt_t e;
    evdt_reset(&e, p);
    u32 ne = 0;
    for (u32 i = 0; i < n; i++) {
        if (!evdt_add_sample(&e, raw[i])) continue;
        if (means) means[ne] = e.ev_mean;
        if (stdvs) stdvs[ne] = e.ev_stdv;
        if (starts) starts[ne] = e.ev_start;
        if (lens) lens[ne] = e.ev_length;
        ne++;
    }
    if (mean_event_len) *mean_event_len = e.len_sum / e.total_events;
    return ne;
}

/* EventProfiler::add_event (reference src/event_profiler.hpp:71-104) driven by get_full_mask (:129-151).  The deque
 * events_ hands out the events in order, so next_evt_ after the k-th pop is event k. */
void orc_profile_events(const float *means, uint32_t n, float win_stdv_min, float *win_mean, float *win_stdv,
                        uint8_t *mask) {
    snorm_t w;
    snorm_init(&w, EVP_WIN, 0.0f, 1.0f);
    snorm_reset(&w);
    u32 to_mask = 0, m = 0;
    int is_full = 0;
    for (u32 i = 0; i < n; i++) {
        snorm_push(&w, means[i]);
        if (snorm_unread(&w) <= EVP_WIN / 2) continue;
        float wm = (float) w.mean;                       /* Normalizer::get_mean */
        float ws = (float) sqrt(w.varsum / w.n);         /* Normalizer::get_stdv */
        if (ws < win_stdv_min) to_mask = EVP_WIN - 1;
        else if (to_mask > 0) to_mask--;
        if (w.is_full) {
            snorm_pop(&w);
            is_full = 1;
        }
        if (is_full) {
            win_mean[m] = wm;
            win_stdv[m] = ws;
            mask[m] = to_mask == 0;
            m++;
        }
    }
    for (; m < n; m++) {
        win_mean[m] = NAN;
        win_stdv[m] = NAN;
        if (to_mask == 0) mask[m] = 1;
        else { mask[m] = 0; to_mask--; }
    }
    free(w.signal);
}

void orc_normalize_full(const orc_model *m, const float *ev, uint32_t n, float *out, float *scale_shift) {
    if (n == 0) return;
    double mean = 0;
    for (u32 i = 0; i < n; i++) mean += ev[i];
    mean /= n;
    double varsum = 0;
    for (u32 i = 0; i < n; i++) {
        double d = ev[i] - mean;
        varsum += d * d;
    }
    float scale = (float) (m->model_stdv / sqrt(varsum / n));
    float shift = (float) (m->model_mean - scale * mean);
    scale_shift[0] = scale;
    scale_shift[1] = shift;
    orc_normalize(m, ev, n, out);
}
