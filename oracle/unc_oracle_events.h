/* oracle/unc_oracle_events.h -- the C restatement of `events` (test infrastructure only): libunc_oracle_events.so,
 * built by oracle/events.mk from unc_oracle_events.c over the detector and profiler of unc_oracle.c. */
#ifndef UNC_ORACLE_EVENTS_H
#define UNC_ORACLE_EVENTS_H
#include "unc_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* EventDetector::get_events (reference src/event_detector.cpp:114-127) with create_event (:296-319): every event that
 * passes min_mean / max_mean.  Each output array (any may be NULL) needs room for n entries.  Returns the number of
 * events; *mean_event_len = EventDetector::mean_event_len (:151-153). */
uint32_t orc_detect_events_full(const orc_params *p, const float *raw, uint32_t n, float *means, float *stdvs,
                                uint32_t *starts, uint32_t *lens, float *mean_event_len);

/* EventProfiler::get_full_mask (reference src/event_profiler.hpp:129-151) over n event means with the default profiler
 * (25-event window, win_stdv_min given): mask[i] as get_full_mask returns it; win_mean[i] / win_stdv[i] those of the
 * add_event call after which event i is next_evt_ (anno_event, :114-121), NaN for the events that never get there. */
void orc_profile_events(const float *means, uint32_t n, float win_stdv_min, float *win_mean, float *win_stdv,
                        uint8_t *mask);

/* orc_normalize (Normalizer::set_signal + pop, reference src/normalizer.cpp:31-44,114-129) for n > 0 means, with the
 * scale and shift of Normalizer::at in scale_shift[0..1]. */
void orc_normalize_full(const orc_model *m, const float *events, uint32_t n, float *out, float *scale_shift);

#ifdef __cplusplus
}
#endif
#endif
