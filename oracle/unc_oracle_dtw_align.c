/* oracle/unc_oracle_dtw_align.c -- CPU restatement of the loop body of the reference's dtw_test driver
 * (src/dtw_test.cpp:94-175) for one signal and one query.  TEST INFRASTRUCTURE ONLY, like unc_oracle.c, whose
 * event detector (orc_detect_events) it calls: built by oracle/dtw_align.mk into libunc_oracle_dtw_align.so,
 * linked against libunc_oracle.so.  Pinned to the reference by tests/golden/dtw_align_golden.json. */
#include "unc_oracle.h"

#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

/* Normalizer(tgt_mean, tgt_stdv) + set_signal + pop() until empty (reference src/normalizer.cpp:22-44,105-129) */
void orc_normalize_to(float tgt_mean, float tgt_stdv, const float *ev, uint32_t n, float *out) {
    if (n == 0) return;
    double mean = 0;
    for (u32 i = 0; i < n; i++) mean += ev[i];
    mean /= n;
    double varsum = 0;
    for (u32 i = 0; i < n; i++) {
        double d = ev[i] - mean;
        varsum += d * d;
    }
    float scale = (float) (tgt_stdv / sqrt(varsum / n));
    float shift = (float) (tgt_mean - scale * mean);
    for (u32 i = 0; i < n; i++) {
        float prod = scale * ev[i];
        out[i] = prod + shift;
    }
}

/* BwaIndex::get_kmers over .pac bases [st, st + n_bases) (src/bwa_index.hpp:234-255, seq_to_kmers src/bp.hpp:126-146),
 * kmers_revcomp (:83-99) unless fwd.  Writes n_bases - 4 k-mers. */
void orc_span_kmers(const uint8_t *pac, uint64_t st, uint64_t n_bases, int fwd, uint16_t *out) {
    const u64 nk = n_bases - 4;
    u16 k = 0;
    for (u64 i = 0; i < n_bases; i++) {
        const u64 p = st + i;
        k = (u16) (((k << 2) & 0x3FF) | ((pac[p >> 2] >> (((3 ^ p) & 3) << 1)) & 3));
        if (i >= 4) out[i - 4] = k;
    }
    if (fwd) return;
    for (u64 i = 0; i < nk / 2; i++) { u16 t = out[i]; out[i] = out[nk - 1 - i]; out[nk - 1 - i] = t; }
    for (u64 i = 0; i < nk; i++) {
        u16 x = (u16) (out[i] ^ 0x3FF), r = 0;
        for (int b = 0; b < 5; b++) { r = (u16) ((r << 2) | (x & 3)); x >>= 2; }
        out[i] = r;
    }
}

/* EventProfiler (reference src/event_profiler.hpp:14-104, defaults src/event_profiler.cpp:4-10) with its window
 * Normalizer of length 25 (push :46-75, unread_size :131-134, get_stdv :97-99) */
#define WIN 25u
#define STDV_MIN 5.0f
typedef struct {
    float sig[WIN];
    u32 n, rd, wr, is_full;
    double mean, varsum;
    float q[WIN + 1];           /* events_: only the means are consumed */
    u32 q_head, q_size, p_is_full, to_mask;
} prof_t;

static void win_push(prof_t *e, float newevt) {
    if (e->is_full) return;
    double oldevt = e->sig[e->wr];
    e->sig[e->wr] = newevt;
    if (e->n == WIN) {
        double oldmean = e->mean;
        e->mean += (newevt - oldevt) / WIN;
        e->varsum += (newevt + oldevt - oldmean - e->mean) * (newevt - oldevt);
    } else {
        e->n++;
        double dt1 = newevt - e->mean;
        e->mean += dt1 / e->n;
        double dt2 = newevt - e->mean;
        e->varsum += dt1 * dt2;
    }
    e->wr = (e->wr + 1) % WIN;
    e->is_full = e->wr == e->rd;
}

/* add_event (:71-104); returns event_ready() */
static int prof_add(prof_t *e, float mean) {
    win_push(e, mean);
    e->q[(e->q_head + e->q_size) % (WIN + 1)] = mean; e->q_size++;
    u32 unread = e->rd < e->wr ? e->wr - e->rd : (e->n - e->rd) + e->wr;
    if (unread <= WIN / 2) return 0;
    float win_stdv = sqrt(e->varsum / e->n);
    if (win_stdv < STDV_MIN) e->to_mask = WIN - 1;
    else if (e->to_mask > 0) e->to_mask--;
    if (e->is_full) {
        e->q_head = (e->q_head + 1) % (WIN + 1); e->q_size--;
        e->rd = (e->rd + 1) % WIN;                  /* window_.pop(): its value is unused */
        e->is_full = 0;
        e->p_is_full = 1;
    }
    return e->p_is_full && e->to_mask == 0;
}

/* EventProfiler::get_full_mask (src/event_profiler.hpp:129-151), tail loop included: the unmasked means, in order, to
 * kept (room for n; may be `means` itself).  Returns their number. */
uint32_t orc_full_mask(const float *means, uint32_t n, float *kept) {
    prof_t e;
    memset(&e, 0, sizeof(e));
    u32 m = 0, nk = 0;
    for (u32 i = 0; i < n; i++) {
        int ready = prof_add(&e, means[i]);
        if (e.p_is_full) {
            if (ready) kept[nk++] = means[m];
            m++;
        }
    }
    for (; m < n; m++) {
        if (e.to_mask == 0) kept[nk++] = means[m];
        else e.to_mask--;
    }
    return nk;
}

/* read_mean / read_stdv of the span from the template model (src/dtw_test.cpp:106-115): a float running sum, then a float
 * sum of pow(float, 2) (a double), sqrt of a float */
void orc_span_target(const orc_model *tmpl, const uint16_t *kmers, uint32_t n, float *mean, float *stdv) {
    float m = 0;
    for (u32 i = 0; i < n; i++) m += tmpl->lv_mean[kmers[i]];
    m /= (float) n;
    float v = 0;
    for (u32 i = 0; i < n; i++) {
        float d = tmpl->lv_mean[kmers[i]] - m;
        v = (float) ((double) v + (double) d * (double) d);
    }
    *mean = m;
    *stdv = sqrtf(v / (float) n);
}

/* DTWr94d {NONE, 1, 1, 1} as dtw_test.cpp compiles it (src/dtw.hpp:31-122,153-173,212-214): the driver includes <math.h>
 * before dtw.hpp, so `abs(e - mean)` in dtwcost_r94d binds to the float overload -- unlike the library's bindings, where
 * it binds to int abs(int) (orc_dtw's cost_kind 1).  Path pairs (column, row) from the end cell back to the start. */
static int dtw_r94d_float(const orc_model *tmpl, const float *means, u64 Cn, const uint16_t *kmers, u64 R, uint64_t *path,
                          uint64_t *path_len, float *score) {
    const float MAX_COST = FLT_MAX / 2.0f;
    if (R == 0 || Cn == 0) return -1;
    float *mat = (float *) malloc(R * Cn * sizeof(float));
    uint8_t *bc = (uint8_t *) malloc(R * Cn);
    if (!mat || !bc) { free(mat); free(bc); return -2; }
    u64 k = 0;
    for (u64 i = 0; i < R; i++) {
        for (u64 j = 0; j < Cn; j++) {
            float cost = fabsf(means[j] - tmpl->lv_mean[kmers[i]]);
            float dsc = (j > 0 && i > 0) ? mat[Cn * (i - 1) + j - 1] : (j == i ? 0 : MAX_COST);
            float hsc = j > 0 ? mat[Cn * i + j - 1] : MAX_COST;
            float vsc = i > 0 ? mat[Cn * (i - 1) + j] : MAX_COST;
            float ds = dsc + cost, hs = hsc + cost, vs = vsc + cost;
            if (ds <= hs && ds <= vs) { mat[k] = ds; bc[k++] = 0; }      /* Move::D */
            else if (hs <= vs) { mat[k] = hs; bc[k++] = 1; }             /* Move::H */
            else { mat[k] = vs; bc[k++] = 2; }                           /* Move::V */
        }
    }
    u64 i = R - 1, j = Cn - 1, n = 0;
    *score = mat[i * Cn + j];
    path[2 * n] = j; path[2 * n + 1] = i; n++;
    k = i * Cn + j;
    while (i != 0 || j != 0) {
        if (i == 0 || bc[k] == 1) { k--; j--; }
        else if (j == 0 || bc[k] == 2) { k -= Cn; i--; }
        else { k -= Cn + 1; i--; j--; }
        path[2 * n] = j; path[2 * n + 1] = i; n++;
    }
    *path_len = n;
    free(mat);
    free(bc);
    return 0;
}

/* One query: events over raw[0, n) (n_events), the mask (n_kept means, normalised to the span's target, to means: room
 * for n), and DTWr94d {NONE, 1, 1, 1} against the n_kmers k-mers (tmpl = orc_model_init(..., complement = 0); path: room
 * for n_kept + n_kmers pairs).  Returns 0 aligned, 1 more than 50 000 means (not aligned), 2 no event left after the
 * mask (not aligned). */
int orc_dtw_align(const orc_params *p, const orc_model *tmpl, const float *raw, uint32_t n, const uint16_t *kmers,
                  uint32_t n_kmers, uint32_t *n_events, uint32_t *n_kept, float tgt[2], float *means, uint64_t *path,
                  uint64_t *path_len, float *score) {
    float *ev = (float *) malloc(((size_t) n + 1) * sizeof(float));
    u32 ne = orc_detect_events(p, raw, n, ev, NULL, NULL, NULL);
    u32 nk = orc_full_mask(ev, ne, ev);
    *n_events = ne; *n_kept = nk;
    orc_span_target(tmpl, kmers, n_kmers, &tgt[0], &tgt[1]);
    orc_normalize_to(tgt[0], tgt[1], ev, nk, means);
    free(ev);
    if (nk == 0) return 2;
    if (nk > 50000) return 1;
    return dtw_r94d_float(tmpl, means, nk, kmers, n_kmers, path, path_len, score) == 0 ? 0 : -1;
}
