/* oracle/unc_oracle.c -- CPU restatement (plain C) of the reference's `uncalled map`
 * hot path.  TEST INFRASTRUCTURE ONLY (see unc_oracle.h).  Parity status: PINNED by
 * tests/test_oracle_pinned.py against the reference's own outputs.
 *
 * Every function cites the reference file:line it restates (paths under /root/reference).
 * Build: gcc -O2 -ffp-contract=off -fPIC -shared -pthread (oracle/Makefile); baseline
 * x86-64 so that float/double rounding is identical to the reference build (no FMA).
 */
#define _GNU_SOURCE
#include "unc_oracle.h"

#include <float.h>
#include <math.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef int32_t i32;
typedef uint64_t u64;

#define KLEN 5
#define KMASK 0x3FF
#define BUF_LEN 13 /* 1 + window_length2*2, reference src/event_detector.cpp:30 */

/* ------------------------------------------------------------------ params */

/* reference src/mapper.cpp:29-52, seed_tracker.cpp:28-32, event_detector.cpp:17-26,
 * read_buffer.cpp:26-32 */
void orc_params_default(orc_params *p) {
    p->seed_len = 22;
    p->min_rep_len = 0;
    p->max_rep_copy = 50;
    p->max_paths = 10000;
    p->max_consec_stay = 8;
    p->max_events = 30000;
    p->max_stay_frac = 0.5f;
    p->min_seed_prob = -3.75f;
    p->min_map_len = 25;
    p->min_mean_conf = 6.00f;
    p->min_top_conf = 1.85f;
    p->window_length1 = 3;
    p->window_length2 = 6;
    p->threshold1 = 1.4f;
    p->threshold2 = 9.0f;
    p->peak_height = 0.2f;
    p->min_mean = 0;
    p->max_mean = 400;
    p->bp_per_sec = 450;
    p->sample_rate = 4000;
}

/* ------------------------------------------------------------------ pore model */

/* reference src/pore_model.hpp:58-62 (init_kmer), :77-103 (vector ctor), :48-56 (init_stdv),
 * complement index src/bp.hpp:77-80 */
void orc_model_init(orc_model *m, const float *ms, int complement) {
    float model_mean = 0;
    for (u32 k = 0; k < ORC_NKMER; k++) {
        float mean = ms[2 * k], stdv = ms[2 * k + 1];
        u32 idx = complement ? (k ^ KMASK) : k;
        m->lv_mean[idx] = mean;
        m->lv_var2[idx] = 2 * stdv * stdv;
        m->lognorm[idx] = (float) log(sqrt(M_PI * m->lv_var2[idx]));
        model_mean += mean;
    }
    model_mean /= (u16) ORC_NKMER;
    m->model_mean = model_mean;
    float model_stdv = 0;
    for (u32 k = 0; k < ORC_NKMER; k++) {
        float d = m->lv_mean[k] - model_mean; /* float subtract */
        model_stdv = (float) ((double) model_stdv + (double) d * (double) d);
    }
    /* sqrt(float/u16): libstdc++'s cmath overload resolves to the float version;
     * (checked against oracle/_ref: ref_model_stdv) */
    m->model_stdv = sqrtf(model_stdv / (u16) ORC_NKMER);
}

/* reference src/pore_model.hpp:163-165: float subtract, then double square / divide /
 * subtract, one rounding to float */
float orc_match_prob(const orc_model *m, float samp, u16 kmer) {
    float d = samp - m->lv_mean[kmer];
    double dd = (double) d;
    return (float) ((-(dd * dd) / (double) m->lv_var2[kmer]) - (double) m->lognorm[kmer]);
}

/* ------------------------------------------------------------------ event detector */

typedef struct {
    i32 def_peak_pos;
    float def_peak_val;
    float threshold;
    u32 window_length;
    u32 masked_to;
    i32 peak_pos;
    float peak_value;
    int valid_peak;
} detector_t;

typedef struct {
    const orc_params *prm;
    double sum[BUF_LEN], sumsq[BUF_LEN];
    u32 t, buf_mid, evt_st;
    double evt_st_sum, evt_st_sumsq;
    float len_sum;
    u32 total_events;
    detector_t sd, ld;
    float ev_mean, ev_stdv;
    u32 ev_start, ev_length;
} evdt_t;

/* reference src/event_detector.cpp:47-77 */
static void evdt_reset(evdt_t *e, const orc_params *p) {
    memset(e->sum, 0, sizeof(e->sum));
    memset(e->sumsq, 0, sizeof(e->sumsq));
    e->prm = p;
    e->t = 1;
    e->evt_st = 0;
    e->evt_st_sum = e->evt_st_sumsq = 0.0;
    e->len_sum = 0;
    e->total_events = 0;
    detector_t s = {-1, FLT_MAX, p->threshold1, p->window_length1, 0, -1, FLT_MAX, 0};
    detector_t l = {-1, FLT_MAX, p->threshold2, p->window_length2, 0, -1, FLT_MAX, 0};
    e->sd = s;
    e->ld = l;
}

/* reference src/event_detector.cpp:174-219 */
static float evdt_tstat(const evdt_t *e, u32 w_length) {
    const float eta = FLT_MIN;
    const float w_lengthf = (float) w_length;
    if (e->t <= 2 * w_length || w_length < 2) return 0;

    u32 i = e->buf_mid % BUF_LEN, st = (e->buf_mid - w_length) % BUF_LEN,
        en = (e->buf_mid + w_length) % BUF_LEN;

    double sum1 = e->sum[i] - e->sum[st];
    double sumsq1 = e->sumsq[i] - e->sumsq[st];
    float sum2 = (float) (e->sum[en] - e->sum[i]);
    float sumsq2 = (float) (e->sumsq[en] - e->sumsq[i]);
    float mean1 = (float) (sum1 / w_lengthf);
    float mean2 = sum2 / w_lengthf;
    float m1sq = mean1 * mean1; /* float products (mulss) */
    float m2sq = mean2 * mean2;
    float q2 = sumsq2 / w_lengthf; /* divss */
    float combined_var = (float) (((sumsq1 / w_lengthf - (double) m1sq) + (double) q2) - (double) m2sq);

    combined_var = fmaxf(combined_var, eta);
    const float delta_mean = mean2 - mean1;
    return fabsf(delta_mean) / sqrtf(combined_var / w_lengthf);
}

/* reference src/event_detector.cpp:221-279 */
static int evdt_peak(evdt_t *e, float current_value, detector_t *d) {
    if (d->masked_to >= e->buf_mid) return 0;

    if (d->peak_pos == d->def_peak_pos) {
        if (current_value < d->peak_value) {
            d->peak_value = current_value;
        } else if (current_value - d->peak_value > e->prm->peak_height) {
            d->peak_value = current_value;
            d->peak_pos = (i32) e->buf_mid;
        }
    } else {
        if (current_value > d->peak_value) {
            d->peak_value = current_value;
            d->peak_pos = (i32) e->buf_mid;
        }
        if (d->window_length == e->sd.window_length) {
            if (d->peak_value > d->threshold) {
                e->ld.masked_to = (u32) d->peak_pos + d->window_length;
                e->ld.peak_pos = e->ld.def_peak_pos;
                e->ld.peak_value = e->ld.def_peak_val;
                e->ld.valid_peak = 0;
            }
        }
        if (d->peak_value - current_value > e->prm->peak_height && d->peak_value > d->threshold) {
            d->valid_peak = 1;
        }
        if (d->valid_peak && (e->buf_mid - (u32) d->peak_pos) > d->window_length / 2) {
            d->peak_pos = d->def_peak_pos;
            d->peak_value = current_value;
            d->valid_peak = 0;
            return 1;
        }
    }
    return 0;
}

/* reference src/event_detector.cpp:296-319 (calibration inside the detector is identity) */
static void evdt_create_event(evdt_t *e, u32 evt_en) {
    u32 evt_en_buf = evt_en % BUF_LEN;
    e->ev_start = e->evt_st;
    e->ev_length = (u32) (float) (evt_en - e->evt_st);
    e->ev_mean = (float) ((e->sum[evt_en_buf] - e->evt_st_sum) / e->ev_length);
    const float deltasqr = (float) (e->sumsq[evt_en_buf] - e->evt_st_sumsq);
    const float var = deltasqr / e->ev_length - e->ev_mean * e->ev_mean;
    e->ev_stdv = sqrtf(fmaxf(var, 0.0f));
    e->ev_mean = (e->ev_mean + 0.0f) * 1.0f;
    e->ev_stdv = (e->ev_stdv + 0.0f) * 1.0f;
    e->evt_st = evt_en;
    e->evt_st_sum = e->sum[evt_en_buf];
    e->evt_st_sumsq = e->sumsq[evt_en_buf];
    e->len_sum += e->ev_length;
    e->total_events++;
}

/* reference src/event_detector.cpp:83-112 */
static int evdt_add_sample(evdt_t *e, float s) {
    u32 t_mod = e->t % BUF_LEN;
    float ss = s * s; /* float product, then promoted */
    if (t_mod > 0) {
        e->sum[t_mod] = e->sum[t_mod - 1] + s;
        e->sumsq[t_mod] = e->sumsq[t_mod - 1] + ss;
    } else {
        e->sum[t_mod] = e->sum[BUF_LEN - 1] + s;
        e->sumsq[t_mod] = e->sumsq[BUF_LEN - 1] + ss;
    }
    e->t++;
    e->buf_mid = e->t - (BUF_LEN / 2) - 1;

    float tstat1 = evdt_tstat(e, e->prm->window_length1), tstat2 = evdt_tstat(e, e->prm->window_length2);
    int p1 = evdt_peak(e, tstat1, &e->sd), p2 = evdt_peak(e, tstat2, &e->ld);

    if (p1 || p2) {
        evdt_create_event(e, e->buf_mid - e->prm->window_length1 + 1);
        return e->ev_mean >= e->prm->min_mean && e->ev_mean <= e->prm->max_mean;
    }
    return 0;
}

/* reference src/event_detector.cpp:114-153 */
uint32_t orc_detect_events(const orc_params *p, const float *raw, uint32_t n, float *means,
                           uint32_t *starts, uint32_t *lens, float *mean_event_len) {
    evdt_t e;
    evdt_reset(&e, p);
    u32 ne = 0;
    for (u32 i = 0; i < n; i++) {
        if (evdt_add_sample(&e, raw[i])) {
            if (means) means[ne] = e.ev_mean;
            if (starts) starts[ne] = e.ev_start;
            if (lens) lens[ne] = e.ev_length;
            ne++;
        }
    }
    if (mean_event_len) *mean_event_len = e.len_sum / e.total_events;
    return ne;
}

/* ------------------------------------------------------------------ normaliser */

/* reference src/normalizer.cpp:31-44 (set_signal) and :114-118 (at, via pop :120-129) */
void orc_normalize(const orc_model *m, const float *ev, uint32_t n, float *out) {
    if (n == 0) return;
    double mean = 0;
    for (u32 i = 0; i < n; i++) mean += ev[i];
    mean /= n;
    double varsum = 0;
    for (u32 i = 0; i < n; i++) {
        double d = ev[i] - mean;
        varsum += d * d;
    }
    float tgt_mean = m->model_mean, tgt_stdv = m->model_stdv;
    float scale = (float) (tgt_stdv / sqrt(varsum / n));
    float shift = (float) (tgt_mean - scale * mean);
    for (u32 i = 0; i < n; i++) {
        float prod = scale * ev[i];
        out[i] = prod + shift;
    }
}

/* ------------------------------------------------------------------ FM index */

struct orc_index {
    u64 primary, L2[5], seq_len, bwt_size;
    u32 *bwt;
    u64 sa_intv, n_sa;
    u64 *sa;
    u64 kmer_st[ORC_NKMER], kmer_en[ORC_NKMER];
    float thresh[64];
    int64_t l_pac;
    int n_seqs;
    char **names;
    int64_t *offsets;
    int32_t *lens;
};

typedef struct {
    u64 n_neighbor_calls, n_occ_blocks, n_sa_steps;
} fm_counters;
static __thread fm_counters *g_cnt = NULL;

/* reference submods/bwa/bwt.c:98-105 (__occ_aux): count 2-bit symbols equal to c */
static inline int occ_aux(u64 y, int c) {
    y = ((c & 2) ? y : ~y) >> 1 & ((c & 1) ? y : ~y) & 0x5555555555555555ull;
    return __builtin_popcountll(y);
}

/* reference submods/bwa/bwt.c:107-129 (bwt_occ); layout bwt.h:37-39,74-75 */
static u64 fm_occ(const orc_index *x, u64 k, u8 c) {
    if (k == x->seq_len) return x->L2[c + 1] - x->L2[c];
    if (k == (u64) -1) return 0;
    k -= (k >= x->primary);
    const u32 *p = x->bwt + ((k >> 7) << 4);
    if (g_cnt) g_cnt->n_occ_blocks++;
    u64 n;
    memcpy(&n, (const char *) p + 8 * c, 8);
    p += 8;
    const u32 *end = p + (((k >> 5) - ((k & ~127ull) >> 5)) << 1);
    for (; p < end; p += 2) n += occ_aux((u64) p[0] << 32 | p[1], c);
    n += occ_aux(((u64) p[0] << 32 | p[1]) & ~((1ull << ((~k & 31) << 1)) - 1), c);
    if (c == 0) n -= ~k & 31;
    return n;
}

/* reference submods/bwa/bwt.c:132-163 (bwt_2occ) */
static void fm_2occ(const orc_index *x, u64 k, u64 l, u8 c, u64 *ok, u64 *ol) {
    u64 _k = (k >= x->primary) ? k - 1 : k;
    u64 _l = (l >= x->primary) ? l - 1 : l;
    if (_l / 128 != _k / 128 || k == (u64) -1 || l == (u64) -1) {
        *ok = fm_occ(x, k, c);
        *ol = fm_occ(x, l, c);
    } else {
        u64 m, n, i, j;
        if (k >= x->primary) --k;
        if (l >= x->primary) --l;
        const u32 *p = x->bwt + ((k >> 7) << 4);
        if (g_cnt) g_cnt->n_occ_blocks++;
        memcpy(&n, (const char *) p + 8 * c, 8);
        p += 8;
        j = k >> 5 << 5;
        for (i = k / 128 * 128; i < j; i += 32, p += 2) n += occ_aux((u64) p[0] << 32 | p[1], c);
        m = n;
        n += occ_aux(((u64) p[0] << 32 | p[1]) & ~((1ull << ((~k & 31) << 1)) - 1), c);
        if (c == 0) n -= ~k & 31;
        *ok = n;
        j = l >> 5 << 5;
        for (; i < j; i += 32, p += 2) m += occ_aux((u64) p[0] << 32 | p[1], c);
        m += occ_aux(((u64) p[0] << 32 | p[1]) & ~((1ull << ((~l & 31) << 1)) - 1), c);
        if (c == 0) m -= ~l & 31;
        *ol = m;
    }
}

/* reference submods/bwa/bwt.c:53-59 (bwt_invPsi), bwt.h:48-55 (bwt_B0) */
static u64 fm_inv_psi(const orc_index *x, u64 k) {
    u64 y = k - (k > x->primary);
    u32 w = x->bwt[((y >> 7) << 4) + 8 + ((y & 0x7f) >> 4)];
    u64 c = (w >> ((~y & 0xf) << 1)) & 3;
    u64 r = x->L2[c] + fm_occ(x, k, (u8) c);
    return k == x->primary ? 0 : r;
}

/* reference submods/bwa/bwt.c:86-96 (bwt_sa) */
uint64_t orc_sa(const orc_index *x, uint64_t k) {
    u64 sa = 0, mask = x->sa_intv - 1;
    while (k & mask) {
        ++sa;
        k = fm_inv_psi(x, k);
        if (g_cnt) g_cnt->n_sa_steps++;
    }
    return sa + x->sa[k / x->sa_intv];
}

/* reference src/bwa_index.hpp:158-162 (get_neighbor) */
void orc_get_neighbor(const orc_index *x, u64 st, u64 en, u8 base, u64 *ost, u64 *oen) {
    u64 os, oe;
    if (g_cnt) g_cnt->n_neighbor_calls++;
    fm_2occ(x, st - 1, en, base, &os, &oe);
    *ost = x->L2[base] + os + 1;
    *oen = x->L2[base] + oe;
}

uint64_t orc_fmi_size(const orc_index *x) { return x->seq_len; }
void orc_kmer_range(const orc_index *x, u16 kmer, u64 *st, u64 *en) {
    *st = x->kmer_st[kmer];
    *en = x->kmer_en[kmer];
}
float orc_prob_thresh(const orc_index *x, int bin) { return x->thresh[bin]; }
int orc_n_seqs(const orc_index *x) { return x->n_seqs; }
const char *orc_seq_name(const orc_index *x, int i) { return x->names[i]; }
uint64_t orc_seq_len(const orc_index *x, int i) { return (u64) x->lens[i]; }

static void *read_file(const char *fn, size_t *sz) {
    FILE *fp = fopen(fn, "rb");
    if (!fp) return NULL;
    fseek(fp, 0, SEEK_END);
    long n = ftell(fp);
    fseek(fp, 0, SEEK_SET);
    char *buf = (char *) malloc((size_t) n + 1);
    if (fread(buf, 1, (size_t) n, fp) != (size_t) n) {
        fclose(fp);
        free(buf);
        return NULL;
    }
    buf[n] = 0;
    fclose(fp);
    *sz = (size_t) n;
    return buf;
}

/* reference submods/bwa/bwt.c:421-462 (bwt_restore_bwt / bwt_restore_sa),
 * submods/bwa/bntseq.c:97-135 (.ann), src/bwa_index.hpp:116-135 (k-mer ranges, incl. the
 * get_base_range quirk :172-174), src/mapper.cpp:123-157 (.uncl thresholds) */
int orc_index_load(const char *prefix, const char *preset, orc_index **out) {
    char fn[4096];
    size_t sz;
    orc_index *x = (orc_index *) calloc(1, sizeof(orc_index));

    snprintf(fn, sizeof fn, "%s.bwt", prefix);
    char *b = (char *) read_file(fn, &sz);
    if (!b) { free(x); return -1; }
    memcpy(&x->primary, b, 8);
    memcpy(&x->L2[1], b + 8, 32);
    x->L2[0] = 0;
    x->bwt_size = (sz - 40) >> 2;
    x->bwt = (u32 *) malloc(x->bwt_size * 4 + 64);
    memcpy(x->bwt, b + 40, x->bwt_size * 4);
    memset((char *) x->bwt + x->bwt_size * 4, 0, 64);
    x->seq_len = x->L2[4];
    free(b);

    snprintf(fn, sizeof fn, "%s.sa", prefix);
    b = (char *) read_file(fn, &sz);
    if (!b) { orc_index_free(x); return -2; }
    u64 primary, seq_len;
    memcpy(&primary, b, 8);
    memcpy(&x->sa_intv, b + 40, 8);
    memcpy(&seq_len, b + 48, 8);
    if (primary != x->primary || seq_len != x->seq_len) { free(b); orc_index_free(x); return -3; }
    x->n_sa = (x->seq_len + x->sa_intv) / x->sa_intv;
    x->sa = (u64 *) calloc(x->n_sa, 8);
    x->sa[0] = (u64) -1;
    memcpy(x->sa + 1, b + 56, (x->n_sa - 1) * 8);
    free(b);

    snprintf(fn, sizeof fn, "%s.ann", prefix);
    FILE *fp = fopen(fn, "r");
    if (!fp) { orc_index_free(x); return -4; }
    long long xx;
    unsigned seed;
    if (fscanf(fp, "%lld%d%u", &xx, &x->n_seqs, &seed) != 3) { fclose(fp); orc_index_free(x); return -5; }
    x->l_pac = xx;
    x->names = (char **) calloc((size_t) x->n_seqs, sizeof(char *));
    x->offsets = (int64_t *) calloc((size_t) x->n_seqs, 8);
    x->lens = (int32_t *) calloc((size_t) x->n_seqs, 4);
    for (int i = 0; i < x->n_seqs; i++) {
        unsigned gi;
        char str[8192];
        int c, n_ambs;
        if (fscanf(fp, "%u%8191s", &gi, str) != 2) { fclose(fp); orc_index_free(x); return -5; }
        x->names[i] = strdup(str);
        while ((c = fgetc(fp)) != '\n' && c != EOF) {}
        if (fscanf(fp, "%lld%d%d", &xx, &x->lens[i], &n_ambs) != 3) { fclose(fp); orc_index_free(x); return -5; }
        x->offsets[i] = xx;
    }
    fclose(fp);

    for (u32 k = 0; k < ORC_NKMER; k++) {
        u8 head = (u8) ((k >> (2 * KLEN - 2)) & 3);
        u64 st = x->L2[head], en = x->L2[head + 1]; /* get_base_range: start NOT +1 */
        for (u8 i = 1; i < KLEN; i++) {
            u8 base = (u8) ((k >> (2 * (KLEN - i - 1))) & 3);
            u64 ns, ne;
            orc_get_neighbor(x, st, en, base, &ns, &ne);
            st = ns;
            en = ne;
        }
        x->kmer_st[k] = st;
        x->kmer_en[k] = en;
    }

    if (preset && !strcmp(preset, "-")) { *out = x; return 0; }   /* index time: no .uncl yet (self_align) */
    snprintf(fn, sizeof fn, "%s.uncl", prefix);
    fp = fopen(fn, "r");
    if (!fp) { orc_index_free(x); return -6; }
    char *line = NULL;
    size_t cap = 0;
    while (getline(&line, &cap, fp) >= 0) {
        size_t L = strlen(line);
        while (L && (line[L - 1] == '\n' || line[L - 1] == '\r')) line[--L] = 0;
        char *name = strtok(line, "\t");
        char *fn_str = strtok(NULL, "\t");
        if (!name) continue;
        if (preset && preset[0] && strcmp(name, preset)) continue;
        u8 fmbin = 63;
        char *tok;
        while ((tok = strtok(fn_str, ",")) != NULL) {
            fn_str = NULL;
            x->thresh[fmbin] = (float) atof(tok);
            fmbin--;
        }
        for (; fmbin < 64; fmbin--) x->thresh[fmbin] = x->thresh[fmbin + 1];
    }
    free(line);
    fclose(fp);
    *out = x;
    return 0;
}

/* self_align (reference src/self_align_ref.cpp:34-91): for every sampled start position i of every
 * sequence (glibc rand() % sample_dist == 0 after srand(0), one draw per position), the FM range lengths of
 * the backward search that walks FORWARD along the reference with complemented bases, from
 * get_base_range (whose start is L2[b], not L2[b]+1, src/bwa_index.hpp:172-174) until the range is unique.
 * Bases come from the .pac file (src/bwa_index.hpp:141-147,257-259).  Two calls: values == NULL counts. */
int orc_self_align(const orc_index *x, const char *prefix, uint32_t sample_dist, uint64_t *n_paths, uint64_t *n_values,
                   uint64_t *offsets, uint64_t *values) {
    char fn[4096];
    snprintf(fn, sizeof fn, "%s.pac", prefix);
    size_t sz = 0;
    u8 *pac = (u8 *) read_file(fn, &sz);
    if (!pac) return -1;
    srand(0);
    u64 st = 0, np = 0, nv = 0;
    for (int s = 0; s < x->n_seqs; s++) {
        const u64 len = (u64) x->lens[s];
        for (u64 i = 0; i < len; i++) {
            if (rand() % sample_dist != 0) continue;
            if (offsets) offsets[np] = nv;
            np++;
            u8 b = (u8) (3 - ((pac[(st + i) >> 2] >> (((3 ^ (st + i)) & 3) << 1)) & 3));
            u64 rs = x->L2[b], re = x->L2[b + 1];
            u64 j = i + 1;
            for (; j < len && re - rs + 1 > 1; j++) {
                if (values) values[nv] = re - rs + 1;
                nv++;
                b = (u8) (3 - ((pac[(st + j) >> 2] >> (((3 ^ (st + j)) & 3) << 1)) & 3));
                u64 ns, ne;
                orc_get_neighbor(x, rs, re, b, &ns, &ne);
                rs = ns; re = ne;
            }
            if (re - rs + 1 > 0) { if (values) values[nv] = re - rs + 1; nv++; }
        }
        st += len;
    }
    if (offsets) offsets[np] = nv;
    free(pac);
    if (n_paths) *n_paths = np;
    if (n_values) *n_values = nv;
    return 0;
}

void orc_index_free(orc_index *x) {
    if (!x) return;
    free(x->bwt);
    free(x->sa);
    if (x->names)
        for (int i = 0; i < x->n_seqs; i++) free(x->names[i]);
    free(x->names);
    free(x->offsets);
    free(x->lens);
    free(x);
}

/* reference submods/bwa/bntseq.c:354-368 (bns_pos2rid) */
static int pos2rid(const orc_index *x, int64_t pos_f) {
    int left, mid, right;
    if (pos_f >= x->l_pac) return -1;
    left = 0; mid = 0; right = x->n_seqs;
    while (left < right) {
        mid = (left + right) >> 1;
        if (pos_f >= x->offsets[mid]) {
            if (mid == x->n_seqs - 1) break;
            if (pos_f < x->offsets[mid + 1]) break;
            left = mid + 1;
        } else right = mid;
    }
    return mid;
}

/* ------------------------------------------------------------------ seed tracker */

typedef struct {
    u64 ref_st, ren_start, ren_end;
    u32 evt_st, evt_en, total_len;
} cluster_t;

typedef struct {
    cluster_t *set; /* sorted: ren_start descending, then evt_en descending (std::set order) */
    u32 n, cap;
    u32 *lens; /* std::multiset<u32>, ascending */
    u32 n_lens, cap_lens;
    cluster_t max_map;
    float len_sum;
} tracker_t;

static const cluster_t NULL_ALN = {0, 1, 0, 1, 0, 0}; /* reference src/seed_tracker.cpp:34-38 */

static void trk_reset(tracker_t *t) {
    t->n = 0;
    t->n_lens = 0;
    t->max_map = NULL_ALN;
    t->len_sum = 0;
}

/* reference src/seed_tracker.cpp:97-102 (operator<) */
static inline int clu_less(const cluster_t *a, const cluster_t *b) {
    if (a->ren_start != b->ren_start) return a->ren_start > b->ren_start;
    return a->evt_en > b->evt_en;
}

static u32 trk_lower_bound(const tracker_t *t, const cluster_t *key) {
    u32 lo = 0, hi = t->n;
    while (lo < hi) {
        u32 mid = (lo + hi) >> 1;
        if (clu_less(&t->set[mid], key)) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

/* std::set::insert: only if no equivalent key exists */
static int trk_insert_unique(tracker_t *t, const cluster_t *c) {
    u32 pos = trk_lower_bound(t, c);
    if (pos < t->n && !clu_less(c, &t->set[pos])) return 0;
    if (t->n == t->cap) {
        t->cap = t->cap ? t->cap * 2 : 1024;
        t->set = (cluster_t *) realloc(t->set, t->cap * sizeof(cluster_t));
    }
    memmove(&t->set[pos + 1], &t->set[pos], (t->n - pos) * sizeof(cluster_t));
    t->set[pos] = *c;
    t->n++;
    return 1;
}

static void trk_erase(tracker_t *t, u32 pos) {
    memmove(&t->set[pos], &t->set[pos + 1], (t->n - pos - 1) * sizeof(cluster_t));
    t->n--;
}

static void lens_insert(tracker_t *t, u32 v) {
    if (t->n_lens == t->cap_lens) {
        t->cap_lens = t->cap_lens ? t->cap_lens * 2 : 1024;
        t->lens = (u32 *) realloc(t->lens, t->cap_lens * 4);
    }
    u32 lo = 0, hi = t->n_lens;
    while (lo < hi) {
        u32 mid = (lo + hi) >> 1;
        if (t->lens[mid] <= v) lo = mid + 1;
        else hi = mid;
    }
    memmove(&t->lens[lo + 1], &t->lens[lo], (t->n_lens - lo) * 4);
    t->lens[lo] = v;
    t->n_lens++;
}

static void lens_erase_one(tracker_t *t, u32 v) {
    u32 lo = 0, hi = t->n_lens;
    while (lo < hi) {
        u32 mid = (lo + hi) >> 1;
        if (t->lens[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    if (lo < t->n_lens && t->lens[lo] == v) {
        memmove(&t->lens[lo], &t->lens[lo + 1], (t->n_lens - lo - 1) * 4);
        t->n_lens--;
    }
}

/* reference src/seed_tracker.cpp:56-73 (SeedCluster::update), u8-truncated growth */
static u8 clu_update(cluster_t *a, const cluster_t *ns) {
    u8 growth = 0;
    if (ns->ren_start < a->ren_end) {
        if (ns->ren_end > a->ren_end) {
            growth = (u8) (ns->ren_end - a->ren_end);
            a->ren_start = ns->ren_start;
            a->ren_end = ns->ren_end;
        } else {
            a->ren_start = ns->ren_start;
        }
    } else {
        growth = (u8) ns->total_len;
        a->ren_start = ns->ren_start;
        a->ren_end = ns->ren_end;
    }
    a->evt_en = ns->evt_en;
    a->total_len += growth;
    return growth;
}

/* reference src/seed_tracker.cpp:157-232 (add_seed) */
static void trk_add_seed(tracker_t *t, const orc_params *p, u64 ref_en, u32 ref_len, u32 evt_st) {
    cluster_t ns;
    ns.ren_start = ref_en - ref_len + 1;
    ns.ren_end = ref_en;
    ns.ref_st = ns.ren_start;
    ns.evt_st = evt_st;
    ns.evt_en = evt_st;
    ns.total_len = (u32) (ns.ren_end - ns.ren_start + 1);

    u32 loc = trk_lower_bound(t, &ns);
    u32 loc_match = t->n; /* == end() */
    u64 e2 = ns.evt_en, r2 = ns.ren_start;

    while (loc != t->n) {
        u64 e1 = t->set[loc].evt_en, r1 = t->set[loc].ren_start;
        int higher_sup = loc_match == t->n || t->set[loc_match].total_len < t->set[loc].total_len;
        int in_range = e1 <= e2 && r2 - r1 <= e2 - e1 && (r2 - r1) >= (e2 - e1) / 12;
        if (higher_sup && in_range) {
            loc_match = loc;
        } else if (r2 - r1 >= e2) {
            break;
        }
        loc++;
    }

    if (loc_match != t->n) {
        cluster_t a = t->set[loc_match];
        u32 prev_len = a.total_len;
        clu_update(&a, &ns);
        if (a.total_len != prev_len) {
            t->len_sum += a.total_len - prev_len;
            lens_insert(t, a.total_len);
            lens_erase_one(t, prev_len);
            if (a.total_len >= p->min_map_len && a.total_len > t->max_map.total_len) t->max_map = a;
        }
        trk_erase(t, loc_match);
        trk_insert_unique(t, &a); /* silently dropped when an equal key exists */
    } else {
        lens_insert(t, ns.total_len);
        t->len_sum += ns.total_len;
        if (ns.total_len >= p->min_map_len && ns.total_len > t->max_map.total_len) t->max_map = ns;
        trk_insert_unique(t, &ns);
    }
}

/* reference src/seed_tracker.cpp:129-143 (get_final), :259-262 (check_map_conf) */
static cluster_t trk_get_final(const tracker_t *t, const orc_params *p) {
    if (t->max_map.total_len < p->min_map_len || t->n_lens < 2) return NULL_ALN;
    float mean_len = t->len_sum / t->n;
    float second_len = (float) t->lens[t->n_lens - 2];
    u32 seed_len = t->max_map.total_len;
    if ((p->min_mean_conf > 0 && seed_len / mean_len >= p->min_mean_conf) ||
        (p->min_top_conf > 0 && seed_len / second_len >= p->min_top_conf))
        return t->max_map;
    return NULL_ALN;
}

/* The seed tracker alone (test hook): feeds the seeds one by one; after seed i out[6i..6i+6) = clusters in the set,
 * max_map (total_len, low word of ren_start, evt_en), total_len of get_final() (0 = none), multiset size.
 * Reference src/seed_tracker.cpp:129-143,157-232. */
int orc_tracker_run(const orc_params *p, const uint64_t *ref_en, const uint32_t *ref_len, const uint32_t *evt, uint32_t n,
                    uint32_t *out) {
    tracker_t t;
    memset(&t, 0, sizeof(t));
    trk_reset(&t);
    for (uint32_t i = 0; i < n; i++) {
        trk_add_seed(&t, p, ref_en[i], ref_len[i], evt[i]);
        cluster_t f = trk_get_final(&t, p);
        out[6 * i + 0] = t.n;
        out[6 * i + 1] = t.max_map.total_len;
        out[6 * i + 2] = (uint32_t) t.max_map.ren_start;
        out[6 * i + 3] = t.max_map.evt_en;
        out[6 * i + 4] = f.total_len;
        out[6 * i + 5] = t.n_lens;
    }
    free(t.set);
    free(t.lens);
    return 0;
}

/* ------------------------------------------------------------------ DTW (SURVEY 8(f) rank 4)
 * reference src/dtw.hpp: DTW<float,u16,Func> :31-183 -- rows = k-mers, columns = event means; compute_matrix :49-74,
 * traceback :76-122, boundary scores :153-173; costs DTWr94p :188-190 (-match_prob of the TEMPLATE model), DTWr94d :212-214
 * (|e - mean_k|).  Path pairs are (column, row) from the end cell back to the start, as get_path() returns them. */
#define DTW_MAX_COST (FLT_MAX / 2.0f)
int orc_dtw(const orc_model *tmpl, int cost_kind, int subseq, float dw, float hw, float vw, const float *means, uint32_t n_cols,
            const uint16_t *kmers, uint32_t n_rows, uint64_t *path, uint64_t *path_len, float *score) {
    const u64 R = n_rows, Cn = n_cols;
    if (R == 0 || Cn == 0) return -1;
    float *mat = (float *) malloc(R * Cn * sizeof(float));
    u8 *bc = (u8 *) malloc(R * Cn);
    if (!mat || !bc) { free(mat); free(bc); return -2; }
    u64 k = 0;
    for (u64 i = 0; i < R; i++) {
        for (u64 j = 0; j < Cn; j++) {
            /* DTWr94d: `abs(e - mean)` in src/dtw.hpp:213 binds to int abs(int) -- the float difference is truncated towards zero
             * first (verified against oracle/_ref: all its r94d scores are whole numbers) */
            float cost = cost_kind == 0 ? -orc_match_prob(tmpl, means[j], kmers[i]) : (float) abs((int) (means[j] - tmpl->lv_mean[kmers[i]]));
            float dsc, hsc, vsc;
            if (j > 0 && i > 0) dsc = mat[Cn * (i - 1) + j - 1];
            else if (j == i || (i == 0 && subseq == 2) || (j == 0 && subseq == 1)) dsc = 0;
            else dsc = DTW_MAX_COST;
            if (j > 0) hsc = mat[Cn * i + j - 1];
            else hsc = subseq == 1 ? 0 : DTW_MAX_COST;
            if (i > 0) vsc = mat[Cn * (i - 1) + j];
            else vsc = subseq == 2 ? 0 : DTW_MAX_COST;
            float ds = dsc + (dw * cost), hs = hsc + (hw * cost), vs = vsc + (vw * cost);
            if (ds <= hs && ds <= vs) { mat[k] = ds; bc[k++] = 0; }      /* Move::D */
            else if (hs <= vs) { mat[k] = hs; bc[k++] = 1; }             /* Move::H */
            else { mat[k] = vs; bc[k++] = 2; }                           /* Move::V */
        }
    }
    u64 i = R - 1, j = Cn - 1;
    if (subseq == 1) {                     /* ROW: best cell of the last column */
        for (u64 q = 0; q < R; q++) if (mat[q * Cn + j] < mat[i * Cn + j]) i = q;
    } else if (subseq == 2) {              /* COL: best cell of the last row */
        for (u64 q = 0; q < Cn; q++) if (mat[i * Cn + q] < mat[i * Cn + j]) j = q;
    }
    *score = mat[i * Cn + j];
    u64 n = 0;
    path[2 * n] = j; path[2 * n + 1] = i; n++;
    k = i * Cn + j;
    while (!(i == 0 || subseq == 1) || !(j == 0 || subseq == 2)) {
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

/* ------------------------------------------------------------------ mapper */

typedef struct {
    u64 fm_start, fm_end;
    u32 event_moves;
    u32 emit_idx;
    float seed_prob;
    u16 kmer;
    u8 length, consec_stays, sa_checked;
    float prob_sums[23];
} path_t;

typedef struct {
    const orc_index *idx;
    const orc_model *model;
    const orc_params *prm;
    path_t *prev, *next;
    u32 prev_size, event_i;
    float kmer_probs[ORC_NKMER];
    u8 sources_added[ORC_NKMER];
    tracker_t trk;
    u32 path_mask, path_tail_move;
    orc_paf_rec *rec;
    orc_trace_seed *tseeds;    /* orc_set_path_trace: the event's seeds so far */
    u32 tseeds_n, tseeds_cap;
} mapper_t;

static orc_trace_fn g_trace = NULL;
static void *g_trace_ud = NULL;
void orc_set_trace(orc_trace_fn fn, void *ud) { g_trace = fn; g_trace_ud = ud; }
static orc_path_trace_fn g_path_trace = NULL;
static void *g_path_trace_ud = NULL;
void orc_set_path_trace(orc_path_trace_fn fn, void *ud) { g_path_trace = fn; g_path_trace_ud = ud; }

static void trace_seed(mapper_t *mp, u64 ref_end, u32 move_count, u32 evt) {
    if (mp->tseeds_n == mp->tseeds_cap) {
        mp->tseeds_cap = mp->tseeds_cap ? 2 * mp->tseeds_cap : 256;
        mp->tseeds = (orc_trace_seed *) realloc(mp->tseeds, (size_t) mp->tseeds_cap * sizeof(orc_trace_seed));
    }
    orc_trace_seed *s = &mp->tseeds[mp->tseeds_n++];
    s->ref_end = ref_end; s->move_count = move_count; s->evt = evt;
}

static void path_trace(mapper_t *mp, u32 nn) {
    orc_trace_row *rows = (orc_trace_row *) calloc((size_t) nn + 1, sizeof(orc_trace_row));
    for (u32 i = 0; i < nn; i++) {
        const path_t *q = &mp->prev[i];
        orc_trace_row *o = &rows[i];
        if (q->length == 0) continue;
        o->fm_start = q->fm_start; o->fm_end = q->fm_end;
        o->kmer = q->kmer; o->length = q->length; o->consec_stays = q->consec_stays; o->sa_checked = q->sa_checked;
        o->event_moves = q->event_moves;
        memcpy(&o->seed_prob, &q->seed_prob, 4);
        memcpy(&o->prob_sum, &q->prob_sums[q->length], 4);
        o->valid = 1;
    }
    u32 flags[ORC_NKMER / 32] = {0};
    for (u32 k = 0; k < ORC_NKMER; k++) if (mp->sources_added[k]) flags[k >> 5] |= 1u << (k & 31u);
    g_path_trace(g_path_trace_ud, mp->event_i, nn, rows, mp->tseeds_n, mp->tseeds, flags);
    free(rows);
}

/* reference src/mapper.cpp:751-772 (make_source) */
static void make_source(path_t *q, u64 st, u64 en, u16 kmer, float prob) {
    q->length = 1;
    q->consec_stays = 0;
    q->event_moves = 1;
    q->seed_prob = prob;
    q->fm_start = st;
    q->fm_end = en;
    q->kmer = kmer;
    q->sa_checked = 0;
    q->prob_sums[0] = 0;
    q->prob_sums[1] = prob;
}

/* reference src/mapper.cpp:775-807 (make_child) */
static void make_child(const mapper_t *mp, path_t *q, const path_t *p, u64 st, u64 en, u16 kmer, float prob,
                       u8 move) {
    u32 seed_len = mp->prm->seed_len;
    u8 stay = 1 - move;
    q->length = p->length + (p->length < seed_len);
    q->fm_start = st;
    q->fm_end = en;
    q->kmer = kmer;
    q->sa_checked = p->sa_checked;
    q->event_moves = ((p->event_moves << 1) | move) & mp->path_mask;
    q->consec_stays = (u8) ((p->consec_stays + stay) * stay);
    if (p->length == seed_len) {
        memcpy(q->prob_sums, &p->prob_sums[1], seed_len * sizeof(float));
        q->prob_sums[seed_len] = q->prob_sums[seed_len - 1] + prob;
        q->seed_prob = (q->prob_sums[seed_len] - q->prob_sums[0]) / seed_len;
        q->event_moves |= mp->path_tail_move;
    } else {
        memcpy(q->prob_sums, p->prob_sums, q->length * sizeof(float));
        q->prob_sums[q->length] = q->prob_sums[q->length - 1] + prob;
        q->seed_prob = q->prob_sums[q->length] / q->length;
    }
}

/* reference src/mapper.cpp:842-863 (is_seed_valid) */
static int is_seed_valid(const mapper_t *mp, const path_t *q, int path_ended) {
    const orc_params *p = mp->prm;
    u8 move_count = (u8) __builtin_popcount(q->event_moves);
    u8 stay_count = (u8) (q->length - move_count);
    u64 len = q->fm_end - q->fm_start + 1;
    return (q->length == p->seed_len && q->seed_prob >= p->min_seed_prob) &&
           ((len == 1 && (q->event_moves & 1) == 1 && stay_count <= p->max_stay_frac * p->seed_len) ||
            (path_ended && len <= p->max_rep_copy && move_count >= p->min_rep_len));
}

/* reference src/mapper.cpp:665-700 (update_seeds) */
static void update_seeds(mapper_t *mp, path_t *q, int path_ended) {
    if (!is_seed_valid(mp, q, path_ended)) return;
    q->sa_checked = 1;
    u8 move_count = (u8) __builtin_popcount(q->event_moves);
    for (u64 s = q->fm_start; s <= q->fm_end; s++) {
        u64 sa_end = mp->idx->seq_len - orc_sa(mp->idx, s);
        trk_add_seed(&mp->trk, mp->prm, sa_end, move_count, mp->event_i - (u32) path_ended);
        if (g_path_trace) trace_seed(mp, sa_end, move_count, mp->event_i - (u32) path_ended);
        mp->rec->n_seeds++;
    }
}

/* reference src/mapper.cpp:866-871 (operator<) + emission order as the documented
 * tie-break (the reference's pdqsort leaves ties unspecified) */
static int path_cmp(const void *a, const void *b) {
    const path_t *p = (const path_t *) a, *q = (const path_t *) b;
    if (p->fm_start != q->fm_start) return p->fm_start < q->fm_start ? -1 : 1;
    if (p->fm_end != q->fm_end) return p->fm_end < q->fm_end ? -1 : 1;
    if (p->seed_prob < q->seed_prob) return -1;
    if (q->seed_prob < p->seed_prob) return 1;
    return p->emit_idx < q->emit_idx ? -1 : (p->emit_idx > q->emit_idx);
}

/* ---- the reference's child sort, restated: pdqsort (reference submods/pdqsort/pdqsort.h, Orson Peters' pattern-defeating
 * quicksort, non-branchless variant because PathBuffer is not arithmetic: pdqsort.h:507-526) under operator< of
 * src/mapper.cpp:866-871.  It is UNSTABLE: children that compare equal end up in an order that depends on the whole
 * array's input order.  orc_set_child_sort(1) selects it, so that the oracle reproduces the unmodified reference even there;
 * the default (0) is the stable order the CUDA path uses (DESIGN.md section 2).  Elements are moved as whole structs, as
 * the reference's memcpy copy constructor does (src/mapper.cpp:742-744). */
static int g_child_sort_pdq = 0;          /* process-wide: the batch entry points map on worker threads */
static unsigned long g_pdq_heapsorts = 0;
void orc_set_child_sort(int pdqsort_mode) { g_child_sort_pdq = pdqsort_mode; }
unsigned long orc_pdq_heapsort_fallbacks(void) { return g_pdq_heapsorts; }

static inline int p_less(const path_t *a, const path_t *b) {
    if (a->fm_start != b->fm_start) return a->fm_start < b->fm_start;
    if (a->fm_end != b->fm_end) return a->fm_end < b->fm_end;
    return a->seed_prob < b->seed_prob;
}
static inline void p_swap(path_t *a, path_t *b) { path_t t = *a; *a = *b; *b = t; }
static inline void p_sort2(path_t *a, path_t *b) { if (p_less(b, a)) p_swap(a, b); }
static inline void p_sort3(path_t *a, path_t *b, path_t *c) { p_sort2(a, b); p_sort2(b, c); p_sort2(a, b); }

/* pdqsort.h:76-97 (guarded) and :99-121 (unguarded: *(begin-1) is known to be <= everything in the range) */
static void pdq_insertion(path_t *begin, path_t *end, int guarded) {
    if (begin == end) return;
    for (path_t *cur = begin + 1; cur != end; ++cur) {
        path_t *sift = cur, *sift_1 = cur - 1;
        if (p_less(sift, sift_1)) {
            path_t tmp = *sift;
            do { *sift-- = *sift_1; } while ((!guarded || sift != begin) && p_less(&tmp, --sift_1));
            *sift = tmp;
        }
    }
}
/* pdqsort.h:123-148: gives up (returns 0) once more than 8 element moves were needed */
static int pdq_partial_insertion(path_t *begin, path_t *end) {
    if (begin == end) return 1;
    long limit = 0;
    for (path_t *cur = begin + 1; cur != end; ++cur) {
        if (limit > 8) return 0;
        path_t *sift = cur, *sift_1 = cur - 1;
        if (p_less(sift, sift_1)) {
            path_t tmp = *sift;
            do { *sift-- = *sift_1; } while (sift != begin && p_less(&tmp, --sift_1));
            *sift = tmp;
            limit += cur - sift;
        }
    }
    return 1;
}
/* pdqsort.h:340-381: elements equal to the pivot go right; *already = the range was partitioned on entry */
static path_t *pdq_partition_right(path_t *begin, path_t *end, int *already) {
    path_t pivot = *begin;
    path_t *first = begin, *last = end;
    while (p_less(++first, &pivot)) {}
    if (first - 1 == begin) { while (first < last && !p_less(--last, &pivot)) {} }
    else { while (!p_less(--last, &pivot)) {} }
    *already = first >= last;
    while (first < last) {
        p_swap(first, last);
        while (p_less(++first, &pivot)) {}
        while (!p_less(--last, &pivot)) {}
    }
    path_t *pivot_pos = first - 1;
    *begin = *pivot_pos;
    *pivot_pos = pivot;
    return pivot_pos;
}
/* pdqsort.h:384-408: elements equal to the pivot go left */
static path_t *pdq_partition_left(path_t *begin, path_t *end) {
    path_t pivot = *begin;
    path_t *first = begin, *last = end;
    while (p_less(&pivot, --last)) {}
    if (last + 1 == end) { while (first < last && !p_less(&pivot, ++first)) {} }
    else { while (!p_less(&pivot, ++first)) {} }
    while (first < last) {
        p_swap(first, last);
        while (p_less(&pivot, --last)) {}
        while (!p_less(&pivot, ++first)) {}
    }
    path_t *pivot_pos = last;
    *begin = *pivot_pos;
    *pivot_pos = pivot;
    return pivot_pos;
}
/* libstdc++'s std::make_heap + std::sort_heap (bits/stl_heap.h: __adjust_heap / __push_heap), pdqsort's fallback after
 * log2(n) highly unbalanced partitions (pdqsort.h:464-468) */
static void heap_adjust(path_t *first, long hole, long len, path_t value) {
    const long top = hole;
    long child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (p_less(first + child, first + (child - 1))) child--;
        first[hole] = first[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        first[hole] = first[child - 1];
        hole = child - 1;
    }
    long parent = (hole - 1) / 2;
    while (hole > top && p_less(first + parent, &value)) {
        first[hole] = first[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    first[hole] = value;
}
static void pdq_heapsort(path_t *first, path_t *last) {
    long len = last - first;
    g_pdq_heapsorts++;
    if (len < 2) return;
    for (long parent = (len - 2) / 2;; parent--) {
        heap_adjust(first, parent, len, first[parent]);
        if (parent == 0) break;
    }
    while (last - first > 1) {
        --last;
        path_t value = *last;
        *last = *first;
        heap_adjust(first, 0, last - first, value);
    }
}
/* pdqsort.h:411-504 */
static void pdq_loop(path_t *begin, path_t *end, int bad_allowed, int leftmost) {
    for (;;) {
        long size = end - begin;
        if (size < 24) { pdq_insertion(begin, end, leftmost); return; }
        long s2 = size / 2;
        if (size > 128) {
            p_sort3(begin, begin + s2, end - 1);
            p_sort3(begin + 1, begin + (s2 - 1), end - 2);
            p_sort3(begin + 2, begin + (s2 + 1), end - 3);
            p_sort3(begin + (s2 - 1), begin + s2, begin + (s2 + 1));
            p_swap(begin, begin + s2);
        } else {
            p_sort3(begin + s2, begin, end - 1);
        }
        if (!leftmost && !p_less(begin - 1, begin)) {
            begin = pdq_partition_left(begin, end) + 1;
            continue;
        }
        int already;
        path_t *pivot_pos = pdq_partition_right(begin, end, &already);
        long l_size = pivot_pos - begin, r_size = end - (pivot_pos + 1);
        int highly_unbalanced = l_size < size / 8 || r_size < size / 8;
        if (highly_unbalanced) {
            if (--bad_allowed == 0) { pdq_heapsort(begin, end); return; }
            if (l_size >= 24) {
                p_swap(begin, begin + l_size / 4);
                p_swap(pivot_pos - 1, pivot_pos - l_size / 4);
                if (l_size > 128) {
                    p_swap(begin + 1, begin + (l_size / 4 + 1));
                    p_swap(begin + 2, begin + (l_size / 4 + 2));
                    p_swap(pivot_pos - 2, pivot_pos - (l_size / 4 + 1));
                    p_swap(pivot_pos - 3, pivot_pos - (l_size / 4 + 2));
                }
            }
            if (r_size >= 24) {
                p_swap(pivot_pos + 1, pivot_pos + (1 + r_size / 4));
                p_swap(end - 1, end - r_size / 4);
                if (r_size > 128) {
                    p_swap(pivot_pos + 2, pivot_pos + (2 + r_size / 4));
                    p_swap(pivot_pos + 3, pivot_pos + (3 + r_size / 4));
                    p_swap(end - 2, end - (1 + r_size / 4));
                    p_swap(end - 3, end - (2 + r_size / 4));
                }
            }
        } else if (already && pdq_partial_insertion(begin, pivot_pos) && pdq_partial_insertion(pivot_pos + 1, end)) {
            return;
        }
        pdq_loop(begin, pivot_pos, bad_allowed, leftmost);
        begin = pivot_pos + 1;
        leftmost = 0;
    }
}
static void pdq_sort(path_t *begin, path_t *end) {
    if (begin == end) return;
    int lg = 0;
    for (long n = end - begin; n >>= 1;) ++lg;
    pdq_loop(begin, end, lg, 1);
}

/* Diagnostics (orc_set_child_sort(2) = pdqsort + statistics): per event, does the survivor of any run of equal ranges --
 * the LAST of the run, reference src/mapper.cpp:569-572 -- differ between pdqsort's order and the stable order in a field
 * that outlives the event?  [0] events with children, [1] events where a survivor differs, [2] children, [3] children in
 * runs whose survivor differs. */
static unsigned long g_tie_stats[4];
void orc_tie_stats(unsigned long out[4]) { memcpy(out, g_tie_stats, sizeof(g_tie_stats)); }
static void tie_stats(const path_t *next, u32 n) {
    path_t *a = (path_t *) malloc((size_t) n * sizeof(path_t)), *b = (path_t *) malloc((size_t) n * sizeof(path_t));
    memcpy(a, next, (size_t) n * sizeof(path_t));
    memcpy(b, next, (size_t) n * sizeof(path_t));
    pdq_sort(a, a + n);
    qsort(b, n, sizeof(path_t), path_cmp);
    unsigned long bad_runs = 0, bad_children = 0;
    for (u32 i = 0; i < n;) {
        u32 j = i;
        while (j + 1 < n && a[j + 1].fm_start == a[i].fm_start && a[j + 1].fm_end == a[i].fm_end) j++;
        const path_t *x = &a[j], *y = &b[j];             /* the survivors (both arrays hold the same multiset of keys) */
        int same = x->event_moves == y->event_moves && x->length == y->length && x->consec_stays == y->consec_stays &&
                   x->sa_checked == y->sa_checked && x->kmer == y->kmer &&
                   !memcmp(x->prob_sums, y->prob_sums, sizeof(x->prob_sums));
        if (!same) { bad_runs++; bad_children += j - i + 1; }
        i = j + 1;
    }
    __sync_fetch_and_add(&g_tie_stats[0], 1);
    __sync_fetch_and_add(&g_tie_stats[1], bad_runs ? 1 : 0);
    __sync_fetch_and_add(&g_tie_stats[2], n);
    __sync_fetch_and_add(&g_tie_stats[3], bad_children);
    free(a);
    free(b);
}

static inline float prob_thresh(const orc_index *x, u64 fmlen) { return x->thresh[__builtin_clzll(fmlen)]; }

/* reference src/mapper.cpp:703-706 (event_to_bp) */
static u32 event_to_bp(const mapper_t *mp, u32 evt_i, int last, float mean_event_len) {
    float bp_per_samp = mp->prm->bp_per_sec / mp->prm->sample_rate;
    float v = (evt_i * mean_event_len * bp_per_samp) + last * (KLEN - 1);
    return (u32) (int64_t) v; /* x86-64 float->u32: cvttss2si to 64 bit, low half kept */
}

/* reference src/mapper.cpp:708-728 (set_ref_loc), src/bwa_index.hpp:213-220 (translate_loc) */
static void set_ref_loc(mapper_t *mp, const cluster_t *sc, float mean_event_len) {
    const orc_index *x = mp->idx;
    orc_paf_rec *r = mp->rec;
    int fwd = sc->ref_st < x->seq_len / 2;
    u64 sa_st = fwd ? sc->ref_st : x->seq_len - (sc->ren_end + KLEN - 1);
    u64 rd_st = event_to_bp(mp, sc->evt_st - mp->prm->seed_len, 0, mean_event_len);
    u64 rd_en = event_to_bp(mp, sc->evt_en, 1, mean_event_len);
    u64 rd_len = event_to_bp(mp, mp->event_i, 1, mean_event_len);
    u64 rf_st = 0, rf_len = 0;
    int rid = pos2rid(x, (int64_t) sa_st);
    if (rid >= 0) {
        rf_st = sa_st - (u64) x->offsets[rid];
        rf_len = (u64) x->lens[rid];
    }
    u64 rf_en = rf_st + (sc->ren_end - sc->ref_st + KLEN);
    r->mapped = 1;
    r->fwd = fwd;
    r->rid = rid;
    r->matches = (u16) (sc->total_len + KLEN - 1);
    r->rd_len = rd_len;
    r->rd_st = rd_st;
    r->rd_en = rd_en;
    r->rf_st = rf_st;
    r->rf_en = rf_en;
    r->rf_len = rf_len;
}

/* reference src/mapper.cpp:433-663 (map_next).  Returns 1 when the read is finished. */
static int map_next_event(mapper_t *mp, float event, float mean_event_len);
static int map_next(mapper_t *mp, const float *events, u32 n_events, float mean_event_len) {
    /* norm_.empty() after n_events pops (reference src/normalizer.cpp:120-129) */
    if (mp->event_i >= n_events || mp->event_i >= mp->prm->max_events) return 1;
    return map_next_event(mp, events[mp->event_i], mean_event_len);
}

/* the body of map_next from `float event = norm_.pop()` on (reference src/mapper.cpp:440-663) */
static int map_next_event(mapper_t *mp, float event, float mean_event_len) {
    const orc_index *x = mp->idx;
    const orc_params *prm = mp->prm;
    for (u32 k = 0; k < ORC_NKMER; k++) mp->kmer_probs[k] = orc_match_prob(mp->model, event, (u16) k);
    const float *probs = mp->kmer_probs;
    const float source_prob = x->thresh[0];
    const u32 maxp = prm->max_paths;
    mp->tseeds_n = 0;

    u32 nn = 0; /* next_path - next_paths_.begin() */

    for (u32 pi = 0; pi < mp->prev_size; pi++) {
        path_t *pp = &mp->prev[pi];
        if (pp->length == 0) continue;
        int child_found = 0;
        u16 prev_kmer = pp->kmer;
        float thr = prob_thresh(x, pp->fm_end - pp->fm_start + 1);

        if (pp->consec_stays < prm->max_consec_stay && probs[prev_kmer] >= thr) {
            make_child(mp, &mp->next[nn], pp, pp->fm_start, pp->fm_end, prev_kmer, probs[prev_kmer], 0);
            mp->next[nn].emit_idx = nn;
            child_found = 1;
            if (++nn == maxp) break;
        }

        for (u8 b = 0; b < 4; b++) {
            u16 next_kmer = (u16) (((prev_kmer << 2) & KMASK) | b);
            if (probs[next_kmer] < thr) continue;
            u64 ns, ne;
            orc_get_neighbor(x, pp->fm_start, pp->fm_end, b, &ns, &ne);
            if (!(ns <= ne)) continue;
            make_child(mp, &mp->next[nn], pp, ns, ne, next_kmer, probs[next_kmer], 1);
            mp->next[nn].emit_idx = nn;
            child_found = 1;
            if (++nn == maxp) break;
        }

        if (!child_found && !pp->sa_checked) update_seeds(mp, pp, 1);
        if (nn == maxp) break;
    }
    mp->rec->n_children += nn;

    if (nn != 0) {
        u32 next_size = nn;
        if (g_child_sort_pdq) {
            if (g_child_sort_pdq == 2) tie_stats(mp->next, next_size);   /* diagnostics: how often does the order of ties matter? */
            pdq_sort(mp->next, mp->next + next_size);
        } else {
            qsort(mp->next, next_size, sizeof(path_t), path_cmp);
        }

        u16 source_kmer, prev_kmer = ORC_NKMER;
        u64 unchecked_st = 1, unchecked_en = 0, src_st, src_en;

        for (u32 i = 0; i < next_size; i++) {
            path_t *ci = &mp->next[i];
            source_kmer = ci->kmer;

            if (source_kmer != prev_kmer && nn != maxp && probs[source_kmer] >= source_prob) {
                mp->sources_added[source_kmer] = 1;
                src_st = x->kmer_st[source_kmer];
                src_en = ci->fm_start - 1;
                if (src_st <= src_en) {
                    make_source(&mp->next[nn], src_st, src_en, source_kmer, probs[source_kmer]);
                    nn++;
                    mp->rec->n_sources++;
                }
                unchecked_st = ci->fm_end + 1;
                unchecked_en = x->kmer_en[source_kmer];
            }
            prev_kmer = source_kmer;

            if (i < next_size - 1 && ci->fm_start == mp->next[i + 1].fm_start &&
                ci->fm_end == mp->next[i + 1].fm_end) {
                ci->length = 0; /* invalidate */
                continue;
            }

            if (nn != maxp && probs[source_kmer] >= source_prob) {
                src_st = unchecked_st;
                src_en = unchecked_en;
                if (i < next_size - 1 && source_kmer == mp->next[i + 1].kmer) {
                    src_en = mp->next[i + 1].fm_start - 1;
                    if (unchecked_st <= mp->next[i + 1].fm_end) unchecked_st = mp->next[i + 1].fm_end + 1;
                }
                if (src_st <= src_en) {
                    make_source(&mp->next[nn], src_st, src_en, source_kmer, probs[source_kmer]);
                    nn++;
                    mp->rec->n_sources++;
                }
            }
            update_seeds(mp, ci, 0);
        }
    }

    for (u32 kmer = 0; kmer < ORC_NKMER && nn != maxp; kmer++) {
        u64 st = x->kmer_st[kmer], en = x->kmer_en[kmer];
        if (!mp->sources_added[kmer] && probs[kmer] >= source_prob && nn != maxp && st <= en) {
            make_source(&mp->next[nn], st, en, (u16) kmer, probs[kmer]);
            nn++;
            mp->rec->n_sources++;
        } else {
            mp->sources_added[kmer] = 0;
        }
    }

    mp->prev_size = nn;
    path_t *tmp = mp->prev;
    mp->prev = mp->next;
    mp->next = tmp;
    if (nn > mp->rec->max_paths_seen) mp->rec->max_paths_seen = nn;

    if (g_trace) {
        u64 h = 1469598103934665603ull;
        for (u32 i = 0; i < nn; i++) {
            const path_t *q = &mp->prev[i];
            if (q->length == 0) continue;
            u32 sp;
            memcpy(&sp, &q->seed_prob, 4);
            u64 v[4] = {q->fm_start, q->fm_end, ((u64) q->kmer << 32) | sp,
                        ((u64) q->length << 40) | ((u64) q->consec_stays << 32) | q->event_moves};
            for (int j = 0; j < 4; j++) { h ^= v[j]; h *= 1099511628211ull; }
        }
        g_trace(g_trace_ud, mp->event_i, nn, mp->trk.n, h);
    }
    if (g_path_trace) path_trace(mp, nn);

    cluster_t sc = trk_get_final(&mp->trk, prm);
    if (sc.evt_st <= sc.evt_en) {
        set_ref_loc(mp, &sc, mean_event_len);
        return 1;
    }
    mp->event_i++;
    return 0;
}

static void mapper_init(mapper_t *mp, const orc_index *idx, const orc_model *m, const orc_params *p) {
    memset(mp, 0, sizeof(*mp));
    mp->idx = idx;
    mp->model = m;
    mp->prm = p;
    mp->prev = (path_t *) calloc(p->max_paths, sizeof(path_t));
    mp->next = (path_t *) calloc(p->max_paths, sizeof(path_t));
    for (u32 i = 0; i < p->seed_len; i++) mp->path_mask |= 1u << i;
    mp->path_tail_move = 1u << (p->seed_len - 1);
}

static void mapper_free(mapper_t *mp) {
    free(mp->prev);
    free(mp->next);
    free(mp->trk.set);
    free(mp->trk.lens);
    free(mp->tseeds);
}

/* reference src/mapper.cpp:188-200 (map_read), :216-246 (reset), read_buffer.cpp:263-266 */
static __thread int g_carry_flags = 0;   /* orc_map_reads_one_mapper: keep sources_added_ from the previous read (see there) */
static void mapper_map_read(mapper_t *mp, const float *raw, u32 n, orc_paf_rec *out, float *ev_buf,
                            float *norm_buf) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    memset(out, 0, sizeof(*out));
    out->rid = -1;
    mp->rec = out;
    mp->prev_size = 0;
    mp->event_i = 0;
    trk_reset(&mp->trk);
    if (!g_carry_flags) memset(mp->sources_added, 0, sizeof(mp->sources_added)); /* fresh Mapper per read */
    fm_counters cnt = {0, 0, 0};
    g_cnt = &cnt;

    float mean_event_len = 0;
    u32 ne = orc_detect_events(mp->prm, raw, n, ev_buf, NULL, NULL, &mean_event_len);
    out->n_events = ne;
    float bp_per_samp = mp->prm->bp_per_sec / mp->prm->sample_rate;
    out->rd_len = (u64) ((u64) n * bp_per_samp);
    if (ne > 0) { /* the reference divides by zero on an event-less read (normalizer.cpp:123) */
        orc_normalize(mp->model, ev_buf, ne, norm_buf);
        while (!map_next(mp, norm_buf, ne, mean_event_len)) {}
    }
    out->events_used = mp->event_i;
    out->n_neighbor_calls = cnt.n_neighbor_calls;
    out->n_occ_blocks = cnt.n_occ_blocks;
    out->n_sa_steps = cnt.n_sa_steps;
    out->n_clusters = mp->trk.n;
    g_cnt = NULL;
    clock_gettime(CLOCK_MONOTONIC, &t1);
    out->map_ms = (float) ((t1.tv_sec - t0.tv_sec) * 1e3 + (t1.tv_nsec - t0.tv_nsec) * 1e-6);
}

int orc_map_read(const orc_index *idx, const orc_model *m, const orc_params *p, const float *raw, uint32_t n,
                 orc_paf_rec *out) {
    mapper_t mp;
    mapper_init(&mp, idx, m, p);
    float *ev = (float *) malloc(((size_t) n + 1) * 4), *nb = (float *) malloc(((size_t) n + 1) * 4);
    mapper_map_read(&mp, raw, n, out, ev, nb);
    free(ev);
    free(nb);
    mapper_free(&mp);
    return 0;
}

/* ONE long-lived Mapper mapping the reads in the given order, as a MapPool thread does (reference
 * src/map_pool.cpp:104-158): Mapper::reset() (src/mapper.cpp:216-246) clears everything except the
 * sources_added_ flags (:88), so a read starts with whatever its predecessor left set.  This is what
 * `uncalled map -t 1` computes for a multi-read input; single-threaded on purpose (the order is the point). */
int orc_map_reads_one_mapper(const orc_index *idx, const orc_model *m, const orc_params *p, const float *samples,
                             const uint64_t *offsets, const uint32_t *lens, uint32_t n_reads, orc_paf_rec *out) {
    mapper_t mp;
    mapper_init(&mp, idx, m, p);
    u32 mx = 0;
    for (u32 i = 0; i < n_reads; i++) if (lens[i] > mx) mx = lens[i];
    float *ev = (float *) malloc(((size_t) mx + 1) * 4), *nb = (float *) malloc(((size_t) mx + 1) * 4);
    g_carry_flags = 1;
    for (u32 i = 0; i < n_reads; i++) mapper_map_read(&mp, samples + offsets[i], lens[i], &out[i], ev, nb);
    g_carry_flags = 0;
    free(ev);
    free(nb);
    mapper_free(&mp);
    return 0;
}

/* One read mapped by a Mapper whose sources_added_ flags (reference src/mapper.cpp:88) start as flags_in
 * (bit k&31 of word k>>5 = k-mer k; NULL = all clear) and are returned as they stand when map_read returns
 * (flags_out, may be NULL).  orc_map_reads_one_mapper is this call chained over the reads; the CUDA path's
 * ordered mode (unc_map_batch_ordered) is checked against both. */
int orc_map_read_flags(const orc_index *idx, const orc_model *m, const orc_params *p, const float *raw, uint32_t n,
                       const uint32_t *flags_in, uint32_t *flags_out, orc_paf_rec *out) {
    mapper_t mp;
    mapper_init(&mp, idx, m, p);
    float *ev = (float *) malloc(((size_t) n + 1) * 4), *nb = (float *) malloc(((size_t) n + 1) * 4);
    for (u32 k = 0; k < ORC_NKMER; k++) mp.sources_added[k] = flags_in ? (u8) ((flags_in[k >> 5] >> (k & 31u)) & 1u) : 0;
    g_carry_flags = 1;
    mapper_map_read(&mp, raw, n, out, ev, nb);
    g_carry_flags = 0;
    if (flags_out) {
        memset(flags_out, 0, (ORC_NKMER / 32) * 4);
        for (u32 k = 0; k < ORC_NKMER; k++) if (mp.sources_added[k]) flags_out[k >> 5] |= 1u << (k & 31u);
    }
    free(ev);
    free(nb);
    mapper_free(&mp);
    return 0;
}

/* ------------------------------------------------------------------ streaming path
 * reference src/mapper.cpp:281-431 (add_chunk / process_chunk / map_chunk), src/normalizer.cpp:46-75,
 * 114-152 (streaming Normalizer), src/event_profiler.hpp:46-104, src/realtime_pool.cpp:108-139,349-356
 * (the order in which a worker thread and try_add_chunk drive one channel), src/read_buffer.cpp:249-296. */

typedef struct {            /* Normalizer as a ring (reference src/normalizer.hpp:72-79) */
    float *signal;
    u32 len, n, rd, wr;
    double mean, varsum;
    int is_full, is_empty;
    float tgt_mean, tgt_stdv;
} snorm_t;

static void snorm_init(snorm_t *z, u32 len, float tgt_mean, float tgt_stdv) {
    memset(z, 0, sizeof(*z));
    z->signal = (float *) calloc(len, sizeof(float));
    z->len = len; z->is_empty = 1; z->tgt_mean = tgt_mean; z->tgt_stdv = tgt_stdv;
}
/* Normalizer::reset (:77-88) */
static void snorm_reset(snorm_t *z) {
    z->n = z->rd = z->wr = 0; z->mean = z->varsum = 0; z->is_full = 0; z->is_empty = 1; z->signal[0] = 0;
}
/* Normalizer::push (:46-75): Welford while filling, rolling update once the ring has wrapped */
static int snorm_push(snorm_t *z, float newevt) {
    if (z->is_full) return 0;
    double oldevt = z->signal[z->wr];
    z->signal[z->wr] = newevt;
    if (z->n == z->len) {
        double oldmean = z->mean;
        z->mean += (newevt - oldevt) / z->len;
        z->varsum += (newevt + oldevt - oldmean - z->mean) * (newevt - oldevt);
    } else {
        z->n++;
        double dt1 = newevt - z->mean;
        z->mean += dt1 / z->n;
        double dt2 = newevt - z->mean;
        z->varsum += dt1 * dt2;
    }
    z->wr = (z->wr + 1) % z->len;
    z->is_empty = 0;
    z->is_full = z->wr == z->rd;
    return 1;
}
/* Normalizer::at + pop (:114-129): scale/shift from the statistics at pop time */
static float snorm_pop(snorm_t *z) {
    float scale = z->tgt_stdv / sqrt(z->varsum / z->n);
    float shift = z->tgt_mean - scale * z->mean;
    float e = scale * z->signal[z->rd] + shift;
    z->rd = (z->rd + 1) % z->len;
    z->is_empty = z->rd == z->wr;
    z->is_full = 0;
    return e;
}
/* Normalizer::unread_size (:131-134) -- note n_, not the ring length */
static u32 snorm_unread(const snorm_t *z) {
    if (z->rd < z->wr) return z->wr - z->rd;
    return (z->n - z->rd) + z->wr;
}
/* Normalizer::skip_unread (:136-152) */
static u32 snorm_skip_unread(snorm_t *z, u32 nkeep) {
    if (nkeep >= snorm_unread(z)) return 0;
    z->is_full = 0;
    z->is_empty = nkeep == 0;
    u32 new_rd;
    if (nkeep <= z->wr) new_rd = z->wr - nkeep;
    else new_rd = z->n - (nkeep - z->wr);
    u32 nskip;
    if (new_rd > z->rd) nskip = new_rd - z->rd;
    else nskip = (z->n - z->rd) + new_rd;
    z->rd = new_rd;
    return nskip;
}

#define EVP_WIN 25u         /* EventProfiler::PRMS_DEF (reference src/event_profiler.cpp:4-10) */
#define EVP_STDV_MIN 5.0f
typedef struct {            /* EventProfiler (reference src/event_profiler.hpp:14-104) */
    snorm_t window;
    float means[EVP_WIN + 1];   /* std::deque<Event> events_: only the means are used downstream */
    u32 q_head, q_size;
    float next_mean;
    int is_full;
    u32 to_mask;
} evprof_t;

static void evprof_reset(evprof_t *e) {
    snorm_reset(&e->window);
    e->q_head = e->q_size = 0; e->next_mean = 0; e->is_full = 0; e->to_mask = 0;
}
/* EventProfiler::add_event (:71-104); returns event_ready() */
static int evprof_add(evprof_t *e, float mean) {
    snorm_push(&e->window, mean);
    e->means[(e->q_head + e->q_size) % (EVP_WIN + 1)] = mean; e->q_size++;
    if (snorm_unread(&e->window) <= EVP_WIN / 2) return 0;
    float win_stdv = sqrt(e->window.varsum / e->window.n);      /* Normalizer::get_stdv: double sqrt -> float */
    if (win_stdv < EVP_STDV_MIN) e->to_mask = EVP_WIN - 1;
    else if (e->to_mask > 0) e->to_mask--;
    if (e->window.is_full) {
        e->next_mean = e->means[e->q_head];
        e->q_head = (e->q_head + 1) % (EVP_WIN + 1); e->q_size--;
        snorm_pop(&e->window);
        e->is_full = 1;
    }
    return e->is_full && e->to_mask == 0;
}

/* One channel of a flow cell: what a RealtimePool keeps per channel between reads -- the Mapper with
 * its streaming normaliser statistics and sources_added_ flags (reference src/realtime_pool.cpp:38-60,
 * src/mapper.cpp:66-95); everything else is reset by Mapper::reset() at new_read (:218-246). */
typedef struct {
    mapper_t mp;
    snorm_t norm;
    evprof_t prof;
    evdt_t ed;
    u64 n_pushed;           /* successful normaliser pushes so far (reporting only) */
} stream_chan_t;

static void chan_init(stream_chan_t *c, const orc_index *idx, const orc_model *m, const orc_params *p) {
    mapper_init(&c->mp, idx, m, p);
    snorm_init(&c->norm, 6000, m->model_mean, m->model_stdv);   /* Normalizer::PRMS_DEF.len; Mapper::Mapper set_target */
    snorm_init(&c->prof.window, EVP_WIN, 0, 0);
    evprof_reset(&c->prof);
    evdt_reset(&c->ed, p);
    c->n_pushed = 0;
}
static void chan_free(stream_chan_t *c) {
    free(c->norm.signal); free(c->prof.window.signal);
    mapper_free(&c->mp);
}

/* One read fed chunk by chunk (chunk_len samples per chunk, full chunks only as
 * ReadBuffer::get_chunks cuts them, at most max_chunks), with the wall-clock limits disabled:
 * process_chunk -> map_chunk (evt_batch_size = 5 events per call) -> the next chunk only once the
 * previous one is fully mapped; no more signal -> request_reset -> FAILURE with the ended flag. */
static void chan_map_read(stream_chan_t *c, const float *raw, uint32_t n, uint32_t chunk_len, uint32_t max_chunks,
                          orc_paf_rec *out, uint32_t *n_chunks_used, int32_t *ended) {
    const orc_params *p = c->mp.prm;
    mapper_t *mp = &c->mp;
    memset(out, 0, sizeof(*out));
    out->rid = -1;
    if (n_chunks_used) *n_chunks_used = 0;
    if (ended) *ended = 0;
    u32 n_chunks = chunk_len ? n / chunk_len : 0;
    if (n_chunks > max_chunks) n_chunks = max_chunks;
    if (n_chunks == 0) return;

    /* Mapper::new_read(Chunk&) -> reset() (reference src/mapper.cpp:210-246) */
    mp->rec = out;
    mp->prev_size = 0;
    mp->event_i = 0;
    trk_reset(&mp->trk);
    snorm_skip_unread(&c->norm, 0);
    evdt_reset(&c->ed, p);
    evprof_reset(&c->prof);
    fm_counters cnt = {0, 0, 0};
    g_cnt = &cnt;
    snorm_t *norm = &c->norm;
    evprof_t *prof = &c->prof;
    evdt_t *ed = &c->ed;
    const float bp_per_samp = p->bp_per_sec / p->sample_rate;
    const u32 evt_batch = 5;                                    /* Mapper::PRMS.evt_batch_size */

    u32 chunk_count = 1, next_chunk = 1, cur = 0;
    u64 raw_len = chunk_len;
    int chunk_processed = 0, reset_req = 0, is_ended = 0, done = 0;
    while (!done) {
        /* ---- process_chunk (:301-363) */
        if (!chunk_processed && !reset_req) {
            u32 nevents = 0;
            const float *ck = raw + (size_t) cur * chunk_len;
            for (u32 i = 0; i < chunk_len; i++) {
                if (!evdt_add_sample(ed, ck[i])) continue;
                if (!evprof_add(prof, ed->ev_mean)) continue;
                float evt_mean = prof->next_mean;
                if (!snorm_push(norm, evt_mean)) {
                    u32 nskip = snorm_skip_unread(norm, nevents);
                    mp->event_i += nskip; mp->prev_size = 0;      /* skip_events */
                    if (!snorm_push(norm, evt_mean)) goto chunk_done;   /* returns with the chunk unprocessed */
                }
                nevents++;
                c->n_pushed++;
            }
            chunk_processed = 1;
        }
    chunk_done:
        /* ---- map_chunk (:381-431) */
        if (reset_req || mp->event_i >= p->max_events) {
            is_ended = 1; done = 1;                                /* set_failed + set_ended */
        } else if (norm->is_empty && chunk_processed && chunk_count >= max_chunks) {
            done = 1;                                              /* set_failed */
        } else if (!norm->is_empty) {
            u32 nev = mp->event_i + evt_batch > p->max_events ? p->max_events - mp->event_i : evt_batch;
            for (u32 i = 0; i < nev && !norm->is_empty; i++) {
                float event = snorm_pop(norm);
                float mel = ed->len_sum / ed->total_events;        /* EventDetector::mean_event_len at this point */
                if (map_next_event(mp, event, mel)) { snorm_skip_unread(norm, 0); done = 1; break; }
            }
        }
        if (done) break;
        /* ---- RealtimePool::try_add_chunk (:108-139) */
        if (chunk_processed && norm->is_empty) {
            if (next_chunk < n_chunks) {
                /* Mapper::add_chunk (:281-299) -> ReadBuffer::add_chunk (:271-284) */
                if (chunk_count >= max_chunks) {                  /* chunks_maxed: set_failed; the next map_chunk's */
                    done = 1;                                     /* first test adds set_ended when event_i_ is at max_events */
                    if (mp->event_i >= p->max_events) is_ended = 1;
                }
                else { cur = next_chunk++; chunk_count++; raw_len += chunk_len; chunk_processed = 0; }
            } else reset_req = 1;
        }
    }
    if (!out->mapped) out->rd_len = (u64) (raw_len * bp_per_samp);   /* ReadBuffer::set_raw_len (:263-266) */
    out->n_events = ed->total_events;
    out->events_used = mp->event_i;
    out->n_neighbor_calls = cnt.n_neighbor_calls;
    out->n_occ_blocks = cnt.n_occ_blocks;
    out->n_sa_steps = cnt.n_sa_steps;
    out->n_clusters = mp->trk.n;
    g_cnt = NULL;
    if (n_chunks_used) *n_chunks_used = chunk_count;
    if (ended) *ended = is_ended;
}

int orc_stream_map_read(const orc_index *idx, const orc_model *m, const orc_params *p, const float *raw,
                        uint32_t n, uint32_t chunk_len, uint32_t max_chunks, orc_paf_rec *out,
                        uint32_t *n_chunks_used, int32_t *ended) {
    stream_chan_t c;
    chan_init(&c, idx, m, p);
    chan_map_read(&c, raw, n, chunk_len, max_chunks, out, n_chunks_used, ended);
    chan_free(&c);
    return 0;
}

/* orc_stream_map_channel, and after every read the channel's streaming normaliser:
 * norm_state (optional, 4 per read): its (mean_, varsum_, n_, wr_) after the read;
 * n_pushed (optional, 1 per read): the channel's normaliser pushes so far. */
int orc_stream_map_channel_norm(const orc_index *idx, const orc_model *m, const orc_params *p, const float *samples,
                                const uint64_t *offsets, const uint32_t *lens, uint32_t n_reads, uint32_t chunk_len,
                                uint32_t max_chunks, orc_paf_rec *out, uint32_t *n_chunks_used, int32_t *ended,
                                double *norm_state, uint64_t *n_pushed) {
    stream_chan_t c;
    chan_init(&c, idx, m, p);
    for (uint32_t i = 0; i < n_reads; i++) {
        chan_map_read(&c, samples + offsets[i], lens[i], chunk_len, max_chunks, out + i,
                      n_chunks_used ? n_chunks_used + i : NULL, ended ? ended + i : NULL);
        if (norm_state) {
            double *s = norm_state + (size_t) 4 * i;
            s[0] = c.norm.mean; s[1] = c.norm.varsum; s[2] = c.norm.n; s[3] = c.norm.wr;
        }
        if (n_pushed) n_pushed[i] = c.n_pushed;
    }
    chan_free(&c);
    return 0;
}

/* Several reads one after the other on ONE channel (the channel's Mapper persists, as in RealtimePool). */
int orc_stream_map_channel(const orc_index *idx, const orc_model *m, const orc_params *p, const float *samples,
                           const uint64_t *offsets, const uint32_t *lens, uint32_t n_reads, uint32_t chunk_len,
                           uint32_t max_chunks, orc_paf_rec *out, uint32_t *n_chunks_used, int32_t *ended) {
    return orc_stream_map_channel_norm(idx, m, p, samples, offsets, lens, n_reads, chunk_len, max_chunks, out,
                                       n_chunks_used, ended, NULL, NULL);
}

/* The events process_chunk pushes into the normaliser, without the mapper: the detector and the event profiler over
 * n_chunks chunks of one read (both start afresh, as at Mapper::new_read).  cum_pushed[k]: pushes after chunk k. */
int orc_stream_chunk_pushes(const orc_params *p, const float *raw, uint32_t n_chunks, uint32_t chunk_len,
                            uint32_t *cum_pushed) {
    evdt_t ed;
    evprof_t prof;
    evdt_reset(&ed, p);
    snorm_init(&prof.window, EVP_WIN, 0, 0);
    evprof_reset(&prof);
    u32 n = 0;
    for (u32 k = 0; k < n_chunks; k++) {
        for (u32 i = 0; i < chunk_len; i++) {
            if (!evdt_add_sample(&ed, raw[(size_t) k * chunk_len + i])) continue;
            if (evprof_add(&prof, ed.ev_mean)) n++;
        }
        cum_pushed[k] = n;
    }
    free(prof.window.signal);
    return 0;
}

typedef struct {
    const orc_index *idx;
    const orc_model *m;
    const orc_params *p;
    const float *samples;
    const u64 *offsets;
    const u32 *lens;
    u32 n_reads;
    u32 *next;
    orc_paf_rec *out;
} mt_job;

static void *mt_worker(void *arg) {
    mt_job *j = (mt_job *) arg;
    mapper_t mp;
    mapper_init(&mp, j->idx, j->m, j->p);
    u32 maxn = 0;
    for (u32 i = 0; i < j->n_reads; i++)
        if (j->lens[i] > maxn) maxn = j->lens[i];
    float *ev = (float *) malloc(((size_t) maxn + 1) * 4), *nb = (float *) malloc(((size_t) maxn + 1) * 4);
    for (;;) {
        u32 i = __atomic_fetch_add(j->next, 1, __ATOMIC_RELAXED);
        if (i >= j->n_reads) break;
        mapper_map_read(&mp, j->samples + j->offsets[i], j->lens[i], &j->out[i], ev, nb);
    }
    free(ev);
    free(nb);
    mapper_free(&mp);
    return NULL;
}

int orc_map_batch_mt(const orc_index *idx, const orc_model *m, const orc_params *p, const float *samples,
                     const uint64_t *offsets, const uint32_t *lens, uint32_t n_reads, int n_threads,
                     orc_paf_rec *out) {
    if (n_threads < 1) n_threads = 1;
    u32 next = 0;
    mt_job j = {idx, m, p, samples, offsets, lens, n_reads, &next, out};
    pthread_t *th = (pthread_t *) malloc(sizeof(pthread_t) * (size_t) n_threads);
    for (int t = 0; t < n_threads; t++) pthread_create(&th[t], NULL, mt_worker, &j);
    for (int t = 0; t < n_threads; t++) pthread_join(th[t], NULL);
    free(th);
    return 0;
}
