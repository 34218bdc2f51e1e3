// unc_k1.cuh -- K1: warp-parallel event detection (reference src/event_detector.cpp:83-319).
//
// The reference detector is a serial FSM over samples; its cost is the two windowed t-statistics
// per sample (mixed float/double arithmetic that must be reproduced bit for bit).  Here one WARP
// owns one read and walks it in tiles of 32 x K1_CH positions:
//
//   load    the tile's raw samples (f32 pA or i16 DAC) arrive in shared memory by one bulk
//           asynchronous copy (TMA, cp.async.bulk) completing on an mbarrier
//   T pass  lane k computes both t-statistics for the K1_CH consecutive positions of its chunk
//           from sliding 3-sample sums kept in registers, and stores them to shared memory
//   FSM     the peak-detector FSM (two coupled detectors) is run SPECULATIVELY: lane k warms up
//           over the last K1_WARM positions of lane k-1's chunk from a neutral state, then runs
//           its own chunk; afterwards every lane compares the state it assumed at its chunk
//           start with the final state of the lane before it and re-runs from the true state
//           on a mismatch (rare: the FSM forgets its past at every fired peak).  The result is
//           exactly the serial FSM's.
//   events  fired peaks -> (end position, prefix sum) lists -> event means, validity, ordered
//           compaction into the read's output row.
//
// Exactness.  The reference accumulates prefix sums of the samples (and of their float squares)
// sequentially in double.  The warp-parallel sums are bit-identical iff no addition rounds,
// which holds when all samples are multiples of 2^e and sum|s| < 2^(53+e)  (true for real
// pA signals and for calibrated DAC values).  That condition is CHECKED per read while the
// samples stream through; a read that fails it (or has >= 2^24 samples) is flagged and redone
// by the serial routine unc_k1_read (k1_fallback kernel), so results never depend on it.
// Divisions by the constant window lengths use the exactly-rounded Markstein sequence
// (q = a*r; q' = fma(fma(-w, q, a), r, q), r = RN(1/w)); tests/arith/k1_arith_check.c
// (run by tests/test_k1_emul.py) checks it exhaustively over all 2^32 floats and on 6*10^8 random doubles against
// IEEE division; below 2^-100, where subnormal quotients can tie, the IEEE division is used.
#pragma once
#include "unc_device.cuh"

#ifndef K1_CH
#define K1_CH 36u              /* positions per lane per tile: a multiple of 3 (even) */
#endif
#ifndef K1_WARM
#define K1_WARM 12u            /* speculative warm-up length (<= K1_CH) */
#endif
#define K1_TS (K1_CH + 1u)     /* padded row stride (words) of the per-lane T rows: conflict-free */
#define K1_TILE (32u * K1_CH)
#define K1_HALO 6u
#define K1_RAW_WORDS (K1_TILE + 2u * K1_HALO + 8u)   /* f32 tile + halo + alignment slack */

struct K1WarpSmem {
    float raw[K1_RAW_WORDS];       // raw tile (f32, or i16 in the first half)  -- 16-byte aligned
    float t1[32 * K1_TS];          // short-window t-statistics, row per lane; later the fired-peak lists
    float t2[32 * K1_TS];          // long-window t-statistics; later the prefix sums of the fired peaks
    u64 bar;                       // mbarrier of the bulk copy
    u64 pad;
};

struct K1Fsm {                     // the two coupled peak detectors (reference event_detector.hpp Detector)
    i32 s_pos; float s_val; u32 s_valid;                 // short: masked_to is never written (stays 0)
    u32 l_masked; i32 l_pos; float l_val; u32 l_valid;   // long
};

// equality of two states as seen from position `at` on: a mask that ended before `at` has no effect
UNC_DEV bool k1_fsm_eq(const K1Fsm &a, const K1Fsm &b, u32 at) {
    u32 ma = a.l_masked >= at ? a.l_masked : 0u, mb = b.l_masked >= at ? b.l_masked : 0u;
    return a.s_pos == b.s_pos && f2u(a.s_val) == f2u(b.s_val) && a.s_valid == b.s_valid && ma == mb &&
           a.l_pos == b.l_pos && f2u(a.l_val) == f2u(b.l_val) && a.l_valid == b.l_valid;
}
UNC_DEV K1Fsm k1_fsm_shfl_up(const K1Fsm &a) {
    K1Fsm r;
    r.s_pos = (i32) w_shfl_up((u32) a.s_pos, 1); r.s_val = u2f(w_shfl_up(f2u(a.s_val), 1)); r.s_valid = w_shfl_up(a.s_valid, 1);
    r.l_masked = w_shfl_up(a.l_masked, 1); r.l_pos = (i32) w_shfl_up((u32) a.l_pos, 1);
    r.l_val = u2f(w_shfl_up(f2u(a.l_val), 1)); r.l_valid = w_shfl_up(a.l_valid, 1);
    return r;
}
UNC_DEV K1Fsm k1_fsm_bcast(const K1Fsm &a, int src) {
    K1Fsm r;
    r.s_pos = (i32) w_shfl((u32) a.s_pos, src); r.s_val = u2f(w_shfl(f2u(a.s_val), src)); r.s_valid = w_shfl(a.s_valid, src);
    r.l_masked = w_shfl(a.l_masked, src); r.l_pos = (i32) w_shfl((u32) a.l_pos, src);
    r.l_val = u2f(w_shfl(f2u(a.l_val), src)); r.l_valid = w_shfl(a.l_valid, src);
    return r;
}

// One step of both detectors at position m (= buf_mid) with t-statistics t1, t2: reference
// src/event_detector.cpp:221-279 (peak_detect, short then long) as called from add_sample :94-98,
// written with selects (the lanes of a warp walk different chunks, so branches would diverge).
// The short detector's `masked_to (0) >= buf_mid` skip at buf_mid == 0 is reproduced by feeding
// t1 = 0 there (k1_fix_head): its state is then {pos -1, value 0} and a zero input changes nothing.
// Returns true when either detector fires.
UNC_DEV bool k1_fsm_step(K1Fsm &f, float t1, float t2, u32 m, float thr1, float thr2, float h) {
    // ---- short detector (window 3: fires when buf_mid - peak_pos > 3/2)
    const bool inA = f.s_pos < 0;
    const bool ltA = t1 < f.s_val;
    const bool riseA = !ltA && f_sub(t1, f.s_val) > h;
    const bool gtB = t1 > f.s_val;
    const float valB = gtB ? t1 : f.s_val;
    const i32 posB = gtB ? (i32) m : f.s_pos;
    const bool overB = valB > thr1;
    const bool resetL = !inA && overB;                            // the short detector masks and resets the long one
    const bool validB = f.s_valid || (f_sub(valB, t1) > h && overB);
    const bool p1 = !inA && validB && (m - (u32) posB) > 1u;
    const float nsv = inA ? ((ltA || riseA) ? t1 : f.s_val) : (p1 ? t1 : valB);
    const i32 nsp = inA ? (riseA ? (i32) m : -1) : (p1 ? -1 : posB);
    f.s_valid = (!inA && !p1 && validB) ? 1u : 0u;
    f.s_val = nsv; f.s_pos = nsp;
    // ---- long detector (window 6: fires when buf_mid - peak_pos > 6/2), after the short one's reset
    const u32 lm = resetL ? (u32) posB + 3u : f.l_masked;
    const i32 lp = resetL ? -1 : f.l_pos;
    const float lv = resetL ? 3.402823466e+38f : f.l_val;
    const bool lvalid = resetL ? false : (f.l_valid != 0u);
    const bool act = lm < m;                                      // !(masked_to >= buf_mid)
    const bool inAL = lp < 0;
    const bool ltAL = t2 < lv;
    const bool riseAL = !ltAL && f_sub(t2, lv) > h;
    const bool gtBL = t2 > lv;
    const float valBL = gtBL ? t2 : lv;
    const i32 posBL = gtBL ? (i32) m : lp;
    const bool validBL = lvalid || (f_sub(valBL, t2) > h && valBL > thr2);
    const bool p2 = act && !inAL && validBL && (m - (u32) posBL) > 3u;
    const float nlv = inAL ? ((ltAL || riseAL) ? t2 : lv) : (p2 ? t2 : valBL);
    const i32 nlp = inAL ? (riseAL ? (i32) m : -1) : (p2 ? -1 : posBL);
    const bool nlvalid = !inAL && !p2 && validBL;
    f.l_masked = lm;
    f.l_val = act ? nlv : lv;
    f.l_pos = act ? nlp : lp;
    f.l_valid = (act ? nlvalid : lvalid) ? 1u : 0u;
    return p1 || p2;
}

// ---- exactly rounded divisions by the window lengths (W = 3 or 6)
// (the double operands are exact sums of floats: zero or >= 2^-149 in magnitude, far from underflow)
template <u32 W> UNC_DEV double k1_ddiv_w(double a) {
    const double r = W == 3u ? 0.33333333333333331 : 0.16666666666666666;   // RN(1/W)
    double q = d_mul(a, r);
    double e = d_fma(-(double) W, q, a);
    return d_fma(e, r, q);
}
// GUARD: operands below 2^-100 take the IEEE division (subnormal quotients can tie, where the
// sequence is not exact).  The window sums never need it: the fast path requires every non-zero
// sample to be >= 2^-38 (k1_exact_ok), so a non-zero float sum or sum of squares is >= 2^-99.
template <u32 W, bool GUARD> UNC_DEV float k1_fdiv_w(float a) {
    const float r = W == 3u ? 0.333333343f : 0.166666672f;                  // RN(1/W)
    if (GUARD && fabsf(a) < 7.8886090522101181e-31f) return f_div(a, (float) W);
    float q = f_mul(a, r);
    float e = f_fma(-(float) W, q, a);
    return f_fma(e, r, q);
}

// compute_tstat (reference src/event_detector.cpp:174-219) from the window sums:
// sum1/sumsq1 = left window (kept in double), sum2/sumsq2 = right window (rounded to float).
template <u32 W> UNC_DEV float k1_tstat(double sum1, double sumsq1, double sum2d, double sumsq2d) {
    float sum2 = (float) sum2d, sumsq2 = (float) sumsq2d;
    float mean1 = (float) k1_ddiv_w<W>(sum1);
    float mean2 = k1_fdiv_w<W, false>(sum2);
    float m1sq = f_mul(mean1, mean1), m2sq = f_mul(mean2, mean2);
    float q2 = k1_fdiv_w<W, false>(sumsq2);
    double cv = d_sub(d_add(d_sub(k1_ddiv_w<W>(sumsq1), (double) m1sq), (double) q2), (double) m2sq);
    float var = fmaxf((float) cv, 1.17549435e-38f);
    float delta = f_sub(mean2, mean1);
    return f_div(fabsf(delta), f_sqrt(k1_fdiv_w<W, true>(var)));
}

struct K1Read {                    // warp-uniform description of the read being processed
    const unsigned char *src;      // address of sample 0
    const unsigned char *buf_end;  // end of the batch's sample buffer (bulk copies never cross it)
    u32 n;                         // samples
    u32 n_pos;                     // FSM positions: m in [0, n_pos), n_pos = n >= 6 ? n - 5 : 0
    float cal_range, cal_offset, cal_digit, cal_inv;   // cal_inv != 0: digitisation is a power of two
    bool i16;                      // raw DAC input (calibrated on the fly) instead of f32 pA
};

struct K1Tile {
    i32 base_idx;                  // sample index of raw element 0
};

UNC_DEV float k1_sample(const K1WarpSmem *sm, const K1Read &R, const K1Tile &T, i32 j) {
    i32 e = j - T.base_idx;
    if (!R.i16) return sm->raw[e];
    u16 raw = ((const u16 *) sm->raw)[e];
    float v = f_mul(R.cal_range, f_add((float) raw, R.cal_offset));     // reference src/read_buffer.cpp:239-242
    return R.cal_inv != 0.0f ? f_mul(v, R.cal_inv) : f_div(v, R.cal_digit);
}

// exactness trackers: sum of |sample| and of the squares (float, only their magnitude matters) and
// the smallest non-zero bit patterns
struct K1Exact { float sum, sum2; u32 mn, mn2; };
UNC_DEV void k1_exact_add(K1Exact &x, float s, float ss) {
    u32 u = f2u(s) & 0x7FFFFFFFu, v = f2u(ss);
    x.sum = f_add(x.sum, fabsf(s)); x.sum2 = f_add(x.sum2, ss);
    x.mn = (u - 1u) < x.mn ? (u - 1u) : x.mn;          // u == 0 wraps to 0xFFFFFFFF: ignored
    x.mn2 = (v - 1u) < x.mn2 ? (v - 1u) : x.mn2;
}
// true when every partial sum of non-negative values with total `tot` and smallest non-zero bit
// pattern mn+1 is exactly representable in double: all values are multiples of 2^(emin-150) and
// every sum is < 2 * tot < 2^(etot-125)
UNC_DEV bool k1_exact_ok(float tot, u32 mn, i32 emin_floor) {
    if (mn == 0xFFFFFFFFu) return true;                   // all zero
    i32 etot = (i32) (f2u(tot) >> 23), emin = (i32) ((mn + 1u) >> 23);
    if (etot >= 254 || emin < emin_floor) return false;   // inf/nan (or a negative "sum"), or a value too small
    return etot + 2 <= 53 + emin - 23;
}

// ---- T pass: lane's chunk [a, a + K1_CH).  D3[j] = s[j]+s[j+1]+s[j+2] (and E3 for the float squares)
// are kept in three 3-deep register windows, one per residue class of the position: at position m
// the class window holds D3[m-6], D3[m-3], D3[m]; the step adds D3[m+3] and shifts.  Window sums
// (reference src/event_detector.cpp:195-205, differences of the double prefix sums -- exact here):
//   w=3: left D3[m-3], right D3[m];   w=6: left D3[m-6]+D3[m-3], right D3[m]+D3[m+3].
// FULL (the `events` kernels): *chunk_sq also receives the sum of the chunk's float squares.
template <bool FULL = false>
UNC_DEV void k1_tpass(K1WarpSmem *sm, const K1Read &R, const K1Tile &T, i32 a, int lane, double *chunk_sum, K1Exact &X,
                      double *chunk_sq = nullptr) {
    double D[3][3], E[3][3];
    double p2, p1, r2, r1;
    {
        double xd[11], qd[11];
#pragma unroll
        for (int t = 0; t < 11; t++) {
            i32 j = a - 6 + t;
            float s = j >= 0 ? k1_sample(sm, R, T, j) : 0.0f;
            float ss = f_mul(s, s);
            if (j >= 0 && (u32) j < R.n) k1_exact_add(X, s, ss);
            xd[t] = (double) s; qd[t] = (double) ss;
        }
#pragma unroll
        for (int t = 0; t < 9; t++) {
            D[t % 3][t / 3] = d_add(d_add(xd[t], xd[t + 1]), xd[t + 2]);
            E[t % 3][t / 3] = d_add(d_add(qd[t], qd[t + 1]), qd[t + 2]);
        }
        p2 = xd[9]; p1 = xd[10]; r2 = qd[9]; r1 = qd[10];
    }
    double acc = 0.0, acc2 = 0.0;
    float *row1 = sm->t1 + (u32) lane * K1_TS, *row2 = sm->t2 + (u32) lane * K1_TS;
#pragma unroll 1
    for (u32 i0 = 0; i0 < K1_CH; i0 += 3) {
#pragma unroll
        for (u32 c = 0; c < 3; c++) {
            const i32 m = a + (i32) (i0 + c);
            const i32 j = m + 5;
            float s = k1_sample(sm, R, T, j);
            float ss = f_mul(s, s);
            if ((u32) j < R.n) k1_exact_add(X, s, ss);
            double sd = (double) s, sq = (double) ss;
            const double dn = d_add(d_add(p2, p1), sd);      // D3[m+3]: samples m+3, m+4, m+5
            const double en = d_add(d_add(r2, r1), sq);
            p2 = p1; p1 = sd; r2 = r1; r1 = sq;
            float v1 = k1_tstat<3>(D[c][1], E[c][1], D[c][2], E[c][2]);
            float v2 = k1_tstat<6>(d_add(D[c][0], D[c][1]), d_add(E[c][0], E[c][1]), d_add(D[c][2], dn), d_add(E[c][2], en));
            if (c == 0) acc = d_add(acc, D[c][2]);           // samples m, m+1, m+2
            if (FULL && c == 0) acc2 = d_add(acc2, E[c][2]);
            D[c][0] = D[c][1]; D[c][1] = D[c][2]; D[c][2] = dn;
            E[c][0] = E[c][1]; E[c][1] = E[c][2]; E[c][2] = en;
            row1[i0 + c] = v1;
            row2[i0 + c] = v2;
        }
    }
    *chunk_sum = acc;
    if (FULL) *chunk_sq = acc2;
}

// t-statistics of the first positions, where the reference's ring indices wrap (u32 buf_mid - w
// for buf_mid < w reads the slot written last, src/event_detector.cpp:195-197) or the window is
// not yet full (t <= 2w -> 0, :185-187).  Tile 0, lane 0 only.
UNC_DEV void k1_fix_head(K1WarpSmem *sm, const K1Read &R, const K1Tile &T) {
    double P[10], Q[10];           // prefix sums P[j] = sum of samples < j, j = 0..9
    P[0] = 0.0; Q[0] = 0.0;
    for (int j = 0; j < 9; j++) {
        float s = (u32) j < R.n ? k1_sample(sm, R, T, j) : 0.0f;
        P[j + 1] = d_add(P[j], (double) s);
        Q[j + 1] = d_add(Q[j], (double) f_mul(s, s));
    }
    for (u32 m = 0; m < 3 && m < R.n_pos; m++) {
        // short window at buf_mid = m < 3: the "start" slot is the one holding P[m+6]
        sm->t1[m] = k1_tstat<3>(d_sub(P[m], P[m + 6]), d_sub(Q[m], Q[m + 6]), d_sub(P[m + 3], P[m]), d_sub(Q[m + 3], Q[m]));
    }
    for (u32 m = 0; m < 6 && m < R.n_pos; m++) sm->t2[m] = 0.0f;
    if (R.n_pos) sm->t1[0] = 0.0f;     // the short detector skips buf_mid == 0 (see k1_fsm_step)
}

// ---- FSM over positions [from, to) of the tile, reading the T rows; fire bits relative to `a`
UNC_DEV u64 k1_fsm_run(const K1WarpSmem *sm, K1Fsm &f, i32 a, int lane, u32 steps, const DevParams &p) {
    const float *row1 = sm->t1 + (u32) lane * K1_TS, *row2 = sm->t2 + (u32) lane * K1_TS;
    u64 fires = 0;
    for (u32 i = 0; i < steps; i++) {
        if (k1_fsm_step(f, row1[i], row2[i], (u32) a + i, p.threshold1, p.threshold2, p.peak_height)) fires |= 1ull << i;
    }
    return fires;
}

// entry i of a lane's fired-peak list (2 words: a double prefix sum, later a float mean): the lane's
// t2 row holds entries 0..17, its t1 row entries 18..35 (a chunk has at most K1_CH fires)
UNC_DEV u32 *k1_list(K1WarpSmem *sm, int lane, u32 i) {
    return i < K1_CH / 2u ? (u32 *) (sm->t2 + (u32) lane * K1_TS) + 2u * i : (u32 *) (sm->t1 + (u32) lane * K1_TS) + 2u * (i - K1_CH / 2u);
}

struct K1Carry {                   // warp-uniform state carried across the tiles of a read
    K1Fsm fsm;
    double base;                   // prefix sum of the samples before the tile's first position
    u32 evt_st; double evt_st_sum; // start of the open event and the prefix sum there
    u32 ne, total_events, len_total;
    K1Exact X;
};

// Where the FULL variant (the `events` kernels, unc_events.cuh) writes read r's events: slots row[r] .. of each array.
// The prefix sums of the float squares at the fired peaks go to a list of its own, `sql` (K1_CH entries of 2 words per
// lane), next to the prefix sums of the samples in the lane's T rows.
struct K1FullOut {
    const u64 *row;
    u32 *start;
    float *length, *mean, *stdv;
};
#define K1_SQL_WORDS (32u * 2u * K1_CH)   /* words of `sql` per warp */

// One read by one warp.  Returns false when the read must be redone by the serial routine.
// FULL: every event (start, length, mean, stdv: reference src/event_detector.cpp:296-319) goes to *fo instead of the
// mean to B.events.  The sums of squares are exact under the same condition as the sums (k1_exact_ok checks both), so
// the same flag sends a read to the serial routine.
template <bool FULL = false>
UNC_DEV bool k1_warp_read(const DevBatch &B, const DevParams &p, u32 r, K1WarpSmem *sm, u32 *bar_phase,
                          const K1FullOut *fo = nullptr, u32 *sql = nullptr) {
    u32 *stats = B.k1_stats;
    const int lane = w_lane();
    const DevReadDesc rd = B.reads[r];
    K1Read R;
    R.i16 = rd.dtype != 0u;
    const u32 esz = R.i16 ? 2u : 4u;
    R.src = (const unsigned char *) B.samples + (size_t) rd.offset * esz;
    R.buf_end = (const unsigned char *) B.samples + B.samples_bytes;
    R.n = rd.n_samples;
    R.n_pos = R.n >= 6u ? R.n - 5u : 0u;
    R.cal_range = rd.cal_range; R.cal_offset = rd.cal_offset; R.cal_digit = rd.cal_digit;
    R.cal_inv = 0.0f;
    if (R.i16) {
        u32 db = f2u(rd.cal_digit);
        // power of two in [2^-60, 2^60]: multiplying by the exact reciprocal equals the division
        if ((db & 0x807FFFFFu) == 0u && (db >> 23) > 67u && (db >> 23) < 187u) R.cal_inv = u2f((254u << 23) - db);
    }
    float *ev = B.events + (size_t) r * B.ev_stride;
    K1Carry C;
    C.fsm.s_pos = -1; C.fsm.s_val = 0.0f; C.fsm.s_valid = 0;          // state after the 5 window-filling steps
    C.fsm.l_masked = 0; C.fsm.l_pos = -1; C.fsm.l_val = 0.0f; C.fsm.l_valid = 0;
    C.base = 0.0; C.evt_st = 0; C.evt_st_sum = 0.0; C.ne = 0; C.total_events = 0; C.len_total = 0;
    C.X.sum = 0.0f; C.X.sum2 = 0.0f; C.X.mn = 0xFFFFFFFFu; C.X.mn2 = 0xFFFFFFFFu;
    double base2 = 0.0, evt_st_sq = 0.0;                           // FULL: the same two carries for the squares
    bool ok = R.n < (1u << 24);
    const u32 n_tiles = ok ? (R.n_pos + K1_TILE - 1u) / K1_TILE : 0u;

    for (u32 t = 0; t < n_tiles; t++) {
        const u32 lo = t * K1_TILE;
        // ---- bulk copy of samples [j0, j1) (tile + halo), from the 16-byte aligned address below j0
        const u32 j0 = lo >= K1_HALO ? lo - K1_HALO : 0u;
        u32 j1 = lo + K1_TILE + K1_HALO; if (j1 > R.n) j1 = R.n;
        const unsigned char *a0 = R.src + (size_t) j0 * esz;
        const unsigned char *al = (const unsigned char *) ((size_t) a0 & ~(size_t) 15);
        const u32 lead = (u32) (a0 - al);
        K1Tile T;
        T.base_idx = (i32) j0 - (i32) (lead / esz);
        u32 want = lead + (j1 - j0) * esz;                      // bytes from `al` that hold needed samples
        u32 bulk = (want + 15u) & ~15u;
        if (al + bulk > R.buf_end) bulk = (u32) ((R.buf_end - al) & ~(size_t) 15);   // never read past the buffer
        if (lane == 0) {
            t_fence_async();
            if (bulk) t_bulk_load(sm->raw, al, bulk, &sm->bar);
        }
        if (bulk < want) {                                      // tail of the buffer: plain 2-byte loads
            const u16 *g = (const u16 *) (al + bulk);
            u16 *s = (u16 *) ((unsigned char *) sm->raw + bulk);
            for (u32 i = (u32) lane; i < (want - bulk) / 2u; i += 32) s[i] = d_ldg(g + i);
        }
        if (bulk) { t_bar_wait(&sm->bar, *bar_phase); *bar_phase ^= 1u; }
        w_sync();

        // ---- T pass
        const i32 a = (i32) (lo + (u32) lane * K1_CH);
        const u32 steps = (u32) a >= R.n_pos ? 0u : (R.n_pos - (u32) a < K1_CH ? R.n_pos - (u32) a : K1_CH);
        double csum = 0.0, csq = 0.0;
        if (steps) k1_tpass<FULL>(sm, R, T, a, lane, &csum, C.X, &csq);
        w_sync();
        if (t == 0 && lane == 0) k1_fix_head(sm, R, T);
        w_sync();
        // exclusive scan of the chunk sums -> prefix sum at the lane's chunk start
        double incl = csum;
        for (int d = 1; d < 32; d <<= 1) {
            double y = u2d(w_shfl_up64(d2u(incl), d));
            if (lane >= d) incl = d_add(incl, y);
        }
        const double lane_base = d_add(C.base, d_sub(incl, csum));
        const double tile_sum = u2d(w_shfl64(d2u(incl), 31));
        double lane_base2 = 0.0, tile_sum2 = 0.0;
        if (FULL) {
            double incl2 = csq;
            for (int d = 1; d < 32; d <<= 1) {
                double y = u2d(w_shfl_up64(d2u(incl2), d));
                if (lane >= d) incl2 = d_add(incl2, y);
            }
            lane_base2 = d_add(base2, d_sub(incl2, csq));
            tile_sum2 = u2d(w_shfl64(d2u(incl2), 31));
        }

        // ---- speculative FSM
        K1Fsm sigma, phi;
        if (lane == 0) sigma = C.fsm;
        else {
            sigma.s_pos = -1; sigma.s_val = 3.402823466e+38f; sigma.s_valid = 0;
            sigma.l_masked = 0; sigma.l_pos = -1; sigma.l_val = 3.402823466e+38f; sigma.l_valid = 0;
            if (steps) {                                         // warm up over the tail of the previous lane's chunk
                const float *w1 = sm->t1 + (u32) (lane - 1) * K1_TS + (K1_CH - K1_WARM), *w2 = sm->t2 + (u32) (lane - 1) * K1_TS + (K1_CH - K1_WARM);
                for (u32 i = 0; i < K1_WARM; i++)
                    k1_fsm_step(sigma, w1[i], w2[i], (u32) a - K1_WARM + i, p.threshold1, p.threshold2, p.peak_height);
            }
        }
        phi = sigma;
        u64 fires = k1_fsm_run(sm, phi, a, lane, steps, p);
        for (;;) {
            K1Fsm prev = k1_fsm_shfl_up(phi);
            bool bad = lane > 0 && steps > 0 && !k1_fsm_eq(prev, sigma, (u32) a);
            u32 m_bad = w_ballot(bad);
            if (!m_bad) break;
            if (stats && lane == 0) { d_atomic_add(stats + 1, 1u); d_atomic_add(stats + 2, (u32) d_popc(m_bad)); }
            if (bad) { sigma = prev; phi = sigma; fires = k1_fsm_run(sm, phi, a, lane, steps, p); }
        }
        C.fsm = k1_fsm_bcast(phi, d_popc(w_ballot(steps > 0)) - 1);
        w_sync();

        // ---- fired peaks -> prefix sums at the event ends, overlaid on the lane's (now dead) T rows
        u32 cnt = 0;
        if (fires) {
            // P[a-2], P[a-1], P[a]: exact subtractions of the two samples before the chunk
            double q0 = lane_base, q1 = lane_base, q2 = lane_base;
            if (a >= 1) { q1 = d_sub(q0, (double) k1_sample(sm, R, T, a - 1)); q2 = q1; }
            if (a >= 2) q2 = d_sub(q1, (double) k1_sample(sm, R, T, a - 2));
            double g0 = lane_base2, g1 = lane_base2, g2 = lane_base2;      // FULL: the same for the squares
            if (FULL) {
                if (a >= 1) { float x = k1_sample(sm, R, T, a - 1); g1 = d_sub(g0, (double) f_mul(x, x)); g2 = g1; }
                if (a >= 2) { float x = k1_sample(sm, R, T, a - 2); g2 = d_sub(g1, (double) f_mul(x, x)); }
            }
            for (u32 i = 0; i < steps; i++) {
                if ((fires >> i) & 1ull) {                   // the event ends at buf_mid - w1 + 1 = m - 2 (:105)
                    u64 bits = d2u(q2);
                    u32 *e = k1_list(sm, lane, cnt);
                    e[0] = (u32) bits; e[1] = (u32) (bits >> 32);
                    if (FULL) {
                        u64 b2 = d2u(g2);
                        u32 *f = sql + (u32) lane * (2u * K1_CH) + 2u * cnt;
                        f[0] = (u32) b2; f[1] = (u32) (b2 >> 32);
                    }
                    cnt++;
                }
                q2 = q1; q1 = q0;
                q0 = d_add(q0, (double) k1_sample(sm, R, T, a + (i32) i));
                if (FULL) {
                    float x = k1_sample(sm, R, T, a + (i32) i);
                    g2 = g1; g1 = g0;
                    g0 = d_add(g0, (double) f_mul(x, x));
                }
            }
        }
        w_sync();
        // the raw tile is no longer needed: the next tile's copy may start (issued at the loop head)

        // ---- events: each fired peak closes the event opened by the previous one (create_event :296-319)
        // previous fire before this lane's first: nearest earlier lane with a fire, else the carry
        u32 lp = 0; u64 ls = 0, ls2 = 0;
        if (cnt) {
            lp = (u32) a + (u32) (63 - d_clzll(fires)) - 2u;
            const u32 *e = k1_list(sm, lane, cnt - 1);
            ls = (u64) e[1] << 32 | e[0];
            if (FULL) { const u32 *f = sql + (u32) lane * (2u * K1_CH) + 2u * (cnt - 1); ls2 = (u64) f[1] << 32 | f[0]; }
        }
        u32 has = cnt ? 1u : 0u;
        for (int d = 1; d < 32; d <<= 1) {                   // inclusive "last fire so far" scan
            u32 oh = w_shfl_up(has, d), op = w_shfl_up(lp, d); u64 os = w_shfl_up64(ls, d);
            u64 os2 = FULL ? w_shfl_up64(ls2, d) : 0ull;
            if (lane >= d && !has && oh) { has = 1u; lp = op; ls = os; if (FULL) ls2 = os2; }
        }
        u32 ph = w_shfl_up(has, 1), pp = w_shfl_up(lp, 1); u64 ps = w_shfl_up64(ls, 1);
        u32 st_pos = (lane > 0 && ph) ? pp : C.evt_st;
        double st_sum = (lane > 0 && ph) ? u2d(ps) : C.evt_st_sum;
        double st_sq = 0.0;
        if (FULL) { u64 ps2 = w_shfl_up64(ls2, 1); st_sq = (lane > 0 && ph) ? u2d(ps2) : evt_st_sq; }
        const u32 st_pos0 = st_pos;
        const double st_sum0 = st_sum;
        const u32 maxcnt = w_max(cnt);
        u32 nvalid = 0, len_acc = 0;
        u64 fl = fires;
        for (u32 i = 0; i < maxcnt; i++) {
            if (i < cnt) {
                u32 bit = (u32) d_ctzll(fl); fl &= fl - 1;
                u32 en = (u32) a + bit - 2u;
                const u32 *e = k1_list(sm, lane, i);
                double en_sum = u2d((u64) e[1] << 32 | e[0]);
                u32 length = en - st_pos;
                float mean = (float) d_div(d_sub(en_sum, st_sum), (double) length);
                len_acc += length;
                if (mean >= p.min_mean && mean <= p.max_mean) { if (!FULL) k1_list(sm, lane, nvalid)[0] = f2u(mean); nvalid++; }
                st_pos = en; st_sum = en_sum;
            }
        }
        u32 tot_valid, off = w_exscan(nvalid, &tot_valid);
        if (!FULL) {
            for (u32 i = 0; i < nvalid; i++) ev[C.ne + off + i] = u2f(k1_list(sm, lane, i)[0]);
        } else {                                             // the lane's events again, now that their slots are known
            u32 sp = st_pos0, k = C.ne + off;
            double ss = st_sum0, sq = st_sq;
            const u64 o = fo->row[r];
            u64 f2 = fires;
            for (u32 i = 0; i < cnt; i++) {
                u32 bit = (u32) d_ctzll(f2); f2 &= f2 - 1;
                u32 en = (u32) a + bit - 2u;
                const u32 *e = k1_list(sm, lane, i);
                const u32 *f = sql + (u32) lane * (2u * K1_CH) + 2u * i;
                double en_sum = u2d((u64) e[1] << 32 | e[0]), en_sq = u2d((u64) f[1] << 32 | f[0]);
                u32 length = en - sp;
                float mean = (float) d_div(d_sub(en_sum, ss), (double) length);
                if (mean >= p.min_mean && mean <= p.max_mean) {
                    // create_event (:307-313): deltasqr rounded to float, var in float, calibrate() = (v + 0) * 1
                    const float deltasqr = (float) d_sub(en_sq, sq);
                    const float var = f_sub(f_div(deltasqr, (float) length), f_mul(mean, mean));
                    fo->start[o + k] = sp;
                    fo->length[o + k] = (float) length;
                    fo->mean[o + k] = f_mul(f_add(mean, 0.0f), 1.0f);
                    fo->stdv[o + k] = f_mul(f_add(f_sqrt(fmaxf(var, 0.0f)), 0.0f), 1.0f);
                    k++;
                }
                sp = en; ss = en_sum; sq = en_sq;
            }
        }
        u32 tot_cnt, dummy = w_exscan(cnt, &tot_cnt); (void) dummy;
        u32 tot_len; dummy = w_exscan(len_acc, &tot_len);
        // carry
        u32 fh = w_shfl(has, 31), fp = w_shfl(lp, 31); u64 fs = w_shfl64(ls, 31);
        if (fh) { C.evt_st = fp; C.evt_st_sum = u2d(fs); }
        if (FULL) {
            u64 fs2 = w_shfl64(ls2, 31);
            if (fh) evt_st_sq = u2d(fs2);
            base2 = d_add(base2, tile_sum2);
        }
        C.ne += tot_valid; C.total_events += tot_cnt; C.len_total += tot_len;
        C.base = d_add(C.base, tile_sum);
        w_sync();
    }
    // exactness of the whole read
    {
        float tot = C.X.sum, tot2 = C.X.sum2;
        for (int d = 16; d > 0; d >>= 1) { tot = f_add(tot, w_shflf(tot, lane ^ d)); tot2 = f_add(tot2, w_shflf(tot2, lane ^ d)); }
        u32 mn = ~w_max(~C.X.mn), mn2 = ~w_max(~C.X.mn2);
        ok = ok && k1_exact_ok(tot, mn, 127 - 38) && k1_exact_ok(tot2, mn2, 127 - 76);
    }
    if (lane == 0) {
        B.n_events[r] = C.ne;
        // len_sum_ is a float sum of integer lengths < 2^24: exact, equal to the integer total
        B.mean_event_len[r] = f_div((float) C.len_total, (float) C.total_events);
        B.k1_flags[r] = ok ? 0u : 1u;
        if (stats) { d_atomic_add(stats + 0, n_tiles); if (!ok) d_atomic_add(stats + 3, 1u); }
    }
    return ok;
}

// The offline Normalizer's scale and shift for ne > 0 means towards (tgt_mean, tgt_stdv) (reference
// src/normalizer.cpp:31-44 + :114-118): sequential double reductions.
UNC_DEV void unc_norm_scale_shift(const float *ev, u32 ne, float tgt_mean, float tgt_stdv, float *scale, float *shift) {
    double mean = 0.0;
    for (u32 i = 0; i < ne; i++) mean = d_add(mean, (double) ev[i]);
    mean = d_div(mean, (double) ne);
    double varsum = 0.0;
    for (u32 i = 0; i < ne; i++) {
        double d = d_sub((double) ev[i], mean);
        varsum = d_add(varsum, d_mul(d, d));
    }
    *scale = (float) d_div((double) tgt_stdv, d_sqrt(d_div(varsum, (double) ne)));
    *shift = (float) d_sub((double) tgt_mean, d_mul((double) *scale, mean));
}

// Normaliser statistics of one read by one thread, towards the model's global mean and stdv.
UNC_DEV void unc_k1_norm_read(const DevBatch &B, const DevParams &p, u32 r) {
    const float *ev = B.events + (size_t) r * B.ev_stride;
    const u32 ne = B.n_events[r];
    float scale = 0.0f, shift = 0.0f;
    if (ne > 0) {
        unc_norm_scale_shift(ev, ne, p.tgt_mean, p.tgt_stdv, &scale, &shift);
        if (B.normed) {
            float *nm = B.normed + (size_t) r * B.ev_stride;
            for (u32 i = 0; i < ne; i++) nm[i] = f_add(f_mul(scale, ev[i]), shift);
        }
    }
    B.scale[r] = scale;
    B.shift[r] = shift;
}

// Warp body of the k1_events kernel (and, FULL, of k_events_warp): reads are pulled from an atomic queue.
template <bool FULL = false>
UNC_DEV void unc_k1_warp_main(const DevBatch &B, const DevParams &p, K1WarpSmem *sm, const K1FullOut *fo = nullptr,
                              u32 *sql = nullptr) {
    const int lane = w_lane();
    if (lane == 0) t_bar_init(&sm->bar);
    w_sync();
    u32 phase = 0;
    for (;;) {
        u32 r = 0;
        if (lane == 0) r = d_atomic_add(B.k1_queue, 1u);
        r = w_shfl(r, 0);
        if (r >= B.n_reads) break;
        k1_warp_read<FULL>(B, p, r, sm, &phase, fo, sql);
    }
}
