/* oracle/unc_oracle_dtw_band.c -- CPU restatement of the banded DTW sweep (uncalled_b200/csrc/unc_dtw_band.cuh): the
 * recurrence of the reference's DTW (src/dtw.hpp:51-120, boundary scores :153-173) restricted to a band of rows, as plain
 * nested loops over the band.  TEST INFRASTRUCTURE ONLY, like unc_oracle.c, whose match_prob it calls: built by
 * oracle/dtw_band.mk into libunc_oracle_dtw_band.so, linked against libunc_oracle.so.
 *
 * R rows (k-mers) x C columns (means), half-width W >= 1:
 *   c(j) = floor(j (R-1) / (C-1)) (64-bit) for C > 1, 0 for C = 1
 *   We   = max(W, ceil((R-1) / (C-1))) for C > 1, R - 1 for C = 1
 *   column j holds rows lo(j) = max(0, c(j) - We) .. hi(j) = min(R-1, c(j) + We)
 * In-band cells: the reference's float operations in its order; a predecessor outside the band scores FLT_MAX / 2, as
 * one outside the matrix.  Global alignment only.  Breadcrumbs column-major, column j at off(j) = the heights of the
 * columns before it. */
#include "unc_oracle.h"

#include <float.h>
#include <math.h>
#include <stdlib.h>

typedef uint8_t u8;
typedef uint64_t u64;

#define MAX_COST (FLT_MAX / 2.0f)

static void band_rows(u64 R, u64 C, u64 we, u64 j, u64 *lo, u64 *hi) {
    const u64 c = C > 1 ? j * (R - 1) / (C - 1) : 0;
    *lo = c > we ? c - we : 0;
    *hi = c + we < R - 1 ? c + we : R - 1;
}

/* cost_kind 0 DTWr94p (-match_prob of the template model), 1 DTWr94d with int abs (the library's bindings), 2 DTWr94d with
 * float abs (the dtw_test driver).  Path pairs (column, row) from the end cell back to (0, 0).  bc (optional): the in-band
 * breadcrumbs, *n_cells (optional) their number.  Returns 0, -1 for an empty problem, -2 out of memory, -3 for subseq != 0,
 * band == 0 or an unknown cost kind. */
int orc_dtw_banded(const orc_model *tmpl, int cost_kind, int subseq, float dw, float hw, float vw, const float *means,
                   uint32_t n_cols, const uint16_t *kmers, uint32_t n_rows, uint32_t band, uint64_t *path, uint64_t *path_len,
                   float *score, uint8_t *bc_out, uint64_t *n_cells) {
    const u64 R = n_rows, C = n_cols;
    if (R == 0 || C == 0) return -1;
    if (subseq != 0 || band == 0 || cost_kind < 0 || cost_kind > 2) return -3;
    u64 we = C > 1 ? (R - 1 + C - 2) / (C - 1) : R - 1;
    if (C > 1 && band > we) we = band;
    u64 *off = (u64 *) malloc((C + 1) * sizeof(u64));
    if (!off) return -2;
    off[0] = 0;
    for (u64 j = 0; j < C; j++) {
        u64 lo, hi;
        band_rows(R, C, we, j, &lo, &hi);
        off[j + 1] = off[j] + (hi - lo + 1);
    }
    float *val = (float *) malloc(off[C] * sizeof(float));
    u8 *bc = (u8 *) malloc(off[C]);
    if (!val || !bc) { free(off); free(val); free(bc); return -2; }
    u64 plo = 1, phi = 0;                            /* the previous column's rows (none before column 0) */
    for (u64 j = 0; j < C; j++) {
        u64 lo, hi;
        band_rows(R, C, we, j, &lo, &hi);
        for (u64 i = lo; i <= hi; i++) {
            const float e = means[j], lv = tmpl->lv_mean[kmers[i]];
            float cost;
            if (cost_kind == 0) cost = -orc_match_prob(tmpl, e, kmers[i]);
            else if (cost_kind == 1) cost = (float) abs((int) (e - lv));
            else cost = fabsf(e - lv);
            float dsc, hsc, vsc;
            if (j > 0 && i > 0) dsc = (i - 1 >= plo && i - 1 <= phi) ? val[off[j - 1] + (i - 1 - plo)] : MAX_COST;
            else dsc = j == i ? 0 : MAX_COST;
            if (j > 0) hsc = (i >= plo && i <= phi) ? val[off[j - 1] + (i - plo)] : MAX_COST;
            else hsc = MAX_COST;
            if (i > 0) vsc = i - 1 >= lo ? val[off[j] + (i - 1 - lo)] : MAX_COST;
            else vsc = MAX_COST;
            const float ds = dsc + (dw * cost), hs = hsc + (hw * cost), vs = vsc + (vw * cost);
            const u64 k = off[j] + (i - lo);
            if (ds <= hs && ds <= vs) { val[k] = ds; bc[k] = 0; }       /* Move::D */
            else if (hs <= vs) { val[k] = hs; bc[k] = 1; }              /* Move::H */
            else { val[k] = vs; bc[k] = 2; }                            /* Move::V */
        }
        plo = lo; phi = hi;
    }
    u64 i = R - 1, j = C - 1, n = 0;
    *score = val[off[C] - 1];
    path[2 * n] = j; path[2 * n + 1] = i; n++;
    int rc = 0;
    while (i != 0 || j != 0) {
        u64 lo, hi;
        band_rows(R, C, we, j, &lo, &hi);
        if (i < lo || i > hi) { rc = -4; break; }      /* never: every in-band cell is reachable through the band */
        const u8 mv = bc[off[j] + (i - lo)];
        if (i == 0 || mv == 1) j--;
        else if (j == 0 || mv == 2) i--;
        else { i--; j--; }
        path[2 * n] = j; path[2 * n + 1] = i; n++;
    }
    *path_len = n;
    if (n_cells) *n_cells = off[C];
    if (bc_out) for (u64 k = 0; k < off[C]; k++) bc_out[k] = bc[k];
    free(off);
    free(val);
    free(bc);
    return rc;
}
