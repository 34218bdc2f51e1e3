// Dynamic time warping of a read's event means against a stretch of reference k-mers (SURVEY section 8(f) rank 4).
// Reference: src/dtw.hpp -- DTW<float, u16, Func> :31-183 (rows = k-mers, columns = event means; compute_matrix :49-74,
// traceback :76-122, boundary scores :153-173), the two bound instances DTWr94p :188-209 (cost = -match_prob of the TEMPLATE
// r9.4 model) and DTWr94d :212-232 (cost = abs(e - mean_k), which binds to int abs(int): the difference is truncated first),
// src/pybinder.cpp:75-91.
//
// One CTA per problem, a sweep over the anti-diagonals of the matrix cut into 8 x 8 TILES: a thread computes a whole tile (64
// cells in registers, row by row) from the bottom row of the tile above (`hrow`, one value per column), the right column of the
// tile to its left (`vcol`, one value per row) and the corner cell between them (three rotating generations per tile row, so
// that the tiles of one diagonal never write what another tile of the diagonal still reads); one barrier per TILE diagonal.
// Every cell is computed with the reference's float operations in the reference's order (score + weight * cost; D if
// ds <= hs && ds <= vs, else H if hs <= vs, else V), so the matrix is bit-identical whatever the evaluation order.  Stored: one
// breadcrumb byte per cell and the matrix's last column and last row (all the traceback reads of the matrix itself).  The
// traceback is the reference's loop, run by one thread.
#pragma once

struct DevDtwProblem {
    u64 mean_off, kmer_off;   // into means / kmers
    u64 bc_off;               // breadcrumbs, n_rows x n_cols bytes, row-major
    u64 diag_off;             // UNC_DTW_WORK_FLOATS(n_rows, n_cols) floats: hrow, vcol, corners
    u64 edge_off;             // last column (n_rows floats), then last row (n_cols floats)
    u64 path_off;             // in (column, row) pairs; room for n_rows + n_cols of them
    u32 n_cols, n_rows;
};
struct DevDtw {
    const float *model;       // template model: lv_mean[1024], lv_var2[1024], lognorm[1024]
    const float *means;
    const u16 *kmers;
    const DevDtwProblem *prob;
    u32 n_prob;
    unsigned char *bc;
    float *diag, *edge;
    u64 *path, *path_len;
    float *score;
    int cost_kind, subseq;    // 0 DTWr94p / 1 DTWr94d / 2 DTWr94d with float abs (the dtw_test driver); DTWSubSeq 0 NONE, 1 ROW, 2 COL
    float dw, hw, vw;
    u32 *queue;
};

#define UNC_DTW_T 8u                                  /* tile edge */
#define UNC_DTW_WORK_FLOATS(nr, nc) ((nc) + (nr) + 3u * (((nr) + UNC_DTW_T - 1u) / UNC_DTW_T) + 8u)
#define UNC_DTW_MAX_COST (3.402823466e+38f / 2.0f)   /* FLT_MAX / 2.0 (src/dtw.hpp:145) */

UNC_DEV float unc_dtw_cost(const DevDtw &D, u32 kmer, float e) {
    if (D.cost_kind == 0) return -unc_match_prob(e, D.model[kmer], D.model[1024 + kmer], D.model[2048 + kmer]);
    if (D.cost_kind == 2) return fabsf(f_sub(e, D.model[kmer]));   // DTWr94d as dtw_test.cpp compiles it: float abs
    const int t = (int) f_sub(e, D.model[kmer]);          // int abs(int): truncation towards zero first
    return (float) (t < 0 ? -t : t);
}

UNC_DEV void unc_dtw_problem(const DevDtw &D, u32 pi) {
    const DevDtwProblem P = D.prob[pi];
    const u32 R = P.n_rows, Cn = P.n_cols;
    const u32 tid = (u32) c_tid(), nt = (u32) c_nthreads();
    const float *means = D.means + P.mean_off;
    const u16 *kmers = D.kmers + P.kmer_off;
    unsigned char *bc = D.bc + P.bc_off;
    const u32 T = UNC_DTW_T, tr = (R + T - 1u) / T, tc = (Cn + T - 1u) / T;     // tile rows / columns
    float *hrow = D.diag + P.diag_off, *vcol = hrow + Cn, *corner = vcol + R;    // corner[g * tr + a], g = tile diagonal % 3
    float *lastcol = D.edge + P.edge_off, *lastrow = lastcol + R;
    const int sub = D.subseq;
    const float dw = D.dw, hw = D.hw, vw = D.vw;
    for (u32 td = 0; td + 1u < tr + tc; td++) {
        const u32 a_lo = td >= tc ? td - (tc - 1u) : 0u, a_hi = td < tr ? td : tr - 1u;
        for (u32 a = a_lo + tid; a <= a_hi; a += nt) {
            const u32 b = td - a, i0 = a * T, j0 = b * T;
            const u32 pn = R - i0 < T ? R - i0 : T, qn = Cn - j0 < T ? Cn - j0 : T;          // valid rows / columns of the tile
            float prow[UNC_DTW_T + 1], ev[UNC_DTW_T];
            // the row above the tile: columns j0 - 1 .. j0 + T - 1 (values that are never read stay 0)
            prow[0] = (a > 0 && b > 0) ? corner[((td + 1u) % 3u) * tr + (a - 1u)] : 0.0f;
#pragma unroll
            for (u32 q = 0; q < UNC_DTW_T; q++) {
                prow[q + 1] = (a > 0 && q < qn) ? hrow[j0 + q] : 0.0f;
                ev[q] = q < qn ? means[j0 + q] : 0.0f;
            }
#pragma unroll 1
            for (u32 p = 0; p < pn; p++) {
                const u32 i = i0 + p;
                const u32 kmer = kmers[i];
                float left = b > 0 ? vcol[i] : 0.0f;                                          // cell (i, j0 - 1)
                float diag = prow[0];                                                         // cell (i - 1, j0 - 1)
                prow[0] = left;
#pragma unroll
                for (u32 q = 0; q < UNC_DTW_T; q++) {
                    if (q < qn) {
                        const u32 j = j0 + q;
                        const float cost = unc_dtw_cost(D, kmer, ev[q]);
                        float dsc, hsc, vsc;                                                  // dscore / hscore / vscore :153-173
                        if (j > 0 && i > 0) dsc = diag;
                        else if (j == i || (i == 0 && sub == 2) || (j == 0 && sub == 1)) dsc = 0.0f;
                        else dsc = UNC_DTW_MAX_COST;
                        if (j > 0) hsc = left;
                        else hsc = sub == 1 ? 0.0f : UNC_DTW_MAX_COST;
                        const float up = prow[q + 1];                                         // cell (i - 1, j)
                        if (i > 0) vsc = up;
                        else vsc = sub == 2 ? 0.0f : UNC_DTW_MAX_COST;
                        const float ds = f_add(dsc, f_mul(dw, cost)), hs = f_add(hsc, f_mul(hw, cost)), vs = f_add(vsc, f_mul(vw, cost));
                        float v; unsigned char mv;
                        if (ds <= hs && ds <= vs) { v = ds; mv = 0; }                        // Move::D
                        else if (hs <= vs) { v = hs; mv = 1; }                               // Move::H
                        else { v = vs; mv = 2; }                                             // Move::V
                        bc[(u64) i * Cn + j] = mv;
                        if (j == Cn - 1u) lastcol[i] = v;
                        if (i == R - 1u) lastrow[j] = v;
                        diag = up;
                        prow[q + 1] = v;
                        left = v;
                    }
                }
                vcol[i] = left;                                                               // cell (i, last column of the tile)
            }
#pragma unroll
            for (u32 q = 0; q < UNC_DTW_T; q++) if (q < qn) hrow[j0 + q] = prow[q + 1];      // the tile's bottom row
            corner[(td % 3u) * tr + a] = prow[UNC_DTW_T];                                     // its bottom-right cell (read only if the tile is full)
        }
        c_sync();
    }
    if (tid == 0) {                                                                  // traceback :76-122
        u64 i = R - 1u, j = Cn - 1u;
        if (sub == 1) { for (u64 q = 0; q < R; q++) if (lastcol[q] < lastcol[i]) i = q; }
        else if (sub == 2) { for (u64 q = 0; q < Cn; q++) if (lastrow[q] < lastrow[j]) j = q; }
        D.score[pi] = sub == 2 ? lastrow[j] : lastcol[i];
        u64 *path = D.path + 2 * P.path_off;
        u64 n = 0;
        path[0] = j; path[1] = i; n = 1;
        u64 k = i * Cn + j;
        while (!(i == 0 || sub == 1) || !(j == 0 || sub == 2)) {
            const unsigned char mv = bc[k];
            if (i == 0 || mv == 1) { k--; j--; }
            else if (j == 0 || mv == 2) { k -= Cn; i--; }
            else { k -= (u64) Cn + 1u; i--; j--; }
            path[2 * n] = j; path[2 * n + 1] = i; n++;
        }
        D.path_len[pi] = n;
    }
    c_sync();
}
