// unc_dtw_band.cuh -- the banded DTW sweep: the recurrence of src/dtw.hpp:51-120 (DTWSubSeq::NONE only) restricted to a band
// of rows around the matrix's diagonal, for reads whose full rows x columns matrix does not fit or is not worth filling.
//
// Problem: R rows (k-mers) x C columns (event means), band half-width W >= 1 in rows.
//   centre of column j    c(j) = floor(j (R-1) / (C-1)) for C > 1 (64-bit), 0 for C = 1
//   effective half-width  We = max(W, ceil((R-1) / (C-1))) for C > 1, R - 1 for C = 1, so that lo(j) <= hi(j-1) + 1: every
//                         in-band cell is reachable from (0, 0) through in-band cells, and (R-1, C-1) is in the band
//   column j holds rows   lo(j) = max(0, c(j) - We) .. hi(j) = min(R-1, c(j) + We)
// An in-band cell is computed with the reference's float operations in its order (unc_dtw_cost; score + weight * cost; D
// before H before V).  A predecessor outside the band reads MAX_COST, as one outside the matrix does in the reference.  The
// traceback is the reference's loop; by the reachability above it never leaves the band (emulator builds assert it).
// We >= R - 1 makes the band the whole matrix, and the sweep is then bit-identical to k_dtw's.
//
// k_dtw_band: one persistent CTA per problem (problems from a queue).  It sweeps the 8 x 8 tiles of unc_dtw.cuh by tile
// anti-diagonal, one barrier per diagonal, but only the tiles that intersect the band: a contiguous run of tile rows on every
// diagonal, tracked by two indices that only move forward.  Stored: one breadcrumb byte per in-band cell, column-major, at
// off(j) + (i - lo(j)), where off is the 64-bit prefix sum of the band heights (unc_band_offsets, computed on the host, which
// plans the workspace from it); the work arrays hrow (C floats), vcol (R floats) and corners are k_dtw's.  Nothing is
// rows x columns.
#pragma once
#include "unc_dtw.cuh"

#ifndef UNC_HD
#ifdef __CUDACC__
#define UNC_HD __host__ __device__
#else
#define UNC_HD
#endif
#endif

// Column geometry of one banded problem.  Columns are stepped without a division: c(j) = j q + floor(j r / den).
struct UncBand {
    u32 R, C, we;            // rows, columns, effective half-width (capped at R - 1, which leaves the band unchanged)
    u32 q, r, den;           // R - 1 = q den + r, den = max(C - 1, 1)
};
struct UncBandCol {
    u32 c, rem;              // c(j) and (j (R-1)) mod den
};

UNC_HD inline UncBand unc_band_make(u32 R, u32 C, u32 W) {
    UncBand b;
    b.R = R; b.C = C;
    b.den = C > 1u ? C - 1u : 1u;
    b.q = C > 1u ? (R - 1u) / b.den : 0u;
    b.r = C > 1u ? (R - 1u) % b.den : 0u;
    u64 we = C > 1u ? ((u64) R - 1u + b.den - 1u) / b.den : (u64) R - 1u;     // ceil((R-1) / (C-1))
    if ((u64) W > we) we = W;
    b.we = (u32) (we < (u64) R - 1u ? we : (u64) R - 1u);
    return b;
}
UNC_HD inline UncBandCol unc_band_col(const UncBand &b, u32 j) {
    const u64 n = (u64) j * (b.R - 1u);
    UncBandCol k;
    k.c = (u32) (n / b.den); k.rem = (u32) (n % b.den);
    return k;
}
UNC_HD inline void unc_band_next(const UncBand &b, UncBandCol &k) {
    k.c += b.q; k.rem += b.r;
    if (k.rem >= b.den) { k.rem -= b.den; k.c++; }
}
UNC_HD inline void unc_band_prev(const UncBand &b, UncBandCol &k) {
    k.c -= b.q;
    if (k.rem < b.r) { k.rem += b.den; k.c--; }
    k.rem -= b.r;
}
UNC_HD inline u32 unc_band_lo(const UncBand &b, const UncBandCol &k) { return k.c > b.we ? k.c - b.we : 0u; }
UNC_HD inline u32 unc_band_hi(const UncBand &b, const UncBandCol &k) { return k.c + b.we < b.R - 1u ? k.c + b.we : b.R - 1u; }

// off[0..C] (optional): the breadcrumb offset of each column's first in-band cell, and the number of in-band cells last.
inline u64 unc_band_offsets(const UncBand &b, u64 *off) {
    UncBandCol k = {0u, 0u};
    u64 s = 0;
    for (u32 j = 0; j < b.C; j++) {
        if (off) off[j] = s;
        s += (u64) unc_band_hi(b, k) - unc_band_lo(b, k) + 1u;
        unc_band_next(b, k);
    }
    if (off) off[b.C] = s;
    return s;
}

struct DevDtwBand {
    DevDtw D;                // problems, inputs, outputs and work arrays as k_dtw takes them; D.subseq is 0, D.edge unused
    const u64 *col_off;      // problem p: its C + 1 band offsets at D.prob[p].edge_off
    u32 band;                // W
};

// the band's tile rows in tile column tb: [lo of its first column, hi of its last column] / T
UNC_DEV u32 unc_band_tile_lo(const UncBand &b, u32 tb) { return unc_band_lo(b, unc_band_col(b, tb * UNC_DTW_T)) / UNC_DTW_T; }
UNC_DEV u32 unc_band_tile_hi(const UncBand &b, u32 tb) {
    const u32 j = tb * UNC_DTW_T + UNC_DTW_T - 1u;
    return unc_band_hi(b, unc_band_col(b, j < b.C ? j : b.C - 1u)) / UNC_DTW_T;
}

UNC_DEV void unc_dtw_band_problem(const DevDtwBand &B, u32 pi) {
    const DevDtw &D = B.D;
    const DevDtwProblem P = D.prob[pi];
    const u32 R = P.n_rows, Cn = P.n_cols;
    const UncBand bd = unc_band_make(R, Cn, B.band);
    const u32 tid = (u32) c_tid(), nt = (u32) c_nthreads();
    const float *means = D.means + P.mean_off;
    const u16 *kmers = D.kmers + P.kmer_off;
    unsigned char *bc = D.bc + P.bc_off;
    const u64 *off = B.col_off + P.edge_off;
    const u32 T = UNC_DTW_T, tr = (R + T - 1u) / T, tc = (Cn + T - 1u) / T;
    float *hrow = D.diag + P.diag_off, *vcol = hrow + Cn, *corner = vcol + R;
    const float dw = D.dw, hw = D.hw, vw = D.vw, MAXC = UNC_DTW_MAX_COST;
    u32 a1 = 0, a2 = 0;                                       // the band's tile rows on tile diagonal td: a1 .. a2
    for (u32 td = 0; td + 1u < tr + tc; td++) {
        const u32 a_lo = td >= tc ? td - (tc - 1u) : 0u, a_hi = td < tr ? td : tr - 1u;
        if (a1 < a_lo) a1 = a_lo;
        while (a1 <= a_hi && a1 < unc_band_tile_lo(bd, td - a1)) a1++;
        if (a2 < a_lo) a2 = a_lo;
        while (a2 < a_hi && a2 + 1u <= unc_band_tile_hi(bd, td - a2 - 1u)) a2++;
        for (u32 a = a1 + tid; a <= a2; a += nt) {
            const u32 b = td - a, i0 = a * T, j0 = b * T;
            const u32 pn = R - i0 < T ? R - i0 : T, qn = Cn - j0 < T ? Cn - j0 : T;
            // rows lo .. hi of columns j0 - 1 .. j0 + T - 1 (index q + 1), and each column's breadcrumb base off(j) - lo(j)
            u32 lo[UNC_DTW_T + 1], hi[UNC_DTW_T + 1];
            u64 base[UNC_DTW_T];
            UncBandCol k = unc_band_col(bd, j0);
            if (j0 > 0) {
                UncBandCol kp = k;
                unc_band_prev(bd, kp);
                lo[0] = unc_band_lo(bd, kp); hi[0] = unc_band_hi(bd, kp);
            } else {
                lo[0] = 1u; hi[0] = 0u;                       // no column to the left: nothing in band there
            }
#pragma unroll
            for (u32 q = 0; q < UNC_DTW_T; q++) {
                lo[q + 1] = unc_band_lo(bd, k); hi[q + 1] = unc_band_hi(bd, k);
                base[q] = q < qn ? off[j0 + q] - lo[q + 1] : 0u;
                unc_band_next(bd, k);
            }
            float prow[UNC_DTW_T + 1], ev[UNC_DTW_T];
            // the row above the tile, columns j0 - 1 .. j0 + T - 1: its in-band cells from the tiles above, MAX_COST elsewhere
            prow[0] = (i0 > 0 && lo[0] <= i0 - 1u && i0 - 1u <= hi[0]) ? corner[((td + 1u) % 3u) * tr + (a - 1u)] : MAXC;
#pragma unroll
            for (u32 q = 0; q < UNC_DTW_T; q++) {
                prow[q + 1] = (q < qn && i0 > 0 && lo[q + 1] <= i0 - 1u && i0 - 1u <= hi[q + 1]) ? hrow[j0 + q] : MAXC;
                ev[q] = q < qn ? means[j0 + q] : 0.0f;
            }
#pragma unroll 1
            for (u32 p = 0; p < pn; p++) {
                const u32 i = i0 + p;
                const u32 kmer = kmers[i];
                float left = (lo[0] <= i && i <= hi[0]) ? vcol[i] : MAXC;                      // cell (i, j0 - 1)
                float diag = prow[0];                                                           // cell (i - 1, j0 - 1)
                prow[0] = left;
#pragma unroll
                for (u32 q = 0; q < UNC_DTW_T; q++) {
                    if (q < qn) {
                        const u32 j = j0 + q;
                        const float up = prow[q + 1];                                           // cell (i - 1, j)
                        float v = MAXC;
                        if (lo[q + 1] <= i && i <= hi[q + 1]) {
                            const float cost = unc_dtw_cost(D, kmer, ev[q]);
                            float dsc, hsc, vsc;                                                // dscore / hscore / vscore :153-173
                            if (j > 0 && i > 0) dsc = diag;
                            else dsc = j == i ? 0.0f : MAXC;
                            hsc = j > 0 ? left : MAXC;
                            vsc = i > 0 ? up : MAXC;
                            const float ds = f_add(dsc, f_mul(dw, cost)), hs = f_add(hsc, f_mul(hw, cost)), vs = f_add(vsc, f_mul(vw, cost));
                            unsigned char mv;
                            if (ds <= hs && ds <= vs) { v = ds; mv = 0; }                      // Move::D
                            else if (hs <= vs) { v = hs; mv = 1; }                             // Move::H
                            else { v = vs; mv = 2; }                                           // Move::V
                            bc[base[q] + i] = mv;
                            if (i == R - 1u && j == Cn - 1u) D.score[pi] = v;
                        }
                        diag = up;
                        prow[q + 1] = v;
                        left = v;
                    }
                }
                vcol[i] = left;                                                                 // cell (i, last column of the tile)
            }
#pragma unroll
            for (u32 q = 0; q < UNC_DTW_T; q++) if (q < qn) hrow[j0 + q] = prow[q + 1];
            corner[(td % 3u) * tr + a] = prow[UNC_DTW_T];
        }
        c_sync();
    }
    if (tid == 0) {                                                                  // traceback :76-122, subseq NONE
        u32 i = R - 1u, j = Cn - 1u;
        UncBandCol k = unc_band_col(bd, j);
        u64 *path = D.path + 2 * P.path_off;
        path[0] = j; path[1] = i;
        u64 n = 1;
        while (i != 0 || j != 0) {
            const u32 lo = unc_band_lo(bd, k);
#ifdef UNC_EMUL
            if (i < lo || i > unc_band_hi(bd, k)) { fprintf(stderr, "banded traceback left the band at (%u, %u)\n", i, j); abort(); }
#endif
            const unsigned char mv = bc[off[j] + (i - lo)];
            if (i == 0 || mv == 1) { j--; unc_band_prev(bd, k); }
            else if (j == 0 || mv == 2) i--;
            else { i--; j--; unc_band_prev(bd, k); }
            path[2 * n] = j; path[2 * n + 1] = i; n++;
        }
        D.path_len[pi] = n;
    }
    c_sync();
}
