// unc_selfalign.cuh -- device half of `self_align` (reference src/self_align_ref.cpp:34-91), the input of
// `uncalled index`'s parameter search: for each sampled reference position, the FM range lengths of the
// backward search that walks forward along the reference with complemented bases until the range is unique.
//
// One thread per sampled path.  A step is two dependent Occ lookups at unrelated rows of the BWT (the
// paths start at random positions), i.e. two 64-byte sectors from HBM/L2 per step and nothing to share
// between threads: the kernel is latency-bound, and what matters is the number of paths in flight
// (small state per thread -> full occupancy) and not doing the walk twice.  Pass 1 counts every path and
// parks its first UNC_SA_STAGE lengths in a transposed staging array (value j of path i at j*n + i, so a
// warp's stores coalesce); pass 2, after the host's prefix sum of the counts, copies the parked values to
// their CSR places and re-walks only paths longer than the stage (repeats).
//
// `find-repeats` (reference src/find_repeats.cpp:61-85) runs the same walk from EVERY position and keeps only its
// number of steps (unc_repeat_length, mode UNC_SA_STEPS): no per-position arrays, one u32 out per position.
#pragma once
#include "unc_device.cuh"

#define UNC_SA_STAGE 48u

struct DevSelfAlign {
    const u8 *pac;          // 2-bit packed forward reference as in the .pac file (reference src/bwa_index.hpp:141-147)
    const u32 *pos, *lim;   // per path: first base / end of its sequence, as .pac positions
    u32 n;
    u32 *count;             // out (pass 1): number of range lengths of path i
    u32 *stage;             // out (pass 1): [UNC_SA_STAGE][n]
    const u64 *offsets;     // in (pass 2): CSR offsets, n + 1
    u64 *values;            // out (pass 2)
};

// what unc_selfalign_walk does with the range lengths
#define UNC_SA_PARK 0       // the first UNC_SA_STAGE go to park[j * n]; returns the number of lengths (pass 1)
#define UNC_SA_WRITE 1      // every length goes to out[j]; returns the number of lengths (pass 2)
#define UNC_SA_STEPS 2      // none is stored; returns the number of get_neighbor steps (find-repeats)

// find-repeats over the .pac window [pac_st, pac_st + n): out[i] = steps of the walk from pac_st + i, which ends at
// the end of its contig, the first of ends[0 .. n_contigs) above it (contigs back to back in .ann order)
struct DevRepeats {
    const u8 *pac;
    const u32 *ends;
    u32 n_contigs;
    u32 pac_st, n;
    u32 *out;
};

// complement of reference base p: BASE_COMP_B[get_base(p)] (src/bwa_index.hpp:257-259, src/bp.hpp)
UNC_DEV u32 unc_pac_comp(const u8 *pac, u32 p) {
    return 3u - (((u32) d_ldg(pac + (p >> 2)) >> (((3u ^ p) & 3u) << 1)) & 3u);
}

// bwt_occ (reference submods/bwa/bwt.c:107-129) for one row and one base, reading only the words it needs
UNC_DEV u32 unc_occ_row(const DevIndex &ix, u32 k, u32 c) {
    if (k == ix.seq_len) return unc_L2(ix, c + 1) - unc_L2(ix, c);
    if (k == 0xFFFFFFFFu) return 0;                                  // (bwtint_t)-1: the range starts at row 0
    const u32 kk = k - (k >= ix.primary);
    return unc_occ_at(ix.bwt + ((size_t) (kk >> 7) << 2), kk, c);
}

// Walks one path; MODE (UNC_SA_*) says what is kept and returned.
// The first range is get_base_range(b) = [L2[b], L2[b+1]] -- its start is NOT L2[b]+1
// (src/bwa_index.hpp:172-174), so row start-1 can be (u64)-1.  Lengths are u32 on the device
// (the index image is limited to < 2^32 rows) with the same wrap-around to 0 for an empty range.
template <int MODE>
UNC_DEV u32 unc_selfalign_walk(const DevIndex &ix, const u8 *pac, u32 pos, u32 lim, u32 *park, u32 n_paths, u64 *out) {
    u32 b = unc_pac_comp(pac, pos);
    u32 rs = unc_L2(ix, b), re = unc_L2(ix, b + 1);
    u32 n = 0;
    for (u32 j = pos + 1u;; j++) {
        const u32 len = re - rs + 1u;
        const bool go = j < lim && len > 1u;
        if (go || len > 0u) {                                        // empty only after an N-derived base
            if (MODE == UNC_SA_PARK) { if (n < UNC_SA_STAGE) park[(size_t) n * n_paths] = len; }
            else if (MODE == UNC_SA_WRITE) out[n] = (u64) len;
            n++;
        }
        if (!go) return MODE == UNC_SA_STEPS ? j - pos - 1u : n;
        b = unc_pac_comp(pac, j);
        const u32 base = unc_L2(ix, b);
        const u32 ns = base + unc_occ_row(ix, rs - 1u, b) + 1u;      // get_neighbor (src/bwa_index.hpp:158-162)
        const u32 ne = base + unc_occ_row(ix, re, b);
        rs = ns; re = ne;
    }
}

UNC_DEV void unc_selfalign_count(const DevIndex &ix, const DevSelfAlign &A, u32 i) {
    A.count[i] = unc_selfalign_walk<UNC_SA_PARK>(ix, A.pac, A.pos[i], A.lim[i], A.stage + i, A.n, nullptr);
}

UNC_DEV void unc_selfalign_write(const DevIndex &ix, const DevSelfAlign &A, u32 i) {
    const u32 cnt = A.count[i];
    u64 *out = A.values + A.offsets[i];
    if (cnt <= UNC_SA_STAGE) {
        for (u32 j = 0; j < cnt; j++) out[j] = (u64) A.stage[(size_t) j * A.n + i];
    } else {
        unc_selfalign_walk<UNC_SA_WRITE>(ix, A.pac, A.pos[i], A.lim[i], nullptr, 0, out);
    }
}

UNC_DEV void unc_repeat_length(const DevIndex &ix, const DevRepeats &R, u32 i) {
    const u32 p = R.pac_st + i;
    u32 lo = 0, hi = R.n_contigs - 1u;                               // the first contig end above p
    while (lo < hi) {
        const u32 m = (lo + hi) >> 1;
        if (d_ldg(R.ends + m) > p) hi = m; else lo = m + 1u;
    }
    R.out[i] = unc_selfalign_walk<UNC_SA_STEPS>(ix, R.pac, p, d_ldg(R.ends + lo), nullptr, 0, nullptr);
}
