// unc_mask.cuh -- device half of `mask-internal`: iterative masking of the most frequent k-mer of a reference
// (the loop of the reference's masking/mask_internal.sh over `jellyfish count` + masking/mask_kmers.py).
//
// The genome is one byte per base: 0-3 = ACGT (either case), UNC_MASK_BRK for any other byte and between records,
// and UNC_MASK_HIT or'ed onto a base masked by an earlier iteration.  Any code >= 4 breaks a k-mer.  Each buffer
// holds UNC_MASK_PAD break codes, then the positions rounded up to whole tiles (break codes past the end), then
// UNC_MASK_PAD more, so a tile and its halo are always inside the buffer.
//
// One pass per iteration (unc_mask_tile): a CTA loads a tile of T = threads x UNC_MASK_W positions plus 32 bytes
// on each side into shared memory, masks every position covered by an occurrence of the previous iteration's k-mer,
// writes the masked tile to the other buffer (ping-pong: no tile reads what another tile writes), and counts every
// k-mer that starts in the tile into the dense 4^k histogram.  Each thread owns UNC_MASK_W consecutive positions
// and rolls the 2-bit code over them: the masking needs the source from k-1 before to 2k-2 after its positions,
// the counting the masked values up to k-1 after, and it recomputes that overlap itself rather than exchanging it.
// Shared memory is skewed by 4 bytes per 32 so that the 32 threads of a warp, 32 bytes apart, hit 32 banks.
// Counts use warp-aggregated atomics: lanes holding the same k-mer (a poly-A run spans many lanes) add once.
//
// unc_mask_argmax_part / unc_mask_argmax_final then pick the k-mer with the highest count, ties to the smallest
// code, and reset the histogram for the next pass.  The choice stays on the device: the next pass reads it from
// `sel`, so all iterations are enqueued without a host round trip.
#pragma once
#include "unc_device.cuh"

#define UNC_MASK_W 32u              // consecutive positions per thread
#define UNC_MASK_BRK 4u             // not ACGT / record separator
#define UNC_MASK_HIT 8u             // masked by an earlier iteration (written back as 'N')
#define UNC_MASK_PAD 32u            // break codes before and after the positions in each buffer (>= 2k-2 for k <= 13)
#define UNC_MASK_MAX_K 13u
#define UNC_MASK_NONE 0xFFFFFFFFu   // never a k-mer code (k <= 13: codes < 2^26)
#define UNC_MASK_MAX_THREADS 256u
// shared bytes of a tile of nt threads: input (tile + 2 x 32) and output (tile), 4 bytes of skew per 32
#define UNC_MASK_SKEW(i) ((i) + ((i) >> 5) * 4u)
#define UNC_MASK_IN_WORDS(nt) (UNC_MASK_SKEW((nt) * UNC_MASK_W + 64u) / 4u)
#define UNC_MASK_OUT_WORDS(nt) (UNC_MASK_SKEW((nt) * UNC_MASK_W) / 4u)

struct DevMaskPass {
    const u8 *src;      // buffer start (UNC_MASK_PAD break codes, then position 0)
    u8 *dst;
    u64 n_tiles;
    u32 k;
    u32 *hist;          // 4^k counts, or null: this pass only masks
    const u64 *prev;    // (count << 32 | code) chosen by the previous iteration, or null (first pass)
};

struct DevMaskArgmax {
    u32 *hist;          // read and reset to 0
    u32 n_bins;         // 4^k
    u64 *part;          // one key per CTA of the first kernel
    u32 n_part;
    u64 *sel;           // out (final kernel): (count << 32 | code)
};

// One tile (positions [tile*T, tile*T + T)) on a CTA of c_nthreads() threads.  s_in / s_out: UNC_MASK_IN_WORDS /
// UNC_MASK_OUT_WORDS words of shared memory.
UNC_DEV void unc_mask_tile(const DevMaskPass &P, u64 tile, u32 *s_in, u32 *s_out) {
    const u32 nt = (u32) c_nthreads(), tid = (u32) c_tid(), T = nt * UNC_MASK_W, k = P.k;
    const u32 kmask = k >= 16u ? 0xFFFFFFFFu : (1u << (2u * k)) - 1u;
    const u64 t0 = tile * (u64) T;
    bool count = P.hist != nullptr;
    u32 pcode = UNC_MASK_NONE;
    if (P.prev) {
        const u64 s = *P.prev;
        if ((s >> 32) == 0) count = false;            // the previous iteration found no k-mer: nothing left to do
        else pcode = (u32) s;
    }
    // buffer bytes [t0, t0 + T + 64) = positions [t0 - 32, t0 + T + 32) -> local bytes [0, T + 64)
    const uint4 *g = (const uint4 *) (P.src + t0);
    for (u32 v = tid; v < (T + 64u) / 16u; v += nt) {
        const uint4 x = d_ldg(g + v);
        u32 *w = s_in + UNC_MASK_SKEW(16u * v) / 4u;
        w[0] = x.x; w[1] = x.y; w[2] = x.z; w[3] = x.w;
    }
    c_sync();
    const u8 *in = (const u8 *) s_in;
    u8 *out = (u8 *) s_out;
    const u32 base = 32u + tid * UNC_MASK_W;          // local byte of this thread's first position a
    // 1. coverage of positions a .. a+W+k-2 (bit r = position a + r) by occurrences of the previous k-mer: the
    //    windows ending at a-k+1+j for j < W+3k-3, i.e. starting at a + j - 2k + 2
    u64 cov = 0;
    if (pcode != UNC_MASK_NONE) {
        u32 code = 0, run = 0;
        const u32 first = base - (k - 1u), steps = UNC_MASK_W + 3u * k - 3u;
        for (u32 j = 0; j < steps; j++) {
            const u32 c = in[UNC_MASK_SKEW(first + j)];
            if (c < 4u) { code = ((code << 2) | c) & kmask; run++; } else run = 0;
            if (run >= k && code == pcode) {
                int lo = (int) j - 2 * (int) k + 2, hi = (int) j - (int) k + 1;
                if (lo < 0) lo = 0;
                if (hi > (int) (UNC_MASK_W + k - 2u)) hi = (int) (UNC_MASK_W + k - 2u);
                if (lo <= hi) cov |= (2ull << hi) - (1ull << lo);
            }
        }
    }
    // 2. the masked values of a .. a+W+k-2: the first W are this thread's output, the k-mers starting at a .. a+W-1
    //    are counted
    u32 code = 0, run = 0;
    const u32 lane = (u32) w_lane();
    for (u32 r = 0; r < UNC_MASK_W + k - 1u; r++) {
        u32 c = in[UNC_MASK_SKEW(base + r)];
        if ((cov >> r) & 1ull) c |= UNC_MASK_HIT;
        if (r < UNC_MASK_W) out[UNC_MASK_SKEW(tid * UNC_MASK_W + r)] = (u8) c;
        if (c < 4u) { code = ((code << 2) | c) & kmask; run++; } else run = 0;
        if (count) {                                   // uniform: every lane takes the same branch
            const bool v = r + 1u >= k && run >= k;
            const u32 peers = w_match(v ? code : UNC_MASK_NONE);
            if (v && (peers & ((1u << lane) - 1u)) == 0) d_atomic_add(P.hist + code, (u32) d_popc(peers));
        }
    }
    c_sync();
    uint4 *d = (uint4 *) (P.dst + UNC_MASK_PAD + t0);
    for (u32 v = tid; v < T / 16u; v += nt) {
        const u32 *w = s_out + UNC_MASK_SKEW(16u * v) / 4u;
        d[v] = make_uint4(w[0], w[1], w[2], w[3]);
    }
    c_sync();                                          // s_in / s_out are reused by the CTA's next tile
}

// argmax key: higher count first, then the smaller code
UNC_DEV u64 unc_mask_key(u32 count, u32 code) { return ((u64) count << 32) | (u64) (~code); }

UNC_DEV u64 unc_mask_cta_max(u64 key, u64 *s_red) {
    for (int d = 16; d > 0; d >>= 1) {
        const u64 y = w_shfl64(key, w_lane() ^ d);
        key = y > key ? y : key;
    }
    const u32 nw = (u32) c_nthreads() / 32u, wid = (u32) c_tid() / 32u;
    if (w_lane() == 0) s_red[wid] = key;
    c_sync();
    key = 0;
    for (u32 i = 0; i < nw; i++) key = s_red[i] > key ? s_red[i] : key;
    c_sync();
    return key;
}

// CTA `blk` of n_part: the best key of its share of the bins, which it resets to 0.  s_red: 32 u64.
UNC_DEV void unc_mask_argmax_part(const DevMaskArgmax &A, u32 blk, u64 *s_red) {
    const u32 per = (A.n_bins + A.n_part - 1u) / A.n_part, lo = blk * per;
    const u32 hi = lo + per < A.n_bins ? lo + per : A.n_bins;
    u64 key = 0;
    for (u32 i = lo + (u32) c_tid(); i < hi; i += (u32) c_nthreads()) {
        const u32 c = A.hist[i];
        const u64 kk = unc_mask_key(c, i);
        key = kk > key ? kk : key;
        if (c) A.hist[i] = 0;
    }
    key = unc_mask_cta_max(key, s_red);
    if (c_tid() == 0) A.part[blk] = key;
}

UNC_DEV void unc_mask_argmax_final(const DevMaskArgmax &A, u64 *s_red) {
    u64 key = 0;
    for (u32 i = (u32) c_tid(); i < A.n_part; i += (u32) c_nthreads()) key = A.part[i] > key ? A.part[i] : key;
    key = unc_mask_cta_max(key, s_red);
    if (c_tid() == 0) {
        const u32 count = (u32) (key >> 32), code = ~(u32) key;
        *A.sel = ((u64) count << 32) | (count ? code : 0u);
    }
}
