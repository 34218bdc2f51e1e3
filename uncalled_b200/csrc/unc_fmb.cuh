// unc_fmb.cuh -- device half of the FM-index builder (unc_index_build_device): the suffix array of the bwa text
// (forward codes, their reverse complement, one smallest sentinel) by prefix doubling, then the BWT, the Occ blocks and
// the sampled SA of the .bwt / .sa files.  The launch sequence is unc_fmb_run.hpp's.
//
// Text.  n symbols, 2 bits each, 16 per u32 with the first symbol in the top bits, zero past n (two zero words of
// padding).  Row g of the suffix array holds the suffix SA[g]; row 0 is the sentinel suffix n.  ISA[i] is the first
// row of the group of suffix i: the rows whose suffixes share the prefix sorted so far.  Group heads are one bit per
// row (bit g of head = row g starts a group; bit N is set, N = n + 1).
//
// Functors.  A per-element functor has `operator()(u64 i)`, run once for every i < count (`Dev::each` of
// unc_fmb_run.hpp: a grid-stride loop on the device, a plain loop in the emulator).  A CTA functor has `tile(u64 t, u32 *smem)` for a
// CTA of UNC_FMB_THREADS threads and SMEM_WORDS words of shared memory; it ends with a barrier so the next tile of the
// same CTA may reuse the shared memory.
#pragma once
#include "unc_device.cuh"

// member functions of the functors (UNC_DEV is `static` under the emulator)
#ifdef UNC_EMUL
#define UNC_FMB_FN inline
#else
#define UNC_FMB_FN __device__ __forceinline__
#endif

#define UNC_FMB_THREADS 256u
#define UNC_FMB_WARPS (UNC_FMB_THREADS / 32u)
#define UNC_FMB_K0_MAX 12u             // bases of the initial counting sort (4^12 buckets) at most
#define UNC_FMB_KOFF 16u               // ranks are stored + UNC_FMB_KOFF in the keys; below it, suffixes past the end
#define UNC_FMB_SCAN_ITEMS 8u
#define UNC_FMB_SCAN_TILE (UNC_FMB_THREADS * UNC_FMB_SCAN_ITEMS)
#define UNC_FMB_RADIX_ITEMS 4u
#define UNC_FMB_RADIX_TILE (UNC_FMB_THREADS * UNC_FMB_RADIX_ITEMS)
#define UNC_FMB_ROWS_PER_TILE (UNC_FMB_THREADS * 32u)   // active-row compaction: one head word per thread

UNC_DEV u32 unc_fmb_sym(const u32 *text, u64 i) { return (text[i >> 4] >> ((15u - (u32) (i & 15)) << 1)) & 3u; }

// the k0 bases from i (zero past the end) as 2 k0 bits, first base on top
UNC_DEV u32 unc_fmb_prefix(const u32 *text, u64 i, u32 k0) {
    const u64 w = ((u64) text[i >> 4] << 32) | text[(i >> 4) + 1];
    return (u32) ((w << ((u32) (i & 15) << 1)) >> (64u - 2u * k0));
}

UNC_DEV u32 unc_fmb_op(u32 a, u32 b, u32 is_max) { return is_max ? (a > b ? a : b) : a + b; }

// exclusive scan over the CTA's threads in thread order (sum, or max with identity 0); *total = the CTA's aggregate.
// smem: UNC_FMB_WARPS words.  Ends with a barrier.
UNC_DEV u32 unc_fmb_cta_exscan(u32 v, u32 is_max, u32 *total, u32 *smem) {
    const int lane = w_lane(), warp = c_tid() >> 5;
    u32 x = v;
    for (int d = 1; d < 32; d <<= 1) {
        const u32 y = w_shfl_up(x, d);
        if (lane >= d) x = unc_fmb_op(x, y, is_max);
    }
    u32 ex = w_shfl_up(x, 1);
    if (lane == 0) ex = 0;
    if (lane == 31) smem[warp] = x;
    c_sync();
    u32 off = 0, all = 0;
    for (int w = 0; w < (int) UNC_FMB_WARPS; w++) {
        if (w < warp) off = unc_fmb_op(off, smem[w], is_max);
        all = unc_fmb_op(all, smem[w], is_max);
    }
    c_sync();
    *total = all;
    return unc_fmb_op(off, ex, is_max);
}

// ---------------------------------------------------------------- device-wide scan of u32 (in place)
// three steps: FmbScanReduce (one aggregate per tile), FmbScanParts (one CTA scans the aggregates, starting at `init`),
// FmbScanApply (every tile scanned from its offset)
struct FmbScan {
    u32 *x;
    u64 n;
    u32 *part;          // one per tile
    u64 n_tiles;
    u32 is_max, inclusive, init;
    u32 *total;         // the aggregate (including init)
};

struct FmbScanReduce {
    FmbScan s;
    static const u32 SMEM_WORDS = UNC_FMB_WARPS;
    UNC_FMB_FN void tile(u64 t, u32 *smem) const {
        const u64 base = t * UNC_FMB_SCAN_TILE + (u64) c_tid() * UNC_FMB_SCAN_ITEMS;
        u32 v = 0, agg = 0;
        for (u32 k = 0; k < UNC_FMB_SCAN_ITEMS; k++)
            if (base + k < s.n) v = unc_fmb_op(v, s.x[base + k], s.is_max);
        unc_fmb_cta_exscan(v, s.is_max, &agg, smem);
        if (c_tid() == 0) s.part[t] = agg;
    }
};

struct FmbScanParts {
    FmbScan s;
    static const u32 SMEM_WORDS = UNC_FMB_WARPS;
    UNC_FMB_FN void tile(u64, u32 *smem) const {
        u32 carry = s.init;
        for (u64 base = 0; base < s.n_tiles; base += UNC_FMB_THREADS) {
            const u64 e = base + (u64) c_tid();
            const u32 v = e < s.n_tiles ? s.part[e] : 0;
            u32 agg = 0;
            const u32 ex = unc_fmb_cta_exscan(v, s.is_max, &agg, smem);
            if (e < s.n_tiles) s.part[e] = unc_fmb_op(carry, ex, s.is_max);
            carry = unc_fmb_op(carry, agg, s.is_max);
        }
        if (c_tid() == 0) *s.total = carry;
        c_sync();
    }
};

struct FmbScanApply {
    FmbScan s;
    static const u32 SMEM_WORDS = UNC_FMB_WARPS;
    UNC_FMB_FN void tile(u64 t, u32 *smem) const {
        const u64 base = t * UNC_FMB_SCAN_TILE + (u64) c_tid() * UNC_FMB_SCAN_ITEMS;
        u32 v[UNC_FMB_SCAN_ITEMS], sum = 0, agg = 0;
        for (u32 k = 0; k < UNC_FMB_SCAN_ITEMS; k++) {
            v[k] = base + k < s.n ? s.x[base + k] : 0;
            sum = unc_fmb_op(sum, v[k], s.is_max);
        }
        u32 run = unc_fmb_op(s.part[t], unc_fmb_cta_exscan(sum, s.is_max, &agg, smem), s.is_max);
        for (u32 k = 0; k < UNC_FMB_SCAN_ITEMS; k++) {
            const u32 next = unc_fmb_op(run, v[k], s.is_max);
            if (base + k < s.n) s.x[base + k] = s.inclusive ? next : run;
            run = next;
        }
    }
};

// ---------------------------------------------------------------- initial counting sort on the first k0 bases
struct FmbHist {          // i < n
    const u32 *text;
    u32 *cnt;
    u32 k0;
    UNC_FMB_FN void operator()(u64 i) const { d_atomic_add(&cnt[unc_fmb_prefix(text, i, k0)], 1u); }
};

// i < n: suffix i goes to the next free row of its bucket; the row that is a bucket's first becomes a group head.
// Within a bucket the rows are in atomic order, which the doubling rounds sort.
struct FmbScatter {
    const u32 *text;
    const u32 *start;     // first row of every bucket (row 0 is the sentinel's)
    u32 *cursor;          // a copy of start
    u32 *SA, *ISA, *head;
    u32 k0;
    UNC_FMB_FN void operator()(u64 i) const {
        const u32 b = unc_fmb_prefix(text, i, k0);
        const u32 p = d_atomic_add(&cursor[b], 1u);
        SA[p] = (u32) i;
        ISA[i] = start[b];
        if (p == start[b]) d_atomic_or(&head[p >> 5], 1u << (p & 31));
    }
};

struct FmbSentinel {      // one element: row 0 is the sentinel suffix n, a group of its own; bit N closes the heads
    u32 *SA, *ISA, *head;
    u64 n;
    UNC_FMB_FN void operator()(u64) const {
        SA[0] = (u32) n;
        ISA[n] = 0;
        d_atomic_or(&head[0], 1u);
        d_atomic_or(&head[(n + 1) >> 5], 1u << ((n + 1) & 31));
    }
};

// ---------------------------------------------------------------- doubling round: the rows of unsorted groups
// a row is active when its group has more than one row: not (head[g] and head[g + 1])
UNC_DEV u32 unc_fmb_active_word(const u32 *head, u64 w, u64 N) {
    const u32 hw = head[w], nb = head[w + 1] & 1u;
    u32 act = ~(hw & ((hw >> 1) | (nb << 31)));
    const u64 row0 = w << 5;
    if (row0 >= N) return 0;
    if (N - row0 < 32) act &= (1u << (u32) (N - row0)) - 1u;
    return act;
}

struct FmbActive {
    const u32 *head;
    u64 N;
    u32 *tile_cnt;        // per tile, then its exclusive scan
    u32 *A;               // out (compact pass): the active rows in order
    u32 compact;
    static const u32 SMEM_WORDS = UNC_FMB_WARPS;
    UNC_FMB_FN void tile(u64 t, u32 *smem) const {
        const u64 w = t * UNC_FMB_THREADS + (u64) c_tid();
        u32 act = unc_fmb_active_word(head, w, N), agg = 0;
        const u32 off = unc_fmb_cta_exscan((u32) d_popc(act), 0, &agg, smem);
        if (!compact) {
            if (c_tid() == 0) tile_cnt[t] = agg;
            return;
        }
        u32 *out = A + tile_cnt[t] + off;
        while (act) {
            const int b = d_ffs(act) - 1;
            *out++ = (u32) ((w << 5) + (u64) b);
            act &= act - 1u;
        }
    }
};

// p < M: the rank of the suffix h after row A[p]'s, read before any rank of this round changes.  A suffix within h of
// the end (only in the first round, h = k0 <= UNC_FMB_K0_MAX < UNC_FMB_KOFF) compares as padded with the sentinel:
// below every rank, and the shorter one first.
struct FmbSnapshot {
    const u32 *A, *SA, *ISA;
    u32 *K;
    u64 n, h;
    UNC_FMB_FN void operator()(u64 p) const {
        const u64 j = (u64) SA[A[p]] + h;
        K[p] = j <= n ? ISA[j] + UNC_FMB_KOFF : UNC_FMB_KOFF - (u32) (j - n);
    }
};

// q < m: the sort key of the batch's q-th active row: its group's first row (relative to the batch's first row g0),
// then the snapshot rank
struct FmbKeys {
    const u32 *A, *SA, *ISA, *K;
    u64 p0;
    u32 g0;
    u64 *key;
    u32 *val;
    UNC_FMB_FN void operator()(u64 q) const {
        const u32 i = SA[A[p0 + q]];
        key[q] = ((u64) (ISA[i] - g0) << 32) | K[p0 + q];
        val[q] = i;
    }
};

// ---------------------------------------------------------------- LSD radix sort of (u64 key, u32 value), 8 bits a pass
struct FmbRadix {
    const u64 *key_in;
    const u32 *val_in;
    u64 *key_out;
    u32 *val_out;
    u64 m, n_tiles;
    u32 shift;
    u32 *hist;            // [256][n_tiles], then its exclusive scan
};

struct FmbRadixHist {
    FmbRadix r;
    static const u32 SMEM_WORDS = 256;
    UNC_FMB_FN void tile(u64 t, u32 *smem) const {
        smem[c_tid()] = 0;
        c_sync();
        for (u32 k = 0; k < UNC_FMB_RADIX_ITEMS; k++) {
            const u64 e = t * UNC_FMB_RADIX_TILE + k * UNC_FMB_THREADS + (u64) c_tid();
            if (e < r.m) s_atomic_add(&smem[(u32) (r.key_in[e] >> r.shift) & 255u], 1u);
        }
        c_sync();
        r.hist[(u64) c_tid() * r.n_tiles + t] = smem[c_tid()];
        c_sync();
    }
};

// stable: within a tile, the elements of one digit keep their order (warp peers by match, warps in order, the tile's
// UNC_FMB_RADIX_ITEMS rounds in order)
struct FmbRadixScatter {
    FmbRadix r;
    static const u32 SMEM_WORDS = UNC_FMB_WARPS * 256 + 512;
    UNC_FMB_FN void tile(u64 t, u32 *smem) const {
        u32 *wc = smem, *run = smem + UNC_FMB_WARPS * 256, *base = run + 256;
        const u32 tid = (u32) c_tid(), warp = tid >> 5;
        base[tid] = r.hist[(u64) tid * r.n_tiles + t];
        run[tid] = 0;
        for (u32 k = 0; k < UNC_FMB_RADIX_ITEMS; k++) {
            const u64 e = t * UNC_FMB_RADIX_TILE + k * UNC_FMB_THREADS + tid;
            const bool valid = e < r.m;
            const u64 key = valid ? r.key_in[e] : 0;
            const u32 d = valid ? (u32) (key >> r.shift) & 255u : 256u;
            for (u32 w = 0; w < UNC_FMB_WARPS; w++) wc[w * 256 + tid] = 0;
            c_sync();
            const u32 peers = w_match(d);
            if (valid && (peers & w_lanemask_lt()) == 0) wc[warp * 256 + d] = (u32) d_popc(peers);
            c_sync();
            u32 off = run[tid];
            for (u32 w = 0; w < UNC_FMB_WARPS; w++) {
                const u32 x = wc[w * 256 + tid];
                wc[w * 256 + tid] = off;
                off += x;
            }
            run[tid] = off;
            c_sync();
            if (valid) {
                const u32 pos = base[d] + wc[warp * 256 + d] + (u32) d_popc(peers & w_lanemask_lt());
                r.key_out[pos] = key;
                r.val_out[pos] = r.val_in[e];
            }
            c_sync();
        }
    }
};

// q < m: the sorted suffixes back into the batch's rows; a row whose key differs from the previous one starts a group.
// mark[q] = the row if it starts a group, else 0 (a max-scan of it gives every row its group's first row).
struct FmbWriteback {
    const u32 *A;
    u64 p0;
    const u64 *key;
    const u32 *val;
    u32 *SA, *head, *mark;
    UNC_FMB_FN void operator()(u64 q) const {
        const u32 g = A[p0 + q];
        SA[g] = val[q];
        const bool h = q == 0 || key[q] != key[q - 1];
        if (h) d_atomic_or(&head[g >> 5], 1u << (g & 31));
        mark[q] = h ? g : 0u;
    }
};

struct FmbRank {          // q < m, after the inclusive max-scan of mark
    const u32 *val, *mark;
    u32 *ISA;
    UNC_FMB_FN void operator()(u64 q) const { ISA[val[q]] = mark[q]; }
};

// ---------------------------------------------------------------- outputs
// w < (n + 15) / 16: output symbols 16w .. 16w+15 (row `primary`, whose suffix is 0, is the dropped '$'), packed into
// the Occ-interleaved payload: block b = w / 8 holds 8 words of counts, then its 8 symbol words
struct FmbBwt {
    const u32 *text, *SA;
    u64 n, primary;
    u32 *out;
    UNC_FMB_FN void operator()(u64 w) const {
        u32 word = 0;
        for (u32 s = 0; s < 16; s++) {
            const u64 j = w * 16 + s;
            if (j >= n) break;
            const u64 row = j < primary ? j : j + 1;
            word |= unc_fmb_sym(text, (u64) SA[row] - 1) << ((15u - s) << 1);
        }
        out[(w >> 3) * 16 + 8 + (w & 7)] = word;
    }
};

struct FmbOccCount {      // b < nb: the symbols of block b, cnt[c * nb + b]
    const u32 *out;
    u64 n, nb;
    u32 *cnt;
    UNC_FMB_FN void operator()(u64 b) const {
        const u64 rem = n - b * 128;
        const u32 len = rem < 128 ? (u32) rem : 128u;
        u32 c[4] = {0, 0, 0, 0};
        for (u32 s = 0; s < len; s++) c[(out[b * 16 + 8 + (s >> 4)] >> ((15u - (s & 15)) << 1)) & 3u]++;
        for (u32 k = 0; k < 4; k++) cnt[k * nb + b] = c[k];
    }
};

struct FmbOccWrite {      // b <= nb: the 4 x u64 counts before block b (b = nb: the totals, at the payload's end)
    const u32 *cnt;       // exclusive scan of FmbOccCount's counts
    u64 nb, n_words;
    u64 total[4];
    u32 *out;
    UNC_FMB_FN void operator()(u64 b) const {
        u32 *o = out + (b < nb ? b * 16 : n_words - 8);
        for (u32 k = 0; k < 4; k++) {
            const u64 v = b < nb ? (u64) (cnt[k * nb + b] - cnt[k * nb]) : total[k];
            o[2 * k] = (u32) v;
            o[2 * k + 1] = (u32) (v >> 32);
        }
    }
};

struct FmbSaSample {      // j < n_sa - 1: SA[32 (j + 1)]
    const u32 *SA;
    u64 *sa;
    UNC_FMB_FN void operator()(u64 j) const { sa[j] = SA[(j + 1) * 32]; }
};
