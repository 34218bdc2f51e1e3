// unc_mask_ext.cuh -- device half of `mask-external`: the copy number of every min_len window of a target reference
// in a full reference (both strands, exact matches), as masking/mask_external.sh gets it from `bowtie -fa -v 0`.
//
// Keys.  A k-mer (k <= 64) is 2 bits per base, first base in the top bits, in a u128; its canonical key is
// min(forward, reverse complement).  A target window w and a full-reference k-mer x share a canonical key exactly
// when x is w or revcomp(w), so adding 1 per full-reference position to the slot of its canonical key counts
// occ(w) + occ(revcomp(w)); a palindrome (x == revcomp(x)) adds 2, since it is an occurrence of both.
//
// Table.  Open addressing with linear probing over `cap` (a power of two, at least twice the target's valid windows)
// 16-byte keys, a u32 count per slot, and a bit per slot that records a count passing UINT32_MAX (the count is then
// saturated).  A free slot holds ~0, which is never a canonical key: for k < 64 its top bits are set, and for k = 64
// its reverse complement is 0.  A bitset `filter` (one bit per key, indexed by other bits of the same hash) is read
// first, so most full-reference positions, which miss a table built from a small target, never touch the keys in HBM.
//
// k_mx_build (unc_mx_build_chunk): one thread per UNC_MX_W consecutive target positions rolls the keys over the
// codes of unc_mask_host.hpp and inserts each valid window with a 16-byte atomicCAS; it stores the window's slot, so
// the marking is a gather.  k_mx_count (unc_mx_count_tile), once per piece of the full reference: a CTA loads a tile
// of threads x UNC_MX_W window starts plus a 64-byte halo of FASTA bytes into shared memory; each thread rolls the
// forward and reverse-complement keys over its UNC_MX_W starts (and k-1 bytes before them) and probes the filter,
// then the table.  Hits are added with warp-aggregated atomics: lanes of one warp that hit the same slot (a
// low-complexity run spanning the warp) add once.  k_mx_mark (unc_mx_mark_chunk): per target position, the count of
// the window starting there, and bit 3 (UNC_MASK_HIT) on every position covered by a window whose count is greater
// than min_copy.
#pragma once
#include "unc_mask.cuh"

typedef unsigned __int128 u128;

#define UNC_MX_MAX_K 64u
#define UNC_MX_W 64u                // consecutive window starts per thread
#define UNC_MX_HALO 64u             // bytes loaded after a tile (>= k - 1)
#define UNC_MX_NONE 0xFFFFFFFFu     // slot of a position where no valid window starts
#define UNC_MX_MAX_THREADS 256u
// shared memory of a count tile: skewed by 4 bytes per UNC_MX_W, so the lanes of a warp, UNC_MX_W bytes apart, read
// 32 different banks
#define UNC_MX_SKEW(i) ((i) + ((i) / UNC_MX_W) * 4u)
#define UNC_MX_TILE_WORDS(nt) (UNC_MX_SKEW((nt) * UNC_MX_W + UNC_MX_HALO) / 4u)

struct DevMxTable {
    u128 *keys;         // cap canonical keys, ~0 where free
    u32 *cnt;           // cap counts
    u32 *ovf;           // cap bits: the count passed UINT32_MAX
    u32 *filter;        // filter_bits bits: set for every key in the table
    u64 cap, filter_bits;   // powers of two; cap <= 2^31
    u32 k;
};

struct DevMxBuild {
    DevMxTable t;
    const u8 *codes;    // the target: n codes of unc_mask_code, UNC_MASK_BRK between records
    u64 n;
    u32 *slot;          // out: per position, the slot of the window starting there, or UNC_MX_NONE
};

struct DevMxCount {
    DevMxTable t;
    const u8 *bytes;    // a piece of the full reference: FASTA sequence bytes, '\n' between records; 16-byte aligned
                        // and readable up to n_tiles x tile + UNC_MX_HALO
    u64 n_starts;       // the windows starting at bytes 0 .. n_starts-1 are counted (bytes up to n_starts+k-2 valid)
    u64 n_tiles;
};

struct DevMxMark {
    DevMxTable t;
    const u32 *slot;
    u8 *codes;          // bit 3 set on every position of a selected window
    u32 *counts;        // out: per position, the count of the window starting there (0 where none)
    u64 n;
    u32 min_copy;
};

UNC_DEV u128 mx_empty() { return ~(u128) 0; }
UNC_DEV u128 mx_kmask(u32 k) { return k >= 64u ? ~(u128) 0 : (((u128) 1) << (2u * k)) - 1u; }

UNC_DEV u64 mx_hash(u128 key) {
    u64 x = (u64) key ^ ((u64) (key >> 64) * 0x9E3779B97F4A7C15ull);
    x ^= x >> 33; x *= 0xFF51AFD7ED558CCDull;
    x ^= x >> 33; x *= 0xC4CEB9FE1A85EC53ull;
    return x ^ (x >> 33);
}
// the slot probing starts at: the low bits; the filter bit: bits 32 and up
UNC_DEV u64 mx_filter_bit(const DevMxTable &t, u64 h) { return (h >> 32) & (t.filter_bits - 1u); }

// unc_mask_code of a FASTA byte: 0-3 for ACGT in either case, UNC_MASK_BRK otherwise
UNC_DEV u32 mx_code(u32 b) {
    const u32 x = b | 0x20u;
    return (x == 'a' || x == 'c' || x == 'g' || x == 't') ? ((x >> 1) ^ (x >> 2)) & 3u : UNC_MASK_BRK;
}

struct MxRoll {
    u128 fwd, rc;       // the last k bases and their reverse complement (valid once run >= k)
    u32 run;            // ACGT bases since the last break
};
UNC_DEV void mx_push(MxRoll &r, u32 c, u32 k, u128 kmask) {
    if (c < 4u) {
        r.fwd = ((r.fwd << 2) | c) & kmask;
        r.rc = (r.rc >> 2) | ((u128) (3u - c) << (2u * k - 2u));
        r.run++;
    } else {
        r.run = 0;
    }
}

// the slot of `key`, inserted if absent
UNC_DEV u32 mx_insert(const DevMxTable &t, u128 key) {
    const u64 h = mx_hash(key);
    u64 s = h & (t.cap - 1u);
    for (;;) {
        const u128 old = d_atomic_cas128(t.keys + s, mx_empty(), key);
        if (old == mx_empty()) {
            const u64 f = mx_filter_bit(t, h);
            d_atomic_or(t.filter + (f >> 5), 1u << (f & 31u));
            break;
        }
        if (old == key) break;
        s = (s + 1u) & (t.cap - 1u);
    }
    return (u32) s;
}

// the slot of `key`, or UNC_MX_NONE
UNC_DEV u32 mx_find(const DevMxTable &t, u128 key) {
    const u64 h = mx_hash(key), f = mx_filter_bit(t, h);
    if (!((d_ldg(t.filter + (f >> 5)) >> (f & 31u)) & 1u)) return UNC_MX_NONE;
    for (u64 s = h & (t.cap - 1u);; s = (s + 1u) & (t.cap - 1u)) {
        const u128 x = t.keys[s];
        if (x == key) return (u32) s;
        if (x == mx_empty()) return UNC_MX_NONE;
    }
}

// the window starts [chunk x UNC_MX_W, + UNC_MX_W) of the target
UNC_DEV void unc_mx_build_chunk(const DevMxBuild &B, u64 chunk) {
    const u32 k = B.t.k;
    const u128 km = mx_kmask(k);
    const u64 a = chunk * UNC_MX_W;
    MxRoll r = {0, 0, 0};
    for (u32 j = 0; j < UNC_MX_W + k - 1u; j++) {
        const u64 p = a + j;
        mx_push(r, p < B.n ? B.codes[p] : UNC_MASK_BRK, k, km);
        if (j + 1u < k) continue;
        const u64 s = p + 1u - k;
        if (s >= B.n) break;
        B.slot[s] = r.run >= k ? mx_insert(B.t, r.fwd < r.rc ? r.fwd : r.rc) : UNC_MX_NONE;
    }
}

// lanes of the warp that hit the same slot add once; `v` is the same for all of them (it depends on the key)
UNC_DEV void mx_add(const DevMxTable &t, u32 slot, u32 v) {
    const u32 peers = w_match(slot);
    if (slot == UNC_MX_NONE || (peers & w_lanemask_lt()) != 0) return;
    const u32 add = v * (u32) d_popc(peers);
    // the total of a slot is below 2^33 (at most 2 per full-reference position), so it wraps at most once and
    // exactly one addition sees it
    if (d_atomic_add(t.cnt + slot, add) > 0xFFFFFFFFu - add) d_atomic_or(t.ovf + (slot >> 5), 1u << (slot & 31u));
}

// one tile (window starts [tile x T, tile x T + T)) of a piece on a CTA of c_nthreads() threads.  s_tile:
// UNC_MX_TILE_WORDS words of shared memory.
UNC_DEV void unc_mx_count_tile(const DevMxCount &P, u64 tile, u32 *s_tile) {
    const u32 nt = (u32) c_nthreads(), tid = (u32) c_tid(), T = nt * UNC_MX_W, k = P.t.k;
    const u64 t0 = tile * (u64) T;
    const uint4 *g = (const uint4 *) (P.bytes + t0);
    for (u32 v = tid; v < (T + UNC_MX_HALO) / 16u; v += nt) {
        const uint4 x = d_ldg(g + v);
        u32 *w = s_tile + UNC_MX_SKEW(16u * v) / 4u;
        w[0] = x.x; w[1] = x.y; w[2] = x.z; w[3] = x.w;
    }
    c_sync();
    const u128 km = mx_kmask(k);
    const u32 base = tid * UNC_MX_W;
    const u64 s0 = t0 + base;                          // this thread's first window start in the piece
    MxRoll r = {0, 0, 0};
    u32 word = 0;
    for (u32 j = 0; j < UNC_MX_W + k - 1u; j++) {      // the same trip count on every lane: mx_add is warp-wide
        if ((j & 3u) == 0) word = s_tile[UNC_MX_SKEW(base + j) / 4u];
        mx_push(r, mx_code((word >> (8u * (j & 3u))) & 0xFFu), k, km);
        u32 slot = UNC_MX_NONE, v = 1;
        if (j + 1u >= k && r.run >= k && s0 + j + 1u - k < P.n_starts) {
            const bool fwd_lo = r.fwd < r.rc;
            if (r.fwd == r.rc) v = 2;
            slot = mx_find(P.t, fwd_lo ? r.fwd : r.rc);
        }
        if (w_ballot(slot != UNC_MX_NONE)) mx_add(P.t, slot, v);
    }
    c_sync();                                          // s_tile is reused by the CTA's next tile
}

UNC_DEV u32 mx_count_of(const DevMxTable &t, u32 slot) {
    if (slot == UNC_MX_NONE) return 0;
    return ((t.ovf[slot >> 5] >> (slot & 31u)) & 1u) ? 0xFFFFFFFFu : t.cnt[slot];
}

// the target positions [chunk x UNC_MX_W, + UNC_MX_W): their window counts, and the mask bit of every position that
// a selected window starting up to k-1 before covers
UNC_DEV void unc_mx_mark_chunk(const DevMxMark &M, u64 chunk) {
    const u32 k = M.t.k;
    const u64 a = chunk * UNC_MX_W;
    u64 cover_end = 0;                                 // positions below it are covered
    for (u32 j = 0; j < UNC_MX_W + k - 1u; j++) {
        if (a + j < k - 1u) continue;
        const u64 s = a + j - (k - 1u);                // a window start, a-k+1 .. a+W-1
        if (s >= M.n) break;
        const u32 c = mx_count_of(M.t, M.slot[s]);
        if (c > M.min_copy) cover_end = s + k;
        if (s < a) continue;
        M.counts[s] = c;
        if (cover_end > s) M.codes[s] |= (u8) UNC_MASK_HIT;
    }
}
