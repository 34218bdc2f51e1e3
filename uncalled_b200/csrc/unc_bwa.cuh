// unc_bwa.cuh -- device half of the reference's BwaIndex queries (src/bwa_index.hpp:158-333): get_neighbor over
// bwt_2occ, bwt_sa, and range_to_fms cut into independent segments.
//
// range_to_fms walks the FM index once per reference position, each step depending on the last: a chromosome is
// ~10^8 dependent Occ lookups on one thread.  Here [pac_min, pac_max] is cut into segments of `seg` positions, and
// each segment starts from the exact row of its first position's suffix (unc_suffix_row): a backward search of the
// slop + 1 text bases that begin that suffix, then a scan of the resulting rows for the one whose SA value is the
// suffix's position.  The suffix begins with the searched bases, so its row is always in the range and the scan cannot
// miss on a consistent index (a miss is reported, never written).  An LF step from an exact row is the exact row of
// the next position, so every segment's list is the exact rows of its positions.
//
// The forward list is then the reference's bit for bit: its anchor is the row whose SA value is pac_max, searched
// inside the forward text where that row is always in its range.  The reverse list is not always: the reference's
// reverse scan compares size() - sa(f) with pac_min, which names the suffix one position before pac_min's reverse
// complement, so its scan usually finds nothing and its walk goes on from the whole range.  unc_fms_fixup runs the
// reference's reverse walk serially from its own anchor until its range is a single row equal to the segment pass's
// row at the same position; from there on the two chains agree and the rest of the segment pass stands.  Outside
// repeats that happens within about slop steps.  It takes the whole span when the reference's scan does match
// (pac_min ends a homopolymer of slop + 2 bases) and its one-row walk then leaves the exact chain.
#pragma once
#include "unc_selfalign.cuh"   // unc_occ_row

// base p of the forward reference: get_base (src/bwa_index.hpp:257-259)
UNC_DEV u32 unc_pac_base(const u8 *pac, u64 p) {
    return ((u32) d_ldg(pac + (p >> 2)) >> (((3u ^ (u32) p) & 3u) << 1)) & 3u;
}

// Occ of base c over words 0..q of a 128-row block, the last word up to symbol (pos & 31)
UNC_DEV u32 unc_occ_words(const uint4 *blk, u32 q, u32 pos, u32 c) {
    u32 cnt = d_ldg((const u32 *) blk + 2u * c);
    const uint2 *wp = (const uint2 *) (blk + 2);
    for (u32 i = 0; i <= q; i++) {
        const uint2 v = d_ldg(wp + i);
        const u64 w = ((u64) v.x << 32) | v.y;
        const u64 m = i < q ? ~0ull : ~((1ull << ((~pos & 31u) << 1)) - 1ull);
        cnt += (u32) d_popcll(unc_match_bits(w, c) & m);
    }
    return cnt;
}

// bwt_2occ (submods/bwa/bwt.c:132-163) as written, for any k and l: when both rows fall in one 128-row block the
// count at l continues from k's 32-symbol word, so an inverted range (l below k's word) counts k's word up to l's bit
UNC_DEV void unc_bwt_2occ(const DevIndex &ix, u32 k, u32 l, u32 c, u32 *ok, u32 *ol) {
    const u32 kk = k - (k >= ix.primary), ll = l - (l >= ix.primary);
    if ((kk >> 7) != (ll >> 7) || k == 0xFFFFFFFFu || l == 0xFFFFFFFFu) {
        *ok = unc_occ_row(ix, k, c);
        *ol = unc_occ_row(ix, l, c);
        return;
    }
    const uint4 *blk = ix.bwt + ((size_t) (kk >> 7) << 2);
    const u32 qk = (kk & 127u) >> 5, ql = (ll & 127u) >> 5;
    *ok = unc_occ_words(blk, qk, kk, c);
    *ol = unc_occ_words(blk, qk > ql ? qk : ql, ll, c);
}

// BwaIndex::get_neighbor (src/bwa_index.hpp:158-162)
UNC_DEV uint2 unc_bwa_neighbor(const DevIndex &ix, u32 st, u32 en, u32 c) {
    u32 os, oe;
    unc_bwt_2occ(ix, st - 1u, en, c, &os, &oe);
    const u32 b = unc_L2(ix, c);
    return make_uint2(b + os + 1u, b + oe);
}

// bwt_sa widened to bwa's u64: row 0 gives (u64)-1
UNC_DEV u64 unc_bwa_sa(const DevIndex &ix, u32 k) {
    u32 a = 0, b = 0;
    const u32 v = unc_sa(ix, k, &a, &b);
    return k == 0u ? ~0ull : (u64) v;
}

// LF step from row k (not primary): the row of the suffix one position earlier (bwt_invPsi, submods/bwa/bwt.c:53-59)
UNC_DEV u32 unc_lf(const DevIndex &ix, u32 k) {
    const u32 x = k - (k > ix.primary);
    const u32 *wp = (const u32 *) ix.bwt + (((size_t) (x >> 7)) << 4) + 8 + ((x & 0x7fu) >> 4);
    const u32 c = (d_ldg(wp) >> ((~x & 0xfu) << 1)) & 3u;
    return unc_L2(ix, c) + unc_occ_row(ix, k, c);
}

struct DevFms {
    const u8 *pac;
    u64 ref_len;          // size() / 2
    u32 slop;             // ceil(log(ref_len) / log(4))
    u64 pac_min, n;       // positions pac_min .. pac_min + n - 1
    u32 seg;              // positions per segment
    u64 n_seg;            // segments per walk
    u64 *fwd;             // fwd[j]: row of position pac_max - j (the reference's second list)
    u64 *rev;             // rev[j]: row of position pac_min + j (the reference's first list)
    u32 *miss;            // set when an anchor scan finds no row
};

// base p of the FM text: the forward reference, then its reverse complement
UNC_DEV u32 unc_text_base(const DevFms &F, u64 p) {
    return p < F.ref_len ? unc_pac_base(F.pac, p) : 3u - unc_pac_base(F.pac, 2u * F.ref_len - 1u - p);
}

// Per lane: where the row of text suffix t (t < seq_len) is.  A suffix of at most slop + 1 bases is reached from the
// `$` row by LF steps (*row).  Any other suffix begins with its slop + 1 bases, so its row is in their backward-search
// range (returned, *row = 0xFFFFFFFF); the range holds ~2 ref_len / 4^(slop+1) <= 1/2 other rows outside repeats.
UNC_DEV uint2 unc_suffix_range(const DevIndex &ix, const DevFms &F, u64 t, u32 *row) {
    const u64 tail = (u64) ix.seq_len - t;
    if (tail <= (u64) F.slop + 1u) {
        u32 k = 0;
        for (u64 i = 0; i < tail; i++) k = unc_lf(ix, k);
        *row = k;
        return make_uint2(1u, 0u);
    }
    *row = 0xFFFFFFFFu;
    const u32 b = unc_text_base(F, t + F.slop);
    uint2 r = make_uint2(unc_L2(ix, b) + 1u, unc_L2(ix, b + 1u));
    for (u64 p = t + F.slop; p > t;) { p--; r = unc_bwa_neighbor(ix, r.x, r.y, unc_text_base(F, p)); }
    return r;
}

// Warp-wide: the row of suffix t of every lane whose `act` is set.  The warp scans the lanes' ranges one after the
// other, 32 rows at a time, for the row whose SA value is t.  0xFFFFFFFF (not a row of a < 2^32 - 256 index) when the
// scan finds none, which a consistent index cannot give.
UNC_DEV u32 unc_suffix_row(const DevIndex &ix, const DevFms &F, u64 t, bool act) {
    u32 row = 0xFFFFFFFFu;
    uint2 r = make_uint2(1u, 0u);
    if (act) r = unc_suffix_range(ix, F, t, &row);
    for (u32 l = 0; l < 32u; l++) {
        const u32 rs = w_shfl(r.x, (int) l), re = w_shfl(r.y, (int) l);     // empty unless lane l scans
        const u64 tl = w_shfl64(t, (int) l);
        for (u32 b0 = rs; b0 <= re; b0 += 32u) {
            const u32 k = b0 + (u32) w_lane();
            const u32 m = w_ballot(k <= re && unc_bwa_sa(ix, k) == tl);
            if (m) {
                if (w_lane() == (int) l) row = b0 + (u32) (d_ffs(m) - 1);
                break;
            }
        }
    }
    return row;
}

// Segment pass: warp `warp` takes segments 32*warp .. 32*warp+31 of both walks (forward ones first), one per lane:
// the exact row of the segment's first position, then LF steps through the segment.
UNC_DEV void unc_fms_segments(const DevIndex &ix, const DevFms &F, u64 warp) {
    const u64 g = warp * 32u + (u64) w_lane();
    const bool act = g < 2u * F.n_seg, rev = g >= F.n_seg;
    const u64 j0 = (rev ? g - F.n_seg : g) * F.seg;
    const u64 a = rev ? F.pac_min + j0 : F.pac_min + F.n - 1u - j0;
    u32 row = unc_suffix_row(ix, F, rev ? (u64) ix.seq_len - 1u - a : a, act);
    if (!act) return;
    if (row == 0xFFFFFFFFu) { *F.miss = 1u; return; }
    u64 *out = rev ? F.rev : F.fwd;
    const u64 j1 = j0 + F.seg < F.n ? j0 + F.seg : F.n;
    out[j0] = row;
    for (u64 j = j0 + 1u; j < j1; j++) {
        const u64 p = rev ? F.pac_min + j : F.pac_min + F.n - 1u - j;
        const u32 c = rev ? 3u - unc_pac_base(F.pac, p) : unc_pac_base(F.pac, p);
        row = unc_L2(ix, c) + unc_occ_row(ix, row - 1u, c) + 1u;      // get_neighbor's start on a one-row range
        out[j] = row;
    }
}

// The reference's reverse walk (src/bwa_index.hpp:303-327) from its own anchor until it joins the segment pass's exact
// chain.  One warp.  Its scan finds the row f in its range with size() - sa(f) == pac_min: the row of suffix
// seq_len - pac_min, if that row is in the range (sa(0) = (u64)-1 matches no pac_min, so pac_min = 0 finds none).
UNC_DEV void unc_fms_fixup(const DevIndex &ix, const DevFms &F) {
    const u64 st = F.pac_min > F.slop ? F.pac_min - F.slop : 0u;
    const u32 b = 3u - unc_pac_base(F.pac, st);
    uint2 r = make_uint2(unc_L2(ix, b), unc_L2(ix, b + 1u));          // get_base_range: from L2[b], not L2[b] + 1
    for (u64 i = st + 1u; i <= F.pac_min; i++) r = unc_bwa_neighbor(ix, r.x, r.y, 3u - unc_pac_base(F.pac, i));
    const u32 f = unc_suffix_row(ix, F, (u64) ix.seq_len - F.pac_min, F.pac_min > 0u && w_lane() == 0);   // one scan
    if (w_lane() != 0) return;
    if (F.pac_min > 0u && f == 0xFFFFFFFFu) { *F.miss = 1u; return; }
    if (F.pac_min > 0u && r.x <= f && f <= r.y) r = make_uint2(f, f);
    for (u64 j = 0; j < F.n; j++) {
        if (j) r = unc_bwa_neighbor(ix, r.x, r.y, 3u - unc_pac_base(F.pac, F.pac_min + j));
        if (r.x == r.y && (u64) r.x == F.rev[j]) return;
        F.rev[j] = r.x;
    }
}
