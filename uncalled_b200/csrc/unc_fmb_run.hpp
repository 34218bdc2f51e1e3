// unc_fmb_run.hpp -- the launch sequence of the device FM-index builder, written once for the library
// (unc_fmb_host.inl, CUDA) and for the emulator build of the tests (tests/emul/emul_index_build.cpp).  The round loop
// is data-dependent: how many doubling rounds run, which rows are active and where the batches end follow from the
// input, and both builds take them from here.
//
// `Dev` supplies memory and execution:
//   T *alloc<T>(u64 count)            nullptr, and error() UNC_E_NOMEM from then on, when it does not fit
//   void release(void *)
//   void zero(void *, u64 bytes); void h2d(void *, const void *, u64); void d2h(void *, const void *, u64);
//   void d2d(void *, const void *, u64)
//   u32 get(const u32 *)              one value, after the work queued so far
//   void each(const F &, u64 count)   a per-element functor of unc_fmb.cuh
//   void tiles(const F &, u64 n_tiles) a CTA functor of unc_fmb.cuh
//   void mark(int)                    phase boundaries 0..3 (timing)
//   int error()                       UNC_OK, or the first failure
#pragma once
#include <algorithm>
#include <vector>

#include "unc_fmb.cuh"
#include "unc_index_host.hpp"

#define UNC_FMB_DEFAULT_WS_ROWS (1ull << 26)   // rows of a doubling batch's sort workspace (grown to the largest group)

struct FmbConfig {
    u64 ws_rows = 0;      // 0 = UNC_FMB_DEFAULT_WS_ROWS
};

struct FmbResult {
    u64 primary = 0;
    std::vector<u32> bwt;          // the .bwt payload after primary and L2
    std::vector<u64> sa;           // the .sa samples SA[32], SA[64], ...
    u32 k0 = 0, rounds = 0;
    u64 ws_rows = 0, max_bucket = 0;
    std::vector<u64> active;       // active rows per doubling round
    std::vector<u64> batches;      // batches per doubling round
};

// bases of the initial counting sort: about log4(n), at most UNC_FMB_K0_MAX
static inline u32 unc_fmb_k0(u64 n) {
    u32 k = 1;
    while (k < UNC_FMB_K0_MAX && (1ull << (2 * k)) < n) k++;
    return k;
}

static inline u32 unc_fmb_bits(u64 v) {
    u32 b = 0;
    while (b < 64 && (v >> b)) b++;
    return b;
}

// device bytes of a build of n symbols with a sort workspace of ws rows: the text, the head bits, SA and ISA throughout,
// then the largest of the initial sort's bucket arrays, the rounds' A and K and workspace, and the output (ISA freed);
// plus the per-tile counts of the compaction and the scans' tile aggregates
static inline u64 unc_fmb_device_bytes(u64 n, u64 ws) {
    const u64 N = n + 1;
    ws = std::min<u64>(ws, N);
    const u64 base = (((n + 15) >> 4) + 2) * 4 + ((N >> 5) + 3) * 4 + 8 * N;
    const u64 initial = 2 * (1ull << (2 * unc_fmb_k0(n))) * 4;
    const u64 rounds = 8 * N + ws * (8 + 8 + 4 + 4) + 256 * ((ws + UNC_FMB_RADIX_TILE - 1) / UNC_FMB_RADIX_TILE) * 4;
    const u64 output = unc_bwa_bwt_words(n) * 4 + 16 * ((n + 127) / 128) + unc_bwa_n_sa(n) * 8;
    const u64 small = (N / UNC_FMB_ROWS_PER_TILE + 1) * 4 + (std::max<u64>(N, 1ull << 24) / UNC_FMB_SCAN_TILE + 2) * 4;
    return base + std::max(initial, std::max(rounds, output)) + small + (1u << 20);
}

namespace fmb {

template <class Dev>
struct Scanner {                   // the device-wide scan of unc_fmb.cuh, with its aggregate buffer
    Dev &d;
    u32 *part = nullptr, *total = nullptr;
    u64 cap = 0;
    explicit Scanner(Dev &dev) : d(dev) {}
    ~Scanner() { d.release(part); d.release(total); }
    // scan x[0, n) in place; returns the aggregate (including init), or 0 after a failure (see d.error())
    u32 run(u32 *x, u64 n, u32 is_max, u32 inclusive, u32 init) {
        const u64 nt = (n + UNC_FMB_SCAN_TILE - 1) / UNC_FMB_SCAN_TILE;
        if (!total && !(total = d.template alloc<u32>(1))) return 0;
        if (nt > cap) {
            d.release(part);
            if (!(part = d.template alloc<u32>(nt))) { cap = 0; return 0; }
            cap = nt;
        }
        FmbScan s;
        s.x = x; s.n = n; s.part = part; s.n_tiles = nt; s.is_max = is_max; s.inclusive = inclusive; s.init = init;
        s.total = total;
        if (nt) d.tiles(FmbScanReduce{s}, nt);
        d.tiles(FmbScanParts{s}, 1);
        if (nt) d.tiles(FmbScanApply{s}, nt);
        return d.get(total);
    }
};

template <class Dev>
struct Buf {                       // a device allocation released on every exit path
    Dev &d;
    void *p = nullptr;
    explicit Buf(Dev &dev) : d(dev) {}
    ~Buf() { d.release(p); }
    template <typename T> T *get(u64 count) {
        d.release(p);
        p = d.template alloc<T>(count ? count : 1);
        return (T *) p;
    }
    void drop() { d.release(p); p = nullptr; }
};

}  // namespace fmb

// The suffix array of text (n symbols packed as unc_fmb.cuh describes, ((n + 15) >> 4) + 2 words), then the .bwt
// payload and the .sa samples.  counts[c] = the occurrences of symbol c in the text.  Returns UNC_OK, UNC_E_NOMEM when
// an allocation fails, or the Dev's error.
template <class Dev>
int unc_fmb_run(Dev &d, const std::vector<u32> &text_words, u64 n, const u64 counts[4], const FmbConfig &cfg,
                FmbResult &res) {
    using fmb::Buf;
    const u64 N = n + 1, head_words = (N >> 5) + 3;
    const u32 k0 = unc_fmb_k0(n);
    const u64 n_buckets = 1ull << (2 * k0);
    res = FmbResult();
    res.k0 = k0;
    fmb::Scanner<Dev> scan(d);
    Buf<Dev> b_text(d), b_SA(d), b_ISA(d), b_head(d), b_start(d), b_cursor(d);
    u32 *text = b_text.template get<u32>(text_words.size());
    u32 *SA = b_SA.template get<u32>(N), *ISA = b_ISA.template get<u32>(N);
    u32 *head = b_head.template get<u32>(head_words);
    u32 *start = b_start.template get<u32>(n_buckets), *cursor = b_cursor.template get<u32>(n_buckets);
    if (!text || !SA || !ISA || !head || !start || !cursor) return UNC_E_NOMEM;
    d.mark(0);
    d.h2d(text, text_words.data(), text_words.size() * 4);
    d.zero(head, head_words * 4);
    d.zero(start, n_buckets * 4);

    // ---- initial sort: counting sort on the first k0 bases; row 0 is the sentinel's
    d.each(FmbHist{text, start, k0}, n);
    d.d2d(cursor, start, n_buckets * 4);
    res.max_bucket = scan.run(cursor, n_buckets, 1, 0, 0);
    scan.run(start, n_buckets, 0, 0, 1);
    d.d2d(cursor, start, n_buckets * 4);
    d.each(FmbScatter{text, start, cursor, SA, ISA, head, k0}, n);
    d.each(FmbSentinel{SA, ISA, head, n}, 1);
    b_start.drop();
    b_cursor.drop();
    if (d.error() != UNC_OK) return d.error();
    d.mark(1);

    // ---- doubling rounds over the rows of unsorted groups
    res.ws_rows = std::max<u64>(std::min<u64>(cfg.ws_rows ? cfg.ws_rows : UNC_FMB_DEFAULT_WS_ROWS, N), res.max_bucket);
    const u64 ws = res.ws_rows, rtiles_max = (ws + UNC_FMB_RADIX_TILE - 1) / UNC_FMB_RADIX_TILE;
    const u64 act_tiles = (N + UNC_FMB_ROWS_PER_TILE - 1) / UNC_FMB_ROWS_PER_TILE;
    Buf<Dev> b_tc(d), b_A(d), b_K(d), b_key0(d), b_key1(d), b_val0(d), b_val1(d), b_hist(d);
    u32 *tile_cnt = b_tc.template get<u32>(act_tiles);
    u64 *key0 = b_key0.template get<u64>(ws), *key1 = b_key1.template get<u64>(ws);
    u32 *val0 = b_val0.template get<u32>(ws), *val1 = b_val1.template get<u32>(ws);
    u32 *hist = b_hist.template get<u32>(256 * rtiles_max);
    if (!tile_cnt || !key0 || !key1 || !val0 || !val1 || !hist) return UNC_E_NOMEM;
    const u32 kbits = unc_fmb_bits(N + UNC_FMB_KOFF);
    for (u64 h = k0;; h *= 2) {
        FmbActive act{head, N, tile_cnt, nullptr, 0};
        d.tiles(act, act_tiles);
        const u64 M = scan.run(tile_cnt, act_tiles, 0, 0, 0);
        if (d.error() != UNC_OK) return d.error();
        if (M == 0) break;
        if (res.rounds == 64) return UNC_E_ARG;       // cannot happen: every round doubles the sorted prefix
        res.rounds++;
        res.active.push_back(M);
        u32 *A = b_A.template get<u32>(M), *K = b_K.template get<u32>(M);
        if (!A || !K) return UNC_E_NOMEM;
        act.A = A;
        act.compact = 1;
        d.tiles(act, act_tiles);
        d.each(FmbSnapshot{A, SA, ISA, K, n, h}, M);
        u64 n_batches = 0;
        for (u64 p0 = 0; p0 < M;) {
            // a batch ends at a group's first row: the group of the row at p0 + ws starts ISA[SA[row]]
            u64 p1 = M;
            if (p0 + ws < M) {
                const u32 g = d.get(A + p0 + ws), gs = d.get(ISA + d.get(SA + g));
                p1 = p0 + ws - (g - gs);
            }
            if (d.error() != UNC_OK) return d.error();
            if (p1 <= p0) return UNC_E_ARG;           // cannot happen: no group is larger than the workspace
            const u64 m = p1 - p0;
            const u32 g0 = d.get(A + p0), span = d.get(A + p1 - 1) - g0;
            d.each(FmbKeys{A, SA, ISA, K, p0, g0, key0, val0}, m);
            FmbRadix r;
            r.m = m;
            r.n_tiles = (m + UNC_FMB_RADIX_TILE - 1) / UNC_FMB_RADIX_TILE;
            r.hist = hist;
            u64 *kin = key0, *kout = key1;
            u32 *vin = val0, *vout = val1;
            const u32 rbits = unc_fmb_bits(span);
            for (u32 shift = 0; shift < 64; shift += 8) {
                if (shift < 32 ? shift >= kbits : shift - 32 >= rbits) continue;
                r.key_in = kin; r.val_in = vin; r.key_out = kout; r.val_out = vout; r.shift = shift;
                d.tiles(FmbRadixHist{r}, r.n_tiles);
                scan.run(hist, 256 * r.n_tiles, 0, 0, 0);
                d.tiles(FmbRadixScatter{r}, r.n_tiles);
                std::swap(kin, kout);
                std::swap(vin, vout);
            }
            u32 *mark = vout;
            d.each(FmbWriteback{A, p0, kin, vin, SA, head, mark}, m);
            scan.run(mark, m, 1, 1, 0);
            d.each(FmbRank{vin, mark, ISA}, m);
            if (d.error() != UNC_OK) return d.error();
            n_batches++;
            p0 = p1;
        }
        res.batches.push_back(n_batches);
    }
    for (Buf<Dev> *b : {&b_tc, &b_A, &b_K, &b_key0, &b_key1, &b_val0, &b_val1, &b_hist}) b->drop();
    d.mark(2);

    // ---- outputs: primary, the Occ-interleaved BWT, the sampled SA
    res.primary = d.get(ISA);
    b_ISA.drop();
    const u64 n_words = unc_bwa_bwt_words(n), nb = (n + 127) / 128, n_sa = unc_bwa_n_sa(n);
    Buf<Dev> b_out(d), b_cnt(d), b_sa(d);
    u32 *out = b_out.template get<u32>(n_words), *cnt = b_cnt.template get<u32>(4 * nb);
    u64 *sa = b_sa.template get<u64>(n_sa - 1);
    if (!out || !cnt || !sa) return UNC_E_NOMEM;
    d.each(FmbBwt{text, SA, n, res.primary, out}, (n + 15) / 16);
    d.each(FmbOccCount{out, n, nb, cnt}, nb);
    scan.run(cnt, 4 * nb, 0, 0, 0);
    FmbOccWrite ow{cnt, nb, n_words, {counts[0], counts[1], counts[2], counts[3]}, out};
    d.each(ow, nb + 1);
    d.each(FmbSaSample{SA, sa}, n_sa - 1);
    res.bwt.resize(n_words);
    res.sa.resize(n_sa - 1);
    d.d2h(res.bwt.data(), out, n_words * 4);
    d.d2h(res.sa.data(), sa, (n_sa - 1) * 8);
    d.mark(3);
    return d.error();
}

// the packed text of unc_fmb.cuh from the forward codes: forward, then the reverse complement
static inline void unc_fmb_pack_text(const std::vector<uint8_t> &fwd, std::vector<u32> &words, u64 counts[4]) {
    const u64 l = fwd.size(), n = 2 * l;
    words.assign(((n + 15) >> 4) + 2, 0u);
    for (int c = 0; c < 4; c++) counts[c] = 0;
    for (u64 i = 0; i < l; i++) {
        const u32 f = fwd[i], r = 3u - fwd[l - 1 - i];
        words[i >> 4] |= f << ((15u - (u32) (i & 15)) << 1);
        words[(l + i) >> 4] |= r << ((15u - (u32) ((l + i) & 15)) << 1);
        counts[f]++;
        counts[r]++;
    }
}

// seq_len = 2 l_pac of the FASTA, counted without parsing it: UNC_E_IO for a missing file or no bases,
// UNC_E_TOO_LARGE at UNC_BWA_DEVICE_MAX_ROWS or more (what unc_index_load refuses)
static inline int unc_fmb_check_size(const char *fasta_path, u64 *seq_len) {
    uint64_t l_pac = 0;
    const int rc = unc_bwa_count_bases(fasta_path, &l_pac);
    if (rc != UNC_OK) return rc;
    if (l_pac == 0) return UNC_E_IO;
    if (2 * l_pac >= UNC_BWA_DEVICE_MAX_ROWS) return UNC_E_TOO_LARGE;
    *seq_len = 2 * l_pac;
    return UNC_OK;
}

// parse, sort and write the five files; nothing is written unless the sort succeeded
template <class Dev>
int unc_fmb_build_files(Dev &d, const char *fasta_path, const std::string &prefix, const FmbConfig &cfg,
                        FmbResult &res) {
    u64 L2[5], counts[4];
    BwaRef R;
    int rc = unc_bwa_read_fasta(fasta_path, R);
    if (rc != UNC_OK) return rc;
    const u64 n = 2 * (u64) R.fwd.size();
    if (n == 0) return UNC_E_IO;
    if (n >= UNC_BWA_DEVICE_MAX_ROWS) return UNC_E_TOO_LARGE;
    {
        std::vector<u32> words;
        unc_fmb_pack_text(R.fwd, words, counts);
        if ((rc = unc_fmb_run(d, words, n, counts, cfg, res)) != UNC_OK) return rc;
    }
    unc_bwa_l2(counts, L2);
    if ((rc = unc_bwa_write_pac_ann_amb(R, prefix)) != UNC_OK) return rc;
    if ((rc = unc_bwa_write_bwt(prefix, res.primary, L2, res.bwt.data(), res.bwt.size())) != UNC_OK) return rc;
    return unc_bwa_write_sa(prefix, res.primary, L2, n, res.sa.data());
}
