// tests/emul/emul_mask_external.cpp -- the device source of `mask-external` (uncalled_b200/csrc/unc_mask_ext.cuh) on
// the CPU under the warp emulator, around the same host steps as unc_mask_external
// (uncalled_b200/csrc/unc_mask_ext_host.inl).  The CTAs of a launch run one after the other, and the build and mark
// threads one after the other: both are orders the GPU may take.
#include <algorithm>
#include <vector>

#include "warp_emul.hpp"      // UNC_EMUL is defined on the command line

// the emulator's counterpart of unc_warp.cuh's 16-byte compare-and-swap: the lanes of the emulator run one at a time
// and switch only inside warp primitives, so a plain compare and store is atomic
static inline unsigned __int128 d_atomic_cas128(unsigned __int128 *p, unsigned __int128 cmp, unsigned __int128 v) {
    unsigned __int128 o = *p;
    if (o == cmp) *p = v;
    return o;
}

#include "unc_mask_ext.cuh"
#include "unc_mask_ext_host.hpp"

thread_local WarpEmu *g_warp = nullptr;

namespace {
struct TileArg { const DevMxCount *P; u64 tile; u32 *s_tile; };
void tile_entry(void *p) { TileArg *a = (TileArg *) p; unc_mx_count_tile(*a->P, a->tile, a->s_tile); }
}  // namespace

// n_threads: threads per count CTA (a multiple of 32, at most UNC_MX_MAX_THREADS).  cap / filter_bits: powers of two
// that replace the table's and the filter's sizes (0 = the library's); cap must exceed the target's distinct keys.
// Returns UNC_OK, or the status unc_mask_external gives before it needs a device.
extern "C" int emu_mask_external(const char *full_fasta, const char *target_fasta, uint32_t min_len, uint32_t min_copy,
                                 const char *out_fasta, const char *out_bed, uint64_t piece_bases, int n_threads,
                                 uint64_t cap, uint64_t filter_bits, uint32_t *window_counts, uint64_t *n_selected,
                                 uint64_t *n_masked_bp) {
    if (n_threads < 32 || n_threads % 32 || n_threads > (int) UNC_MX_MAX_THREADS) return UNC_E_ARG;
    std::string err;
    int rc = unc_mx_check_args(min_len, min_copy, out_fasta, out_bed, err);
    if (rc != UNC_OK) { fprintf(stderr, "%s\n", err.c_str()); return rc; }
    MaskFasta Tg, G;
    if ((rc = unc_mask_read_fasta(target_fasta, Tg)) != UNC_OK) { fprintf(stderr, "%s\n", Tg.error.c_str()); return rc; }
    if ((rc = unc_mask_read_fasta(full_fasta, G)) != UNC_OK) { fprintf(stderr, "%s\n", G.error.c_str()); return rc; }
    const uint32_t k = min_len;
    const uint64_t n = Tg.seq.size(), T = (uint64_t) n_threads * UNC_MX_W;
    std::vector<uint8_t> codes(n);
    unc_mask_codes(Tg, codes.data());
    uint64_t c0 = 0, f0 = 0;
    if (unc_mx_table_size(unc_mx_count_windows(codes.data(), n, k), &c0, &f0) != UNC_OK) return UNC_E_TOO_LARGE;
    DevMxTable t;
    t.cap = cap ? cap : c0;
    t.filter_bits = filter_bits ? filter_bits : f0;
    t.k = k;
    std::vector<u128> keys(t.cap, ~(u128) 0);
    std::vector<u32> cnt(t.cap, 0), ovf((t.cap + 31) / 32, 0), filter((t.filter_bits + 31) / 32, 0), slot(n), counts(n);
    t.keys = keys.data(); t.cnt = cnt.data(); t.ovf = ovf.data(); t.filter = filter.data();
    const uint64_t chunks = (n + UNC_MX_W - 1) / UNC_MX_W;
    DevMxBuild B;
    B.t = t; B.codes = codes.data(); B.n = n; B.slot = slot.data();
    for (u64 c = 0; c < chunks; c++) unc_mx_build_chunk(B, c);

    const MxPieces pc(G.seq.size(), k, piece_bases);
    const uint64_t piece_tiles = (std::min(pc.piece, std::max<uint64_t>(pc.n_starts, 1)) + T - 1) / T;
    // 16-byte aligned like cudaMalloc's (the tile loads are uint4); bytes past a piece are left from the previous one
    std::vector<uint4> buf((piece_tiles * T + UNC_MX_HALO) / 16);
    std::vector<u32> s_tile(UNC_MX_TILE_WORDS(UNC_MX_MAX_THREADS));
    for (uint64_t i = 0; i < pc.n_pieces; i++) {
        const uint64_t starts = pc.starts(i);
        memcpy(buf.data(), G.seq.data() + pc.off(i), starts + k - 1);
        DevMxCount P;
        P.t = t; P.bytes = (const u8 *) buf.data(); P.n_starts = starts; P.n_tiles = (starts + T - 1) / T;
        for (u64 tl = 0; tl < P.n_tiles; tl++) {
            TileArg a = {&P, tl, s_tile.data()};
            emu_run_cta(tile_entry, &a, n_threads);
        }
    }

    DevMxMark M;
    M.t = t; M.slot = slot.data(); M.codes = codes.data(); M.counts = counts.data(); M.n = n; M.min_copy = min_copy;
    for (u64 c = 0; c < chunks; c++) unc_mx_mark_chunk(M, c);
    if (window_counts) std::copy(counts.begin(), counts.end(), window_counts);
    if ((rc = unc_mx_write_outputs(Tg, codes.data(), counts.data(), min_copy, out_fasta, out_bed, n_selected,
                                   n_masked_bp, err)) != UNC_OK) {
        fprintf(stderr, "%s\n", err.c_str());
        return rc;
    }
    return UNC_OK;
}
