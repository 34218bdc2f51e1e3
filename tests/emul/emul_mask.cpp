// tests/emul/emul_mask.cpp -- the device source of `mask-internal` (uncalled_b200/csrc/unc_mask.cuh) on the CPU under
// the warp emulator, around the same host steps as unc_mask_internal (uncalled_b200/csrc/unc_mask_host.inl).  The
// CTAs of a launch run one after the other; with ping-pong buffers that is one of the orders the GPU may take.
#include <algorithm>
#include <vector>

#include "unc_mask.cuh"   // UNC_EMUL is defined on the command line
#include "unc_mask_host.hpp"

thread_local WarpEmu *g_warp = nullptr;

namespace {
struct TileArg { const DevMaskPass *P; u64 tile; u32 *s_in, *s_out; };
void tile_entry(void *p) { TileArg *a = (TileArg *) p; unc_mask_tile(*a->P, a->tile, a->s_in, a->s_out); }
struct ArgmaxArg { const DevMaskArgmax *A; u32 blk; u64 *s_red; };
void part_entry(void *p) { ArgmaxArg *a = (ArgmaxArg *) p; unc_mask_argmax_part(*a->A, a->blk, a->s_red); }
void final_entry(void *p) { ArgmaxArg *a = (ArgmaxArg *) p; unc_mask_argmax_final(*a->A, a->s_red); }
}  // namespace

// n_threads: threads per CTA (a multiple of 32, at most UNC_MASK_MAX_THREADS): the tile is n_threads x UNC_MASK_W
// positions.  Returns UNC_OK, or the status unc_mask_internal gives before it needs a device.
extern "C" int emu_mask_internal(const char *fasta_in, const char *out_fasta, uint32_t k, uint32_t iters, int n_threads,
                                 uint64_t *kmer_codes, uint64_t *counts, uint32_t *n_done) {
    if (k < 1 || k > UNC_MASK_MAX_K || iters < 1 || n_threads < 32 || n_threads % 32 || n_threads > (int) UNC_MASK_MAX_THREADS)
        return UNC_E_ARG;
    MaskFasta F;
    int rc = unc_mask_read_fasta(fasta_in, F);
    if (rc != UNC_OK) { fprintf(stderr, "%s\n", F.error.c_str()); return rc; }
    const uint64_t n = F.seq.size(), T = (uint64_t) n_threads * UNC_MASK_W;
    const uint64_t n_tiles = (n + T - 1) / T, bytes = UNC_MASK_PAD + n_tiles * T + UNC_MASK_PAD;
    const uint32_t n_bins = 1u << (2 * k), n_part = std::min<uint32_t>(1024u, (n_bins + 4095u) / 4096u);
    // 16-byte aligned like cudaMalloc's (the tile loads are uint4)
    std::vector<uint4> b0((bytes + 15) / 16), b1((bytes + 15) / 16);
    u8 *buf[2] = {(u8 *) b0.data(), (u8 *) b1.data()};
    memset(buf[0], UNC_MASK_BRK, bytes);
    unc_mask_codes(F, buf[0] + UNC_MASK_PAD);
    memcpy(buf[1], buf[0], bytes);
    std::vector<u32> hist(n_bins, 0), s_in(UNC_MASK_IN_WORDS(UNC_MASK_MAX_THREADS)), s_out(UNC_MASK_OUT_WORDS(UNC_MASK_MAX_THREADS));
    std::vector<u64> part(n_part), sel(iters), s_red(32);
    int cur = 0;
    for (uint32_t p = 0; p <= iters; p++) {
        DevMaskPass P;
        P.src = buf[cur]; P.dst = buf[cur ^ 1]; P.n_tiles = n_tiles; P.k = k;
        P.hist = p < iters ? hist.data() : nullptr;
        P.prev = p ? sel.data() + (p - 1) : nullptr;
        for (u64 t = 0; t < n_tiles; t++) {
            TileArg a = {&P, t, s_in.data(), s_out.data()};
            emu_run_cta(tile_entry, &a, n_threads);
        }
        cur ^= 1;
        if (p < iters) {
            DevMaskArgmax A;
            A.hist = hist.data(); A.n_bins = n_bins; A.part = part.data(); A.n_part = n_part; A.sel = sel.data() + p;
            for (u32 blk = 0; blk < n_part; blk++) {
                ArgmaxArg a = {&A, blk, s_red.data()};
                emu_run_cta(part_entry, &a, 64);
            }
            ArgmaxArg a = {&A, 0, s_red.data()};
            emu_run_cta(final_entry, &a, 64);
        }
    }
    uint32_t done = 0;
    while (done < iters && (sel[done] >> 32) != 0) done++;
    for (uint32_t i = 0; i < iters; i++) {
        kmer_codes[i] = i < done ? (uint32_t) sel[i] : 0;
        counts[i] = i < done ? sel[i] >> 32 : 0;
    }
    std::string err;
    if ((rc = unc_mask_write_fasta(F, buf[cur] + UNC_MASK_PAD, out_fasta, err)) != UNC_OK) { fprintf(stderr, "%s\n", err.c_str()); return rc; }
    *n_done = done;
    return UNC_OK;
}
