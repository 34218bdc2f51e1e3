// tests/emul/emul_dtw_band.cpp -- the DTW sweeps on the CPU under the warp emulator: the banded sweep (unc_dtw_band.cuh) and
// k_dtw's full one (unc_dtw.cuh), one CTA of n_threads fibers taking the problems in turn as the persistent kernels do.  The
// workspace is planned, sized and carved by unc_dtw_plan.hpp, as unc_dtw_batch / unc_dtw_batch_banded plan theirs, in one
// buffer.  Test vehicle only.
#include "unc_device.cuh"   // UNC_EMUL is defined on the command line
#include "unc_dtw_plan.hpp"

#include <vector>

thread_local WarpEmu *g_warp = nullptr;

struct SweepArgs { const DevDtwBand *B; };
static void band_entry(void *vp) {
    const DevDtwBand *B = ((SweepArgs *) vp)->B;
    for (u32 pi = 0; pi < B->D.n_prob; pi++) unc_dtw_band_problem(*B, pi);
}
static void full_entry(void *vp) {
    const DevDtwBand *B = ((SweepArgs *) vp)->B;
    for (u32 pi = 0; pi < B->D.n_prob; pi++) unc_dtw_problem(B->D, pi);
}

extern "C" {

// n problems: means[mean_off[p] .. mean_off[p+1]) against kmers[kmer_off[p] .. kmer_off[p+1]).  band >= 1: the banded sweep
// (subseq 0 only); band 0: k_dtw's full sweep with subseq 0 NONE, 1 ROW or 2 COL.  Out: path (room for rows + columns pairs
// at path_off[p]), path_len, score, and (optional) every problem's breadcrumbs one after the other (banded: the in-band cells
// column-major; full: rows x columns row-major), their total in *n_bc.
int emu_dtw_sweep(const float *model_means_stdvs, int cost_kind, int subseq, float dw, float hw, float vw, uint32_t band,
                  uint32_t n, const float *means, const uint64_t *mean_off, const uint16_t *kmers, const uint64_t *kmer_off,
                  uint64_t *path, const uint64_t *path_off, uint64_t *path_len, float *score, uint8_t *bc_out,
                  uint64_t *n_bc, int n_threads) {
    if (band && subseq) return -1;
    DtwPlan P(band);
    for (u32 i = 0; i < n; i++) {
        const u64 nc = mean_off[i + 1] - mean_off[i], nr = kmer_off[i + 1] - kmer_off[i];
        if (nc == 0 || nr == 0) return -1;
        P.add((u32) nr, (u32) nc, mean_off[i], kmer_off[i], path_off[i]);
    }
    const std::vector<float> model = dtw_model_table(model_means_stdvs);
    P.stage(model.data(), means, mean_off[n], kmers, kmer_off[n]);
    P.t.path = path_off[n];
    // one buffer as the device workspace: unwritten bytes and floats stay recognisable (a read of one would show up as a
    // wrong result), and a region the layout undercounts or overlaps corrupts its neighbour
    const DtwLayout L = dtw_layout(P.t);
    std::vector<u64> ws(L.bytes / 8);
    char *w = (char *) ws.data();
    memset(w, 0xEE, L.bytes);
    std::fill((float *) (w + L.diag), (float *) (w + L.diag) + P.t.diag, -12345.0f);
    if (!band) std::fill((float *) (w + L.edge), (float *) (w + L.edge) + P.t.edge, -12345.0f);
    DevDtwBand B;
    dtw_carve(P, w, B);
    memcpy(w + L.model, P.h_model, 3 * 1024 * 4);
    memcpy(w + L.means, means, P.t.means * 4);
    memcpy(w + L.kmers, kmers, P.t.kmers * 2);
    memcpy(w + L.prob, P.prob.data(), P.prob.size() * sizeof(DevDtwProblem));
    if (band) memcpy(w + L.edge, P.col_off.data(), P.col_off.size() * 8);
    memset(w + L.queue, 0, 4);
    B.D.cost_kind = cost_kind; B.D.subseq = subseq; B.D.dw = dw; B.D.hw = hw; B.D.vw = vw;
    SweepArgs a = {&B};
    emu_run_cta(band ? band_entry : full_entry, &a, n_threads > 0 ? n_threads : 64);
    memcpy(path_len, w + L.plen, (size_t) n * 8);
    memcpy(score, w + L.score, (size_t) n * 4);
    memcpy(path + 2 * path_off[0], B.D.path + 2 * path_off[0], (path_off[n] - path_off[0]) * 16);
    if (bc_out) memcpy(bc_out, B.D.bc, P.t.bc);
    if (n_bc) *n_bc = P.t.bc;
    return 0;
}

// the workspace bytes the span aligner plans for one R x C problem (band 0: the full sweep)
uint64_t emu_dtw_plan_bytes(uint32_t R, uint32_t C, uint32_t band) {
    DtwPlan P(band);
    P.add(R, C, 0, 0, 0);
    return dtw_layout(P.t).bytes;
}

// the span aligner's launches (dtw_pack): launch[k] of problem k (rows[k] x cols[k]), 0xFFFFFFFF for a skipped one
uint32_t emu_dtw_pack(uint32_t band, uint32_t n, const uint32_t *rows, const uint32_t *cols, uint64_t budget, uint32_t *launch) {
    return dtw_pack(band, n, rows, cols, budget, launch);
}

// the in-band cells of an R x C problem at half-width band (unc_band_offsets)
uint64_t emu_dtw_band_cells(uint32_t R, uint32_t C, uint32_t band) { return unc_band_offsets(unc_band_make(R, C, band), nullptr); }

}  // extern "C"
