// tests/emul/emul_dtw_band.cpp -- the banded DTW sweep (unc_dtw_band.cuh) and, for comparison, k_dtw's routine
// (unc_dtw.cuh) on the CPU under the warp emulator, one CTA of n_threads fibers taking the problems in turn as the
// persistent kernels do.  Workspace carved as unc_dtw_batch / unc_dtw_batch_banded carve it.  Test vehicle only.
#include "unc_device.cuh"   // UNC_EMUL is defined on the command line
#include "unc_dtw_band.cuh"

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

// n problems: means[mean_off[p] .. mean_off[p+1]) against kmers[kmer_off[p] .. kmer_off[p+1]), subseq NONE.  band >= 1:
// the banded sweep; band 0: k_dtw's full sweep.  Out: path (room for rows + columns pairs at path_off[p]), path_len,
// score, and (optional) every problem's breadcrumbs one after the other (banded: the in-band cells column-major; full:
// rows x columns row-major), their total in *n_bc.
int emu_dtw_sweep(const float *model_means_stdvs, int cost_kind, float dw, float hw, float vw, uint32_t band, uint32_t n,
                  const float *means, const uint64_t *mean_off, const uint16_t *kmers, const uint64_t *kmer_off,
                  uint64_t *path, const uint64_t *path_off, uint64_t *path_len, float *score, uint8_t *bc_out,
                  uint64_t *n_bc, int n_threads) {
    std::vector<float> model(3 * 1024);
    for (u32 k = 0; k < 1024; k++) {
        const float mean = model_means_stdvs[2 * k], stdv = model_means_stdvs[2 * k + 1];
        model[k] = mean;
        model[1024 + k] = 2 * stdv * stdv;
        model[2048 + k] = (float) std::log(std::sqrt(M_PI * model[1024 + k]));
    }
    std::vector<DevDtwProblem> prob(n);
    std::vector<u64> col_off;
    u64 bc_total = 0, diag_total = 0, edge_total = 0;
    for (u32 i = 0; i < n; i++) {
        const u64 nc = mean_off[i + 1] - mean_off[i], nr = kmer_off[i + 1] - kmer_off[i];
        if (nc == 0 || nr == 0) return -1;
        DevDtwProblem &P = prob[i];
        P.mean_off = mean_off[i]; P.kmer_off = kmer_off[i]; P.n_cols = (u32) nc; P.n_rows = (u32) nr;
        P.bc_off = bc_total; P.diag_off = diag_total; P.edge_off = edge_total; P.path_off = path_off[i];
        diag_total += UNC_DTW_WORK_FLOATS(nr, nc);
        if (band) {
            col_off.resize(edge_total + nc + 1);
            bc_total += unc_band_offsets(unc_band_make((u32) nr, (u32) nc, band), col_off.data() + edge_total);
            edge_total += nc + 1;
        } else {
            bc_total += nr * nc; edge_total += nr + nc;
        }
    }
    // unwritten bytes and floats stay recognisable (a read of one would show up as a wrong result)
    std::vector<unsigned char> bc(bc_total + 1, 0xEE);
    std::vector<float> diag(diag_total + 1, -12345.0f), edge(band ? 1 : edge_total + 1, -12345.0f);
    u32 queue = 0;
    DevDtwBand B;
    DevDtw &D = B.D;
    D.model = model.data(); D.means = means; D.kmers = kmers; D.prob = prob.data(); D.n_prob = n;
    D.bc = bc.data(); D.diag = diag.data(); D.edge = edge.data(); D.path = path; D.path_len = path_len; D.score = score;
    D.cost_kind = cost_kind; D.subseq = 0; D.dw = dw; D.hw = hw; D.vw = vw; D.queue = &queue;
    B.col_off = col_off.data(); B.band = band;
    SweepArgs a = {&B};
    emu_run_cta(band ? band_entry : full_entry, &a, n_threads > 0 ? n_threads : 64);
    if (bc_out) memcpy(bc_out, bc.data(), bc_total);
    if (n_bc) *n_bc = bc_total;
    return 0;
}

// the in-band cells of an R x C problem at half-width band (unc_band_offsets)
uint64_t emu_dtw_band_cells(uint32_t R, uint32_t C, uint32_t band) { return unc_band_offsets(unc_band_make(R, C, band), nullptr); }

}  // extern "C"
