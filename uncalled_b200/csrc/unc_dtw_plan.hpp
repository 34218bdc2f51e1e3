// unc_dtw_plan.hpp -- the host-side plan of a DTW sweep (k_dtw, k_dtw_band): the problem table and the layout of the sweep's
// workspace, for unc_dtw_batch, the span aligner's launches and the emulator.  Host code only (no CUDA runtime call), so it
// compiles both in unc_abi.cu and in the emulator libraries.
//
// The workspace is one buffer of 256-byte aligned regions, in this order: inputs staged by the plan (the 3 x 1024 model table,
// the means, the k-mers; the aligner's stay in its own buffers), the problem table, the breadcrumbs, the work arrays
// (hrow / vcol / corners), the full sweep's last column and row or the banded sweep's column offsets, the path room, the path
// lengths, the scores and the queue counter.  dtw_layout is the only place that decides it: the byte count and the carve both
// come from it.
#pragma once
#include "unc_dtw_band.cuh"

#include <algorithm>
#include <cmath>
#include <vector>

// PoreModel(means_stdvs, false)'s tables as the sweeps read them: means, 2 stdv^2, log norm (reference
// src/pore_model.hpp:58-62,77-103)
inline std::vector<float> dtw_model_table(const float *model_means_stdvs) {
    std::vector<float> model(3 * 1024);
    for (uint32_t k = 0; k < 1024; k++) {
        const float mean = model_means_stdvs[2 * k], stdv = model_means_stdvs[2 * k + 1];
        model[k] = mean;
        model[1024 + k] = 2 * stdv * stdv;
        model[2048 + k] = (float) std::log(std::sqrt(M_PI * model[1024 + k]));
    }
    return model;
}

inline size_t dtw_align(size_t x) { return (x + 255) & ~(size_t) 255; }

// breadcrumb bytes of an nr x nc problem: every cell, or (band >= 1) the in-band cells
inline u64 dtw_cells(u32 nr, u32 nc, u32 band) {
    return band ? unc_band_offsets(unc_band_make(nr, nc, band), nullptr) : (u64) nr * nc;
}

// What the layout is computed from.  Copying it is O(1), so a planner can try one more problem before committing to it.
struct DtwTotals {
    u32 band = 0;                    // 0: the full sweep; else the banded sweep's half-width W
    u64 n = 0, bc = 0, diag = 0;     // problems, breadcrumb bytes (= cells swept), work floats
    u64 edge = 0, path = 0;          // last-column and last-row floats (full) or column offsets (banded); path room in pairs
    bool staged = false;             // inputs in the workspace: the model table, `means` floats and `kmers` codes
    u64 means = 0, kmers = 0;

    explicit DtwTotals(u32 band_ = 0) : band(band_) {}
    // one more nr x nc problem with `cells` breadcrumbs, its path at path_off with room for nr + nc pairs
    void add(u32 nr, u32 nc, u64 cells, u64 path_off) {
        n++;
        bc += cells;
        diag += UNC_DTW_WORK_FLOATS((u64) nr, (u64) nc);
        edge += band ? (u64) nc + 1 : (u64) nr + nc;
        path = std::max<u64>(path, path_off + nr + nc);
    }
};

// byte offsets of the regions, and the whole
struct DtwLayout {
    size_t model, means, kmers, prob, bc, diag, edge, path, plen, score, queue, bytes;
};
inline DtwLayout dtw_layout(const DtwTotals &t) {
    DtwLayout L;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += dtw_align(bytes); return o; };
    L.model = take(t.staged ? 3 * 1024 * 4 : 0); L.means = take(t.means * 4); L.kmers = take(t.kmers * 2);
    L.prob = take(t.n * sizeof(DevDtwProblem)); L.bc = take(t.bc); L.diag = take(t.diag * 4);
    L.edge = take(t.edge * (t.band ? 8 : 4)); L.path = take(t.path * 16); L.plen = take(t.n * 8); L.score = take(t.n * 4);
    L.queue = take(4);
    L.bytes = off;
    return L;
}

// The problems of one sweep.
struct DtwPlan {
    DtwTotals t;
    std::vector<DevDtwProblem> prob;
    std::vector<u64> col_off;        // banded: C + 1 offsets per problem, at its edge_off
    u64 max_we = 0;                  // banded: the widest effective half-width (threads per CTA)
    const float *h_model = nullptr, *h_means = nullptr;   // staged inputs (stage())
    const u16 *h_kmers = nullptr;

    explicit DtwPlan(u32 band) : t(band) {}
    // means[mean_off ..) of nc columns against kmers[kmer_off ..) of nr rows, its path at path_off
    void add(u32 nr, u32 nc, u64 mean_off, u64 kmer_off, u64 path_off) {
        DevDtwProblem P;
        P.mean_off = mean_off; P.kmer_off = kmer_off; P.n_cols = nc; P.n_rows = nr;
        P.bc_off = t.bc; P.diag_off = t.diag; P.edge_off = t.edge; P.path_off = path_off;
        u64 cells = (u64) nr * nc;
        if (t.band) {
            const UncBand b = unc_band_make(nr, nc, t.band);
            col_off.resize(t.edge + nc + 1);
            cells = unc_band_offsets(b, col_off.data() + t.edge);
            max_we = std::max<u64>(max_we, b.we);
        }
        t.add(nr, nc, cells, path_off);
        prob.push_back(P);
    }
    // carry the host inputs in the workspace: model (3 x 1024, dtw_model_table), means[0 .. n_means), kmers[0 .. n_kmers)
    void stage(const float *model, const float *means, u64 n_means, const u16 *kmers, u64 n_kmers) {
        h_model = model; h_means = means; h_kmers = kmers;
        t.staged = true; t.means = n_means; t.kmers = n_kmers;
    }
};

// Points B's workspace fields (and the inputs, when the plan stages them) into the workspace at base, laid out by dtw_layout.
// The caller sets the cost parameters, and the inputs when they are not staged.
inline void dtw_carve(const DtwPlan &P, char *base, DevDtwBand &B) {
    const DtwLayout L = dtw_layout(P.t);
    DevDtw &D = B.D;
    if (P.t.staged) {
        D.model = (const float *) (base + L.model); D.means = (const float *) (base + L.means); D.kmers = (const u16 *) (base + L.kmers);
    }
    D.prob = (const DevDtwProblem *) (base + L.prob); D.n_prob = (u32) P.t.n;
    D.bc = (unsigned char *) (base + L.bc); D.diag = (float *) (base + L.diag); D.edge = (float *) (base + L.edge);
    D.path = (u64 *) (base + L.path); D.path_len = (u64 *) (base + L.plen); D.score = (float *) (base + L.score);
    D.queue = (u32 *) (base + L.queue);
    B.col_off = (const u64 *) (base + L.edge); B.band = P.t.band;
}

const u32 DTW_SKIP = 0xFFFFFFFFu;

// The aligner's launches: n problems (rows[k] x cols[k], paths packed) in order, a launch closed when the next problem would
// take its workspace past `budget` bytes.  launch[k]: the launch of problem k, or DTW_SKIP when it alone exceeds the budget.
// Returns the number of launches.
inline u32 dtw_pack(u32 band, u32 n, const u32 *rows, const u32 *cols, u64 budget, u32 *launch) {
    u32 n_launch = 0;
    DtwTotals need(band);
    for (u32 k = 0; k < n; k++) {
        const u64 cells = dtw_cells(rows[k], cols[k], band);
        DtwTotals t = need;
        t.add(rows[k], cols[k], cells, t.path);
        if (need.n && dtw_layout(t).bytes > budget) {          // the launch is full: this problem opens the next one
            n_launch++;
            t = need = DtwTotals(band);
            t.add(rows[k], cols[k], cells, 0);
        }
        if (dtw_layout(t).bytes > budget) { launch[k] = DTW_SKIP; continue; }
        need = t;
        launch[k] = n_launch;
    }
    return n_launch + (need.n ? 1u : 0u);
}
