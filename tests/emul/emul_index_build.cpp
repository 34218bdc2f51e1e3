// tests/emul/emul_index_build.cpp -- the device FM-index builder (uncalled_b200/csrc/unc_fmb.cuh) on the CPU under the
// warp emulator, driven by the library's own launch sequence (uncalled_b200/csrc/unc_fmb_run.hpp) and host steps
// (unc_index_host.hpp).  Per-element functors run as plain loops and the tiles of a CTA functor one after the other in
// one emulated CTA: both are orders the GPU may take.
#include <algorithm>
#include <vector>

#include "warp_emul.hpp"      // UNC_EMUL is defined on the command line

#include "unc_fmb_run.hpp"

thread_local WarpEmu *g_warp = nullptr;

namespace {
struct EmuDev {
    int err = UNC_OK;
    std::vector<std::pair<void *, u64>> live;
    u64 cur = 0, peak = 0;
    ~EmuDev() { for (auto &a : live) free(a.first); }
    int error() const { return err; }
    template <typename T> T *alloc(u64 count) {
        // poisoned, as device memory is not zeroed
        void *p = malloc(count * sizeof(T) + 16);
        if (!p) { err = UNC_E_NOMEM; return nullptr; }
        memset(p, 0xA5, count * sizeof(T) + 16);
        live.push_back({p, count * sizeof(T)});
        cur += count * sizeof(T);
        peak = std::max(peak, cur);
        return (T *) p;
    }
    void release(void *p) {
        if (!p) return;
        for (size_t i = 0; i < live.size(); i++)
            if (live[i].first == p) {
                free(p);
                cur -= live[i].second;
                live.erase(live.begin() + (long) i);
                return;
            }
    }
    void zero(void *p, u64 b) { memset(p, 0, b); }
    void h2d(void *d, const void *h, u64 b) { memcpy(d, h, b); }
    void d2h(void *h, const void *d, u64 b) { memcpy(h, d, b); }
    void d2d(void *d, const void *x, u64 b) { memcpy(d, x, b); }
    u32 get(const u32 *p) { return *p; }
    template <class F> void each(const F &f, u64 n) {
        for (u64 i = 0; i < n; i++) f(i);
    }
    template <class F> struct TileArg { const F *f; u64 n_tiles; u32 *smem; };
    template <class F> static void tile_entry(void *p) {
        TileArg<F> *a = (TileArg<F> *) p;
        for (u64 t = 0; t < a->n_tiles; t++) a->f->tile(t, a->smem);
    }
    template <class F> void tiles(const F &f, u64 n_tiles) {
        std::vector<u32> smem(F::SMEM_WORDS, 0xA5A5A5A5u);
        TileArg<F> a = {&f, n_tiles, smem.data()};
        emu_run_cta(tile_entry<F>, &a, (int) UNC_FMB_THREADS);
    }
    void mark(int) {}
};
FmbResult g_res;
u64 g_peak = 0, g_model = 0;
}  // namespace

// ws_rows: rows of a doubling batch's sort workspace (0 = the library's); a small value forces many batches.
// Returns what unc_index_build_device returns, apart from its device checks.
extern "C" int emu_index_build(const char *fasta_path, const char *prefix, uint64_t ws_rows) {
    u64 n = 0;
    int rc = unc_fmb_check_size(fasta_path, &n);
    if (rc != UNC_OK) return rc;
    EmuDev d;
    FmbConfig cfg;
    cfg.ws_rows = ws_rows;
    rc = unc_fmb_build_files(d, fasta_path, prefix, cfg, g_res);
    g_peak = d.peak;
    g_model = unc_fmb_device_bytes(n, g_res.ws_rows);
    return rc;
}

// the last build's doubling rounds: active rows and batches per round; returns the number of rounds.  bytes[0] = the
// most memory the build held at once, bytes[1] = what unc_fmb_device_bytes gives for it (the device's memory check).
extern "C" uint32_t emu_index_build_rounds(uint64_t *active, uint64_t *batches, uint32_t cap, uint64_t *ws_rows,
                                           uint64_t bytes[2]) {
    bytes[0] = g_peak;
    bytes[1] = g_model;
    const uint32_t k = std::min<uint32_t>(cap, g_res.rounds);
    std::copy(g_res.active.begin(), g_res.active.begin() + k, active);
    std::copy(g_res.batches.begin(), g_res.batches.begin() + k, batches);
    *ws_rows = g_res.ws_rows;
    return g_res.rounds;
}
