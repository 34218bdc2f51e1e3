// tests/emul/emul_bwa_index.cpp -- the BwaIndex queries on the CPU: unc_bwa_neighbor, unc_bwa_sa and the two
// range_to_fms passes (uncalled_b200/csrc/unc_bwa.cuh) under the warp emulator, around the same host steps as
// unc_bwa_neighbor / unc_bwa_sa / unc_bwa_range_to_fms (uncalled_b200/csrc/unc_bwa_host.inl).  The segment length is
// an argument so that short spans still cut into several segments.  Test vehicle only.
#include <cmath>

#include "unc_device.cuh"   // UNC_EMUL is defined on the command line
#include "unc_bwa.cuh"
#include "unc_host_index.hpp"

thread_local WarpEmu *g_warp = nullptr;

namespace {
struct Loaded {
    HostIndex h;
    std::vector<char> pac;
    DevIndex ix{};
    uint64_t l_pac = 0;
};

bool load(const char *prefix, Loaded &L) {
    if (!hix_load_fm(L.h, prefix) || !hix_read_file(std::string(prefix) + ".pac", L.pac)) return false;
    for (uint32_t l : L.h.lens) L.l_pac += l;
    if (L.l_pac == 0 || 2 * L.l_pac != L.h.seq_len || L.pac.size() * 4 < L.l_pac) return false;
    L.pac.resize(L.pac.size() + 16, 0);
    L.h.bwt.resize(L.h.bwt.size() + 16, 0);      // the device image's 64-byte pad
    L.ix.bwt = (const uint4 *) L.h.bwt.data();
    L.ix.sa = L.h.sa32.data();
    L.ix.primary = (u32) L.h.primary;
    L.ix.seq_len = (u32) L.h.seq_len;
    for (int i = 0; i < 5; i++) L.ix.L2[i] = (u32) L.h.L2[i];
    return true;
}

struct SegArgs { const DevIndex *ix; const DevFms *F; u64 warp0; };
void seg_entry(void *p) {
    const SegArgs *a = (const SegArgs *) p;
    unc_fms_segments(*a->ix, *a->F, a->warp0 + (u64) (g_warp->cur >> 5));
}
struct FixArgs { const DevIndex *ix; const DevFms *F; };
void fix_entry(void *p) {
    const FixArgs *a = (const FixArgs *) p;
    unc_fms_fixup(*a->ix, *a->F);
}
}  // namespace

extern "C" {

// -1: the index does not load
int emu_bwa_neighbor(const char *prefix, uint64_t n, const uint64_t *st, const uint64_t *en, const uint8_t *base,
                     uint64_t *os, uint64_t *oe) {
    Loaded L;
    if (!load(prefix, L)) return -1;
    for (uint64_t i = 0; i < n; i++) {
        const uint2 r = unc_bwa_neighbor(L.ix, (u32) st[i], (u32) en[i], base[i]);
        os[i] = r.x; oe[i] = r.y;
    }
    return 0;
}

int emu_bwa_sa(const char *prefix, uint64_t n, const uint64_t *rows, uint64_t *out) {
    Loaded L;
    if (!load(prefix, L)) return -1;
    for (uint64_t i = 0; i < n; i++) out[i] = unc_bwa_sa(L.ix, (u32) rows[i]);
    return 0;
}

// range_to_fms over .pac positions [pac_min, pac_min + n) with `seg` positions per segment.  -1: the index does not
// load; -2: the span is outside the reference; -3: an anchor scan found no row.
int emu_bwa_range_to_fms(const char *prefix, uint64_t pac_min, uint64_t n, uint32_t seg, uint64_t *first,
                         uint64_t *second) {
    Loaded L;
    if (!load(prefix, L)) return -1;
    const uint64_t ref_len = L.h.seq_len / 2;
    if (!n || !seg || pac_min >= ref_len || n > ref_len - pac_min) return -2;
    u32 miss = 0;
    DevFms F{};
    F.pac = (const u8 *) L.pac.data();
    F.ref_len = ref_len;
    F.slop = (u32) static_cast<int>(ceil(log((double) ref_len) / log(4)));
    F.pac_min = pac_min; F.n = n; F.seg = seg;
    F.n_seg = (n + seg - 1) / seg;
    F.fwd = second; F.rev = first; F.miss = &miss;
    const uint64_t warps = (2 * F.n_seg + 31) / 32;
    for (uint64_t w = 0; w < warps; w += 4) {                       // CTAs of 128 threads, as k_bwa_fms_segments
        SegArgs a = {&L.ix, &F, w};
        emu_run_cta(seg_entry, &a, 128);
    }
    FixArgs b = {&L.ix, &F};
    emu_run_warp(fix_entry, &b);
    return miss ? -3 : 0;
}

}  // extern "C"
