// tests/emul/emul_repeats.cpp -- `find-repeats` on the CPU: unc_repeat_length (uncalled_b200/csrc/unc_selfalign.cuh),
// one "thread" after the other, around the same host steps as unc_repeats_create / unc_repeats_lengths
// (uncalled_b200/csrc/unc_repeats_host.inl).  Test vehicle only.
#include "unc_device.cuh"   // UNC_EMUL is defined on the command line
#include "unc_selfalign.cuh"
#include "unc_selfalign_host.hpp"
#include "unc_host_index.hpp"

thread_local WarpEmu *g_warp = nullptr;

extern "C" {

// out[i] = L(pac_st + i), i < n.  -1: the index does not load; -2: the window lies past the end of the reference.
int emu_repeat_lengths(const char *prefix, uint64_t pac_st, uint32_t n, uint32_t *out) {
    HostIndex h;
    std::vector<char> pac;
    if (!hix_load_fm(h, prefix) || !hix_read_file(std::string(prefix) + ".pac", pac)) return -1;
    uint64_t total = 0;
    for (uint32_t l : h.lens) total += l;
    if (h.lens.empty() || total == 0 || pac.size() * 4 < total || 2 * total != h.seq_len) return -1;
    if (pac_st > total || n > total - pac_st) return -2;
    pac.resize(pac.size() + 16, 0);
    const std::vector<u32> ends = unc_repeats_ends(h.lens);
    DevIndex ix{};
    ix.bwt = (const uint4 *) h.bwt.data();
    ix.primary = (u32) h.primary; ix.seq_len = (u32) h.seq_len;
    for (int i = 0; i < 5; i++) ix.L2[i] = (u32) h.L2[i];
    DevRepeats R{};
    R.pac = (const u8 *) pac.data(); R.ends = ends.data(); R.n_contigs = (u32) ends.size();
    R.pac_st = (u32) pac_st; R.n = n; R.out = out;
    for (u32 i = 0; i < n; i++) unc_repeat_length(ix, R, i);
    return 0;
}

}  // extern "C"
