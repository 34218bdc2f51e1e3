/* oracle/unc_oracle_repeats.c -- the C restatement of `find-repeats` (test infrastructure only).
 *
 * unc_oracle.c is compiled into this library (included below), so that its get_neighbor is reused as it is and
 * unc_oracle.c itself stays unchanged; the library stands alone. */
#include "unc_oracle.c"
#include "unc_oracle_repeats.h"

static u8 pac_comp(const u8 *pac, u64 q) { return (u8) (3 - ((pac[q >> 2] >> (((3 ^ q) & 3) << 1)) & 3)); }

int orc_repeat_lengths(const orc_index *x, const char *prefix, uint64_t pac_st, uint64_t n, uint32_t *out) {
    char fn[4096];
    snprintf(fn, sizeof fn, "%s.pac", prefix);
    size_t sz = 0;
    u8 *pac = (u8 *) read_file(fn, &sz);
    if (!pac) return -1;
    u64 st = 0, total = 0;
    for (int s = 0; s < x->n_seqs; s++) total += (u64) x->lens[s];
    if (pac_st > total || n > total - pac_st || sz * 4 < total) { free(pac); return -2; }
    for (int s = 0; s < x->n_seqs; s++) {
        const u64 len = (u64) x->lens[s];
        for (u64 i = 0; i < len; i++) {
            if (st + i < pac_st || st + i >= pac_st + n) continue;
            u8 b = pac_comp(pac, st + i);
            u64 rs = x->L2[b], re = x->L2[b + 1];           /* get_base_range: start L2[b] (src/bwa_index.hpp:172-174) */
            u64 j = i + 1;
            for (; j < len && re - rs + 1 > 1; j++) {
                u64 ns, ne;
                orc_get_neighbor(x, rs, re, pac_comp(pac, st + j), &ns, &ne);
                rs = ns; re = ne;
            }
            j--;
            out[st + i - pac_st] = (uint32_t) (j - i);
        }
        st += len;
    }
    free(pac);
    return 0;
}
