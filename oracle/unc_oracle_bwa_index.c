/* oracle/unc_oracle_bwa_index.c -- the C restatement of BwaIndex::range_to_fms (reference src/bwa_index.hpp:265-333)
 * and get_neighbor (:158-162), serial as the reference runs them (test infrastructure only).
 *
 * unc_oracle.c is compiled into this library (included below), so that its bwt_2occ / bwt_sa restatements are reused
 * as they are and unc_oracle.c itself stays unchanged; the library stands alone. */
#include <math.h>

#include "unc_oracle.c"

static u8 pac_base(const u8 *pac, u64 i) { return (u8) ((pac[i >> 2] >> (((3 ^ i) & 3) << 1)) & 3); }

/* get_neighbor for n (start, end, base) items */
void orc_bwa_neighbors(const orc_index *x, uint64_t n, const uint64_t *st, const uint64_t *en, const uint8_t *base,
                       uint64_t *ost, uint64_t *oen) {
    for (u64 i = 0; i < n; i++) orc_get_neighbor(x, st[i], en[i], base[i], ost + i, oen + i);
}

/* range_to_fms over .pac positions [pac_min, pac_min + n): first[n] and second[n] as the reference returns them.
 * pac holds the .pac; the caller has checked pac_min + n <= size() / 2. */
void orc_range_to_fms(const orc_index *x, const uint8_t *pac, uint64_t pac_min, uint64_t n, uint64_t *first,
                      uint64_t *second) {
    const u64 ref_len = x->seq_len / 2, pac_max = pac_min + n - 1;
    const u32 slop = (u32) (int) ceil(log((double) ref_len) / log(4));
    u64 fwd_st = ref_len - pac_max > slop ? pac_max + slop : ref_len - 1;
    u64 rs = x->L2[pac_base(pac, fwd_st)], re = x->L2[pac_base(pac, fwd_st) + 1], a, b;
    for (u64 i = fwd_st - 1; i >= pac_max && i <= fwd_st; i--) {
        orc_get_neighbor(x, rs, re, pac_base(pac, i), &a, &b);
        rs = a; re = b;
    }
    for (u64 f = rs; f <= re; f++)
        if (orc_sa(x, f) == pac_max) { rs = re = f; break; }
    u64 k = 0;
    second[k++] = rs;
    for (u64 i = pac_max - 1; i >= pac_min && i < pac_max; i--) {
        orc_get_neighbor(x, rs, re, pac_base(pac, i), &a, &b);
        rs = a; re = b;
        second[k++] = rs;
    }
    const u64 rev_st = pac_min > slop ? pac_min - slop : 0;
    rs = x->L2[3 - pac_base(pac, rev_st)]; re = x->L2[3 - pac_base(pac, rev_st) + 1];
    for (u64 i = rev_st + 1; i <= pac_min; i++) {
        orc_get_neighbor(x, rs, re, 3 - pac_base(pac, i), &a, &b);
        rs = a; re = b;
    }
    for (u64 f = rs; f <= re; f++)
        if (x->seq_len - orc_sa(x, f) == pac_min) { rs = re = f; break; }
    k = 0;
    first[k++] = rs;
    for (u64 i = pac_min + 1; i <= pac_max; i++) {
        orc_get_neighbor(x, rs, re, 3 - pac_base(pac, i), &a, &b);
        rs = a; re = b;
        first[k++] = rs;
    }
}
