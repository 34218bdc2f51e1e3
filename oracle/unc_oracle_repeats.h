/* oracle/unc_oracle_repeats.h -- the C restatement of `find-repeats` (test infrastructure only): libunc_oracle_repeats.so,
 * built by oracle/repeats.mk from unc_oracle_repeats.c over the FM index of unc_oracle.c. */
#ifndef UNC_ORACLE_REPEATS_H
#define UNC_ORACLE_REPEATS_H
#include "unc_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The loop of find_repeats (reference src/find_repeats.cpp:65-85) with the bases complemented as self_align does
 * (src/self_align_ref.cpp:75,79): out[i] = j - p after the loop's j--, for .pac positions p = pac_st + i, i < n.  Load
 * the index with preset "-".  Returns -1 when the .pac cannot be read, -2 for a window past the end of the reference. */
int orc_repeat_lengths(const orc_index *idx, const char *bwa_prefix, uint64_t pac_st, uint64_t n, uint32_t *out);

#ifdef __cplusplus
}
#endif
#endif
