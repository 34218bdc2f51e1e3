// unc_index_build.cpp -- bwa-compatible FM-index construction (host C++).
//
// Replaces BwaIndex::create -> bwa_idx_build (reference src/bwa_index.hpp:92-101,
// submods/bwa/bwtindex.c:255-323) for the `uncalled index` command.  Writes the same five
// files, byte for byte, that `bwa index` writes:
//   <p>.pac  forward-only 2-bit packed sequence          (bntseq.c:306-322)
//   <p>.ann  <p>.amb  sequence / ambiguity tables          (bntseq.c:66-95)
//   <p>.bwt  primary, L2[1..4], Occ-interleaved BWT of fwd+revcomp   (bwtindex.c:64-130,
//            bwt_bwtupdate_core :132-163, bwt.c:381-393)
//   <p>.sa   SA sampled every 32 rows                      (bwt.c:61-84,395-405)
// The BWT is a mathematical object, so it is built here with a linear-time SA-IS suffix
// sorter written for this project rather than with bwa's is.c / bwt_gen.c.
// Ambiguous bases become lrand48()&3 after srand48(11) exactly as bwa does (bntseq.c:266,296).
// The host steps (FASTA, .pac/.ann/.amb, the .bwt/.sa layout) are unc_index_host.hpp's, shared with the device
// builder unc_index_build_device (unc_fmb_host.inl); this file's own part is the suffix sort and the BWT / Occ / SA.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "unc_index_host.hpp"

namespace {

// ---- SA-IS (induced sorting).  s[n-1] must be a unique smallest sentinel (value 0).
template <typename T>
void sais(const T *s, int32_t *SA, int32_t n, int32_t K) {
    std::vector<bool> t((size_t) n);  // true = S-type
    t[n - 1] = true;
    for (int32_t i = n - 2; i >= 0; i--) t[i] = s[i] < s[i + 1] || (s[i] == s[i + 1] && t[i + 1]);
    auto is_lms = [&](int32_t i) { return i > 0 && t[i] && !t[i - 1]; };
    std::vector<int32_t> bkt((size_t) K + 1);
    auto buckets = [&](bool end) {
        std::fill(bkt.begin(), bkt.end(), 0);
        for (int32_t i = 0; i < n; i++) bkt[s[i]]++;
        int32_t sum = 0;
        for (int32_t c = 0; c <= K; c++) {
            sum += bkt[c];
            bkt[c] = end ? sum : sum - bkt[c];
        }
    };
    auto induce = [&]() {
        buckets(false);
        for (int32_t i = 0; i < n; i++) {
            int32_t j = SA[i] - 1;
            if (SA[i] > 0 && !t[j]) SA[bkt[s[j]]++] = j;
        }
        buckets(true);
        for (int32_t i = n - 1; i >= 0; i--) {
            int32_t j = SA[i] - 1;
            if (SA[i] > 0 && t[j]) SA[--bkt[s[j]]] = j;
        }
    };
    // stage 1: sort the LMS substrings
    buckets(true);
    for (int32_t i = 0; i < n; i++) SA[i] = -1;
    for (int32_t i = 1; i < n; i++)
        if (is_lms(i)) SA[--bkt[s[i]]] = i;
    induce();
    int32_t n1 = 0;
    for (int32_t i = 0; i < n; i++)
        if (is_lms(SA[i])) SA[n1++] = SA[i];
    for (int32_t i = n1; i < n; i++) SA[i] = -1;
    int32_t name = 0, prev = -1;
    for (int32_t i = 0; i < n1; i++) {
        int32_t pos = SA[i];
        bool diff = false;
        for (int32_t d = 0;; d++) {
            if (prev == -1 || s[pos + d] != s[prev + d] || t[pos + d] != t[prev + d]) { diff = true; break; }
            if (d > 0 && (is_lms(pos + d) || is_lms(prev + d))) break;
        }
        if (diff) { name++; prev = pos; }
        SA[n1 + pos / 2] = name - 1;
    }
    for (int32_t i = n - 1, j = n - 1; i >= n1; i--)
        if (SA[i] >= 0) SA[j--] = SA[i];
    // stage 2: solve the reduced problem
    int32_t *SA1 = SA, *s1 = SA + n - n1;
    if (name < n1) sais<int32_t>(s1, SA1, n1, name - 1);
    else for (int32_t i = 0; i < n1; i++) SA1[s1[i]] = i;
    // stage 3: induce the final order
    buckets(true);
    for (int32_t i = 1, j = 0; i < n; i++)
        if (is_lms(i)) s1[j++] = i;
    for (int32_t i = 0; i < n1; i++) SA1[i] = s1[SA1[i]];
    for (int32_t i = n1; i < n; i++) SA[i] = -1;
    for (int32_t i = n1 - 1; i >= 0; i--) {
        int32_t j = SA[i];
        SA[i] = -1;
        SA[--bkt[s[j]]] = j;
    }
    induce();
}

}  // namespace

extern "C" int unc_index_build(const char *fasta_path, const char *prefix_c) {
    if (!fasta_path || !prefix_c) return UNC_E_ARG;
    const std::string prefix = prefix_c;
    BwaRef R;
    int rc = unc_bwa_read_fasta(fasta_path, R);
    if (rc != UNC_OK) return rc;
    const std::vector<uint8_t> &fwd = R.fwd;
    const int64_t l_pac = (int64_t) fwd.size();
    if (l_pac == 0) return UNC_E_IO;
    if (2 * l_pac + 1 >= 0x7FFFFFF0ll) return UNC_E_TOO_LARGE;
    if ((rc = unc_bwa_write_pac_ann_amb(R, prefix)) != UNC_OK) return rc;

    // ---- text = forward + reverse complement, suffix array, BWT
    const int64_t n = 2 * l_pac;  // bwt->seq_len
    std::vector<uint8_t> text((size_t) n + 1);
    for (int64_t i = 0; i < l_pac; i++) text[(size_t) i] = (uint8_t) (fwd[(size_t) i] + 1);
    for (int64_t i = 0; i < l_pac; i++) text[(size_t) (l_pac + i)] = (uint8_t) (3 - fwd[(size_t) (l_pac - 1 - i)] + 1);
    text[(size_t) n] = 0;  // sentinel
    std::vector<int32_t> SA((size_t) n + 1);
    sais<uint8_t>(text.data(), SA.data(), (int32_t) (n + 1), 4);

    uint64_t L2[5] = {0, 0, 0, 0, 0};
    for (int64_t i = 0; i < n; i++) L2[text[(size_t) i]]++;  // text value c+1 -> L2[c+1]
    for (int i = 2; i <= 4; i++) L2[i] += L2[i - 1];
    // BWT over rows 0..n (row 0 = sentinel suffix); '$' (row `primary`) is dropped
    uint64_t primary = 0;
    std::vector<uint8_t> bw((size_t) n);
    {
        size_t k = 0;
        for (int64_t i = 0; i <= n; i++) {
            if (SA[(size_t) i] == 0) primary = (uint64_t) i;
            else bw[k++] = (uint8_t) (text[(size_t) SA[(size_t) i] - 1] - 1);
        }
    }
    // Occ interleave: 4 x u64 cumulative counts before every 128 symbols, plus the final totals
    const uint64_t n_occ = (uint64_t) ((n + 127) / 128 + 1);
    const uint64_t bwt_words = (uint64_t) ((n + 15) >> 4) + n_occ * 8;
    std::vector<uint32_t> out((size_t) bwt_words, 0u);
    {
        uint64_t c[4] = {0, 0, 0, 0};
        size_t k = 0;
        for (int64_t i = 0; i < n; i++) {
            if ((i & 127) == 0) { memcpy(&out[k], c, 32); k += 8; }
            if ((i & 15) == 0) k++;
            out[k - 1] |= (uint32_t) bw[(size_t) i] << ((15 - (i & 15)) << 1);
            c[bw[(size_t) i]]++;
        }
        memcpy(&out[k], c, 32);
        if (k + 8 != bwt_words) return UNC_E_IO;
    }
    if ((rc = unc_bwa_write_bwt(prefix, primary, L2, out.data(), out.size())) != UNC_OK) return rc;
    // ---- sampled SA: rows 32, 64, ...
    {
        const uint64_t seq_len = (uint64_t) n, n_sa = unc_bwa_n_sa(seq_len);
        std::vector<uint64_t> sa((size_t) n_sa, 0);
        for (uint64_t j = 1; j < n_sa; j++) sa[(size_t) j] = (uint64_t) SA[(size_t) (j * UNC_BWA_SA_INTV)];
        if ((rc = unc_bwa_write_sa(prefix, primary, L2, seq_len, sa.data() + 1)) != UNC_OK) return rc;
    }
    return UNC_OK;
}
