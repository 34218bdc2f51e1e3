// unc_mask_ext_host.hpp -- host half of `mask-external` (no CUDA): argument checks, table and piece sizes, and the
// outputs (masked FASTA and BED runs).  Shared by unc_mask_ext_host.inl and the emulator build of the tests.  The
// FASTA files are read by unc_mask_read_fasta, as `mask-internal` reads them.
#pragma once
#include <sys/stat.h>

#include <algorithm>

#include "unc_mask_host.hpp"

#define UNC_MX_DEFAULT_PIECE (64ull << 20)   // full-reference window starts per piece
#define UNC_MX_MAX_FILTER_BITS (1ull << 28)  // 32 MB: stays in the H100's 50 MB L2

// the directory part of `path` exists ("" = the working directory)
static inline bool unc_mx_dir_exists(const char *path) {
    std::string d(path);
    const size_t cut = d.find_last_of('/');
    if (cut == std::string::npos) return true;
    d.resize(cut == 0 ? 1 : cut);
    struct stat st;
    return stat(d.c_str(), &st) == 0 && S_ISDIR(st.st_mode);
}

// UNC_OK or UNC_E_ARG with err set
static inline int unc_mx_check_args(uint32_t min_len, uint32_t min_copy, const char *out_fasta, const char *out_bed,
                                    std::string &err) {
    if (min_len < 2 || min_len > 64) { err = "min_len must be 2 .. 64 (keys are 128-bit)"; return UNC_E_ARG; }
    if (min_copy < 1) { err = "min_copy must be at least 1"; return UNC_E_ARG; }
    for (const char *p : {out_fasta, out_bed})
        if (!unc_mx_dir_exists(p)) { err = std::string("the directory of ") + p + " does not exist"; return UNC_E_ARG; }
    return UNC_OK;
}

// the number of valid k-windows (k bases, all ACGT) of codes[0, n)
static inline uint64_t unc_mx_count_windows(const uint8_t *codes, uint64_t n, uint32_t k) {
    uint64_t w = 0, run = 0;
    for (uint64_t i = 0; i < n; i++) {
        run = codes[i] < 4 ? run + 1 : 0;
        w += run >= k;
    }
    return w;
}

// the table: a power of two of at least twice the windows; the filter: 16 bits per window, at most
// UNC_MX_MAX_FILTER_BITS.  UNC_E_TOO_LARGE past 2^31 slots (slots are 32-bit).
static inline int unc_mx_table_size(uint64_t n_windows, uint64_t *cap, uint64_t *filter_bits) {
    uint64_t c = 16;
    while (c < 2 * n_windows) c <<= 1;
    if (c > (1ull << 31)) return UNC_E_TOO_LARGE;
    uint64_t f = 1024;
    while (f < 16 * n_windows && f < UNC_MX_MAX_FILTER_BITS) f <<= 1;
    *cap = c;
    *filter_bits = f;
    return UNC_OK;
}

// the full reference's window starts [0, n - k + 1) in pieces of `piece` starts; piece i reads the bytes
// [i x piece, i x piece + starts + k - 1), so consecutive pieces overlap by k - 1 bytes
struct MxPieces {
    uint64_t n_starts = 0, piece = 0, n_pieces = 0;
    MxPieces(uint64_t n, uint32_t k, uint64_t piece_bases) {
        n_starts = n >= k ? n - k + 1 : 0;
        piece = piece_bases ? piece_bases : UNC_MX_DEFAULT_PIECE;
        n_pieces = (n_starts + piece - 1) / piece;
    }
    uint64_t off(uint64_t i) const { return i * piece; }
    uint64_t starts(uint64_t i) const { return std::min(piece, n_starts - i * piece); }
};

// the masked FASTA (unc_mask_write_fasta) and one BED line `name\tstart\tend` per maximal run of masked positions,
// in record order; *n_selected / *n_masked_bp from the window counts and the mask bits
static inline int unc_mx_write_outputs(const MaskFasta &F, const uint8_t *codes, const uint32_t *counts,
                                       uint32_t min_copy, const char *out_fasta, const char *out_bed,
                                       uint64_t *n_selected, uint64_t *n_masked_bp, std::string &err) {
    uint64_t sel = 0, masked = 0;
    for (size_t i = 0; i < F.seq.size(); i++) {
        sel += counts[i] > min_copy;
        masked += (codes[i] & 8u) != 0;
    }
    int rc = unc_mask_write_fasta(F, codes, out_fasta, err);
    if (rc != UNC_OK) return rc;
    FILE *fp = fopen(out_bed, "wb");
    if (!fp) { err = std::string("cannot create ") + out_bed; return UNC_E_IO; }
    bool ok = true;
    for (size_t r = 0; r < F.headers.size() && ok; r++) {
        const std::string &h = F.headers[r];
        size_t e = 1;
        while (e < h.size() && !unc_mask_space((unsigned char) h[e])) e++;
        const std::string name = h.substr(1, e - 1);       // the first word after '>', as samtools faidx names it
        const uint8_t *c = codes + F.rec_off[r];
        const uint64_t len = F.rec_len[r];
        for (uint64_t j = 0; j < len && ok;) {
            if (!(c[j] & 8u)) { j++; continue; }
            uint64_t e2 = j;
            while (e2 < len && (c[e2] & 8u)) e2++;
            ok = fprintf(fp, "%s\t%llu\t%llu\n", name.c_str(), (unsigned long long) j, (unsigned long long) e2) > 0;
            j = e2;
        }
    }
    if (fclose(fp) != 0) ok = false;
    if (!ok) { err = std::string("cannot write ") + out_bed; return UNC_E_IO; }
    *n_selected = sel;
    *n_masked_bp = masked;
    return UNC_OK;
}
