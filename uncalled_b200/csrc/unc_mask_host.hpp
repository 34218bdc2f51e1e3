// unc_mask_host.hpp -- host half of `mask-internal` (no CUDA): reading the FASTA the way masking/mask_kmers.py
// reads it, the byte codes of unc_mask.cuh, and writing the masked FASTA.  Shared by unc_mask_host.inl and the
// emulator build of the tests.
//
// Reading: lines end at \n, \r\n or \r (Python's universal newlines).  A line whose first byte is '>' starts a
// record and its header is the line stripped of whitespace; every other line is stripped and appended to the
// record's sequence, so lines are joined and a space inside a line stays a (non-ACGT) byte of the sequence.
#pragma once
#include <stdint.h>
#include <stdio.h>

#include <string>
#include <vector>

#include "../../include/unc_b200.h"

struct MaskFasta {
    std::vector<std::string> headers;
    std::vector<uint64_t> rec_off, rec_len;   // record i: positions [rec_off[i], rec_off[i] + rec_len[i])
    std::string seq;                          // every record's sequence, one separator byte between records
    uint64_t n_bases = 0;
    std::string error;
};

// ASCII whitespace as Python's str.strip() removes it
static inline bool unc_mask_space(unsigned char c) { return c == ' ' || (c >= 9 && c <= 13) || (c >= 28 && c <= 31); }

// 0-3 for ACGT in either case, UNC_MASK_BRK (4) for every other byte
static inline uint8_t unc_mask_code(unsigned char c) {
    switch (c | 0x20) {
        case 'a': return 0;
        case 'c': return 1;
        case 'g': return 2;
        case 't': return 3;
    }
    return 4;
}

// UNC_OK, or UNC_E_IO / UNC_E_ARG / UNC_E_TOO_LARGE with F.error set
static inline int unc_mask_read_fasta(const char *path, MaskFasta &F) {
    FILE *fp = fopen(path, "rb");
    if (!fp) { F.error = std::string("cannot open ") + path; return UNC_E_IO; }
    std::string data;
    char buf[1 << 16];
    size_t got;
    while ((got = fread(buf, 1, sizeof buf, fp)) > 0) data.append(buf, got);
    const bool bad = ferror(fp) != 0;
    fclose(fp);
    if (bad) { F.error = std::string("cannot read ") + path; return UNC_E_IO; }
    if (data.empty()) { F.error = "empty FASTA file"; return UNC_E_ARG; }
    if (data[0] != '>') { F.error = "the first line of the FASTA file does not start with '>'"; return UNC_E_ARG; }
    F.seq.reserve(data.size());
    const size_t n = data.size();
    size_t i = 0;
    auto close_record = [&]() -> bool {
        if (F.headers.empty()) return true;
        F.rec_len.push_back(F.seq.size() - F.rec_off.back());
        return F.rec_len.back() > 0;
    };
    while (i < n) {
        size_t e = i;
        while (e < n && data[e] != '\n' && data[e] != '\r') e++;
        size_t b = i, f = e;
        while (b < f && unc_mask_space((unsigned char) data[b])) b++;
        while (f > b && unc_mask_space((unsigned char) data[f - 1])) f--;
        if (e > i && data[i] == '>') {
            if (!close_record()) { F.error = "record '" + F.headers.back() + "' has no sequence"; return UNC_E_ARG; }
            if (!F.headers.empty()) F.seq.push_back('\n');            // the separator: not ACGT, breaks every k-mer
            F.headers.push_back(data.substr(b, f - b));
            F.rec_off.push_back(F.seq.size());
        } else {
            F.seq.append(data, b, f - b);
        }
        i = e;
        if (i < n && data[i] == '\r') i++;
        if (i < n && data[i] == '\n' && (i == e || data[i - 1] == '\r')) i++;
    }
    if (!close_record()) { F.error = "record '" + F.headers.back() + "' has no sequence"; return UNC_E_ARG; }
    for (uint64_t l : F.rec_len) F.n_bases += l;
    if (F.n_bases >= (1ull << 32)) { F.error = "a genome of 2^32 or more bases (the counts are 32-bit)"; return UNC_E_TOO_LARGE; }
    return UNC_OK;
}

static inline void unc_mask_codes(const MaskFasta &F, uint8_t *dst) {
    for (size_t i = 0; i < F.seq.size(); i++) dst[i] = unc_mask_code((unsigned char) F.seq[i]);
}

// header, then the whole sequence on one line, '\n' line ends; positions whose code has UNC_MASK_HIT become 'N'
static inline int unc_mask_write_fasta(const MaskFasta &F, const uint8_t *codes, const char *path, std::string &err) {
    FILE *fp = fopen(path, "wb");
    if (!fp) { err = std::string("cannot create ") + path; return UNC_E_IO; }
    std::string line;
    bool ok = true;
    for (size_t r = 0; r < F.headers.size() && ok; r++) {
        line.assign(F.headers[r]);
        line.push_back('\n');
        const uint64_t o = F.rec_off[r];
        line.append(F.seq, o, F.rec_len[r]);
        for (uint64_t j = 0; j < F.rec_len[r]; j++)
            if (codes[o + j] & 8u) line[F.headers[r].size() + 1 + j] = 'N';
        line.push_back('\n');
        ok = fwrite(line.data(), 1, line.size(), fp) == line.size();
    }
    if (fclose(fp) != 0) ok = false;
    if (!ok) { err = std::string("cannot write ") + path; return UNC_E_IO; }
    return UNC_OK;
}
