// unc_index_host.hpp -- the host steps of bwa-compatible FM-index construction, shared by the host builder
// (unc_index_build.cpp), the device builder (unc_fmb_host.inl) and the emulator build of the tests: FASTA parsing with
// kseq semantics, ambiguous bases as lrand48()&3 after srand48(11) in file order (bntseq.c:266,296), the .pac / .ann /
// .amb files (bntseq.c:66-95,306-322), and the layout of the .bwt and .sa files (bwt.c:381-405).  Only the suffix sort
// and the construction of the BWT, the Occ blocks and the sampled SA differ between the builders.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/unc_b200.h"

#define UNC_BWA_SA_INTV 32u
// the device image (unc_index_load, the mapper's u32 FM rows) holds seq_len = 2 * l_pac < UNC_BWA_DEVICE_MAX_ROWS
#define UNC_BWA_DEVICE_MAX_ROWS 0xFFFFFF00ull

struct BwaAnn { std::string name, anno; int64_t offset; int32_t len, n_ambs; };
struct BwaAmb { int64_t offset; int32_t len; char amb; };
struct BwaRef {
    std::vector<BwaAnn> anns;
    std::vector<BwaAmb> ambs;
    std::vector<uint8_t> fwd;  // one 2-bit code per byte, ambiguous bases already replaced
};

static inline int unc_bwa_nt4(int c) {
    switch (c) {
        case 'A': case 'a': return 0;
        case 'C': case 'c': return 1;
        case 'G': case 'g': return 2;
        case 'T': case 't': return 3;
        default: return 4;
    }
}

static inline bool unc_bwa_space(char ch) { return ch == '\n' || ch == '\r' || ch == ' ' || ch == '\t'; }

static inline bool unc_bwa_write_file(const std::string &fn, const void *p, size_t n) {
    FILE *fp = fopen(fn.c_str(), "wb");
    if (!fp) return false;
    bool ok = n == 0 || fwrite(p, 1, n, fp) == n;
    return fclose(fp) == 0 && ok;
}

// l_pac of a FASTA file without holding it in memory: unc_bwa_read_fasta's rules (lines before the first header are
// skipped, a '>' inside a record starts the next header, every byte but whitespace in a record is a base)
static inline int unc_bwa_count_bases(const char *fasta_path, uint64_t *l_pac) {
    FILE *fp = fopen(fasta_path, "rb");
    if (!fp) return UNC_E_IO;
    std::vector<char> buf(1u << 20);
    uint64_t n = 0;
    enum { SKIP, SKIP_LINE, HEADER, SEQ } st = SKIP;
    size_t got;
    while ((got = fread(buf.data(), 1, buf.size(), fp)) > 0) {
        for (size_t i = 0; i < got; i++) {
            const char ch = buf[i];
            switch (st) {
                case SKIP: st = ch == '>' ? HEADER : ch == '\n' ? SKIP : SKIP_LINE; break;
                case SKIP_LINE: if (ch == '\n') st = SKIP; break;
                case HEADER: if (ch == '\n') st = SEQ; break;
                case SEQ:
                    if (ch == '>') st = HEADER;
                    else n += !unc_bwa_space(ch);
                    break;
            }
        }
    }
    fclose(fp);
    *l_pac = n;
    return UNC_OK;
}

// parse the FASTA (kseq semantics: name = first word of the header, comment = the rest); consumes lrand48 after
// srand48(11) for every ambiguous base in file order
static inline int unc_bwa_read_fasta(const char *fasta_path, BwaRef &R) {
    FILE *fp = fopen(fasta_path, "rb");
    if (!fp) return UNC_E_IO;
    srand48(11);
    std::vector<char> buf;
    fseek(fp, 0, SEEK_END);
    long sz = ftell(fp);
    fseek(fp, 0, SEEK_SET);
    buf.resize((size_t) sz);
    if (sz > 0 && fread(buf.data(), 1, (size_t) sz, fp) != (size_t) sz) { fclose(fp); return UNC_E_IO; }
    fclose(fp);
    size_t i = 0, n = buf.size();
    while (i < n) {
        while (i < n && buf[i] != '>') {  // skip to the next header
            while (i < n && buf[i] != '\n') i++;
            if (i < n) i++;
        }
        if (i >= n) break;
        i++;  // '>'
        size_t ls = i;
        while (i < n && buf[i] != '\n') i++;
        std::string header(buf.data() + ls, buf.data() + i);
        if (!header.empty() && header.back() == '\r') header.pop_back();
        if (i < n) i++;
        BwaAnn a;
        size_t sp = header.find_first_of(" \t");
        a.name = header.substr(0, sp);
        a.anno = "(null)";
        if (sp != std::string::npos && sp + 1 < header.size()) a.anno = header.substr(sp + 1);
        a.offset = (int64_t) R.fwd.size();
        a.n_ambs = 0;
        int lasts = 0;
        int64_t len = 0;
        while (i < n && buf[i] != '>') {
            char ch = buf[i++];
            if (unc_bwa_space(ch)) continue;
            int c = unc_bwa_nt4(ch);
            if (c >= 4) {
                if (lasts == ch) {
                    R.ambs.back().len++;
                } else {
                    BwaAmb h = {a.offset + len, 1, ch};
                    R.ambs.push_back(h);
                    a.n_ambs++;
                }
                c = (int) (lrand48() & 3);
            }
            lasts = ch;
            R.fwd.push_back((uint8_t) c);
            len++;
        }
        a.len = (int32_t) len;
        R.anns.push_back(a);
    }
    return UNC_OK;
}

// <prefix>.pac (forward only), .ann, .amb
static inline int unc_bwa_write_pac_ann_amb(const BwaRef &R, const std::string &prefix) {
    const int64_t l_pac = (int64_t) R.fwd.size();
    std::vector<uint8_t> pac((size_t) (l_pac >> 2) + ((l_pac & 3) == 0 ? 0 : 1), 0);
    for (int64_t l = 0; l < l_pac; l++) pac[(size_t) (l >> 2)] |= (uint8_t) (R.fwd[(size_t) l] << ((~l & 3) << 1));
    if ((l_pac % 4) == 0) pac.push_back(0);
    pac.push_back((uint8_t) (l_pac % 4));
    if (!unc_bwa_write_file(prefix + ".pac", pac.data(), pac.size())) return UNC_E_IO;
    FILE *fa = fopen((prefix + ".ann").c_str(), "w");
    if (!fa) return UNC_E_IO;
    fprintf(fa, "%lld %d %u\n", (long long) l_pac, (int) R.anns.size(), 11u);
    for (const BwaAnn &a : R.anns) {
        fprintf(fa, "%d %s", 0, a.name.c_str());
        if (!a.anno.empty()) fprintf(fa, " %s\n", a.anno.c_str());
        else fprintf(fa, "\n");
        fprintf(fa, "%lld %d %d\n", (long long) a.offset, a.len, a.n_ambs);
    }
    fclose(fa);
    fa = fopen((prefix + ".amb").c_str(), "w");
    if (!fa) return UNC_E_IO;
    fprintf(fa, "%lld %d %u\n", (long long) l_pac, (int) R.anns.size(), (unsigned) R.ambs.size());
    for (const BwaAmb &h : R.ambs) fprintf(fa, "%lld %d %c\n", (long long) h.offset, h.len, h.amb);
    fclose(fa);
    return UNC_OK;
}

// L2[1..4] from the occurrences of each symbol in the forward + reverse-complement text (L2[0] = 0)
static inline void unc_bwa_l2(const uint64_t counts[4], uint64_t L2[5]) {
    L2[0] = 0;
    for (int c = 0; c < 4; c++) L2[c + 1] = L2[c] + counts[c];
}

// the .bwt payload: (n + 15) / 16 words of 16 two-bit symbols plus 8 words (4 x u64 counts) before every 128 symbols
// and after the last one
static inline uint64_t unc_bwa_bwt_words(uint64_t n) { return ((n + 15) >> 4) + ((n + 127) / 128 + 1) * 8; }

static inline int unc_bwa_write_bwt(const std::string &prefix, uint64_t primary, const uint64_t L2[5],
                                    const uint32_t *words, uint64_t n_words) {
    FILE *fb = fopen((prefix + ".bwt").c_str(), "wb");
    if (!fb) return UNC_E_IO;
    fwrite(&primary, 8, 1, fb);
    fwrite(&L2[1], 8, 4, fb);
    fwrite(words, 4, (size_t) n_words, fb);
    return fclose(fb) == 0 ? UNC_OK : UNC_E_IO;
}

// the sampled SA: rows 32, 64, ... (row 0 is written as -1 on load and not stored); sa[j - 1] = SA[32 j]
static inline uint64_t unc_bwa_n_sa(uint64_t seq_len) { return (seq_len + UNC_BWA_SA_INTV) / UNC_BWA_SA_INTV; }

static inline int unc_bwa_write_sa(const std::string &prefix, uint64_t primary, const uint64_t L2[5], uint64_t seq_len,
                                   const uint64_t *sa) {
    const uint64_t sa_intv = UNC_BWA_SA_INTV, n_sa = unc_bwa_n_sa(seq_len);
    FILE *fs = fopen((prefix + ".sa").c_str(), "wb");
    if (!fs) return UNC_E_IO;
    fwrite(&primary, 8, 1, fs);
    fwrite(&L2[1], 8, 4, fs);
    fwrite(&sa_intv, 8, 1, fs);
    fwrite(&seq_len, 8, 1, fs);
    fwrite(sa, 8, (size_t) (n_sa - 1), fs);
    return fclose(fs) == 0 ? UNC_OK : UNC_E_IO;
}
