// unc_host_index.hpp -- host-side parsing of the bwa/UNCALLED index files and of the pore
// model into the flat arrays the device image is built from.  Plain C++ (no CUDA), shared by
// the C-ABI implementation (unc_abi.cu) and by the CPU emulation build used in tests.
//
// File formats: reference submods/bwa/bwt.c:421-462 (.bwt/.sa), submods/bwa/bntseq.c:97-135
// (.ann), src/mapper.cpp:123-157 (.uncl); pore model: src/pore_model.hpp:48-103.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

struct HostIndex {
    uint64_t primary = 0, L2[5] = {0, 0, 0, 0, 0}, seq_len = 0;
    std::vector<uint32_t> bwt;   // Occ-interleaved BWT words, padded to whole 64-byte blocks
    std::vector<uint32_t> sa32;  // sampled SA narrowed to 32 bits (sa[0] = 0xFFFFFFFF)
    uint64_t sa_intv = 0;
    int64_t l_pac = 0;
    std::vector<std::string> names;
    std::vector<uint64_t> offsets;
    std::vector<uint32_t> lens;
    float thresh[64];
    // pore model, complement order (reference pmodel_r94_complement, src/model_r94.inl:1036)
    std::vector<float> lv_mean, lv_var2, lognorm;
    float model_mean = 0, model_stdv = 0;
    std::string error;
};

static inline bool hix_read_file(const std::string &fn, std::vector<char> &buf) {
    FILE *fp = fopen(fn.c_str(), "rb");
    if (!fp) return false;
    fseek(fp, 0, SEEK_END);
    long n = ftell(fp);
    fseek(fp, 0, SEEK_SET);
    buf.resize((size_t) n);
    bool ok = n == 0 || fread(buf.data(), 1, (size_t) n, fp) == (size_t) n;
    fclose(fp);
    return ok;
}

// PoreModel vector constructor + init_kmer + init_stdv (reference src/pore_model.hpp:48-103)
static inline bool hix_load_model(HostIndex &h, const std::string &table_path) {
    std::vector<char> buf;
    if (!hix_read_file(table_path, buf) || buf.size() != 1024 * 2 * sizeof(float)) {
        h.error = "cannot read pore model table " + table_path;
        return false;
    }
    const float *ms = (const float *) buf.data();
    h.lv_mean.assign(1024, 0.f);
    h.lv_var2.assign(1024, 0.f);
    h.lognorm.assign(1024, 0.f);
    float model_mean = 0;
    for (uint32_t k = 0; k < 1024; k++) {
        float mean = ms[2 * k], stdv = ms[2 * k + 1];
        uint32_t idx = k ^ 0x3FFu;  // kmer_comp (reference src/bp.hpp:77-80)
        h.lv_mean[idx] = mean;
        h.lv_var2[idx] = 2 * stdv * stdv;
        h.lognorm[idx] = (float) std::log(std::sqrt(M_PI * h.lv_var2[idx]));
        model_mean += mean;
    }
    model_mean /= (uint16_t) 1024;
    float model_stdv = 0;
    for (uint32_t k = 0; k < 1024; k++) {
        float d = h.lv_mean[k] - model_mean;
        model_stdv = (float) ((double) model_stdv + (double) d * (double) d);
    }
    h.model_mean = model_mean;
    h.model_stdv = sqrtf(model_stdv / (uint16_t) 1024);
    return true;
}

static inline bool hix_load_ann(HostIndex &h, const std::string &prefix);

// The FM index proper (.bwt, .sa, .ann) -- all `uncalled index` has before the thresholds exist
static inline bool hix_load_fm(HostIndex &h, const std::string &prefix) {
    std::vector<char> b;
    if (!hix_read_file(prefix + ".bwt", b) || b.size() < 40) { h.error = "cannot read " + prefix + ".bwt"; return false; }
    memcpy(&h.primary, b.data(), 8);
    memcpy(&h.L2[1], b.data() + 8, 32);
    h.L2[0] = 0;
    h.seq_len = h.L2[4];
    size_t nwords = (b.size() - 40) >> 2;
    size_t nblocks = (size_t) ((h.seq_len + 127) >> 7) + 1;
    h.bwt.assign(nblocks * 16, 0u);
    if (nwords > h.bwt.size()) { h.error = "inconsistent .bwt size"; return false; }
    memcpy(h.bwt.data(), b.data() + 40, nwords * 4);

    if (!hix_read_file(prefix + ".sa", b) || b.size() < 56) { h.error = "cannot read " + prefix + ".sa"; return false; }
    uint64_t primary, seq_len;
    memcpy(&primary, b.data(), 8);
    memcpy(&h.sa_intv, b.data() + 40, 8);
    memcpy(&seq_len, b.data() + 48, 8);
    if (primary != h.primary || seq_len != h.seq_len) { h.error = "SA-BWT inconsistency"; return false; }
    if (h.sa_intv != 32) { h.error = "unsupported SA interval (device image assumes 32)"; return false; }
    uint64_t n_sa = (h.seq_len + h.sa_intv) / h.sa_intv;
    if (b.size() < 56 + (n_sa - 1) * 8) { h.error = "truncated .sa"; return false; }
    h.sa32.assign(n_sa, 0u);
    h.sa32[0] = 0xFFFFFFFFu;  // (u64)-1 narrowed: sa + steps wraps to steps-1 exactly as in 64 bit
    for (uint64_t i = 1; i < n_sa; i++) {
        uint64_t v;
        memcpy(&v, b.data() + 56 + (i - 1) * 8, 8);
        h.sa32[i] = (uint32_t) v;
    }

    return hix_load_ann(h, prefix);
}

// The contigs of the .ann: names, .pac offsets and lengths (bns_restore, reference submods/bwa/bntseq.c)
static inline bool hix_load_ann(HostIndex &h, const std::string &prefix) {
    FILE *fp = fopen((prefix + ".ann").c_str(), "r");
    if (!fp) { h.error = "cannot read " + prefix + ".ann"; return false; }
    long long xx;
    int n_seqs;
    unsigned seed;
    if (fscanf(fp, "%lld%d%u", &xx, &n_seqs, &seed) != 3) { fclose(fp); h.error = "bad .ann"; return false; }
    h.l_pac = xx;
    for (int i = 0; i < n_seqs; i++) {
        unsigned gi;
        char str[8192];
        int c, len, n_ambs;
        if (fscanf(fp, "%u%8191s", &gi, str) != 2) { fclose(fp); h.error = "bad .ann"; return false; }
        h.names.push_back(str);
        while ((c = fgetc(fp)) != '\n' && c != EOF) {}
        if (fscanf(fp, "%lld%d%d", &xx, &len, &n_ambs) != 3) { fclose(fp); h.error = "bad .ann"; return false; }
        h.offsets.push_back((uint64_t) xx);
        h.lens.push_back((uint32_t) len);
    }
    fclose(fp);
    return true;
}

static inline bool hix_load(HostIndex &h, const std::string &prefix, const std::string &preset) {
    if (!hix_load_fm(h, prefix)) return false;
    // .uncl: "<preset>\t<thr for range len 1>,<2-3>,<4-7>,...\t<prob>\t<speed>"
    // (reference src/mapper.cpp:123-157); atof semantics incl. "nan"
    for (int i = 0; i < 64; i++) h.thresh[i] = 0.f;
    FILE *fp = fopen((prefix + ".uncl").c_str(), "r");
    if (!fp) { h.error = "cannot read " + prefix + ".uncl"; return false; }
    char *line = NULL;
    size_t cap = 0;
    while (getline(&line, &cap, fp) >= 0) {
        size_t L = strlen(line);
        while (L && (line[L - 1] == '\n' || line[L - 1] == '\r')) line[--L] = 0;
        char *save1 = NULL;
        char *name = strtok_r(line, "\t", &save1);
        char *fn_str = strtok_r(NULL, "\t", &save1);
        if (!name) continue;
        if (!preset.empty() && preset != name) continue;
        uint8_t fmbin = 63;
        char *save2 = NULL, *tok;
        while ((tok = strtok_r(fn_str, ",", &save2)) != NULL) {
            fn_str = NULL;
            h.thresh[fmbin] = (float) atof(tok);
            fmbin--;
        }
        for (; fmbin < 64; fmbin--) h.thresh[fmbin] = h.thresh[fmbin + 1];
    }
    free(line);
    fclose(fp);
    return true;
}

// The k-mer buckets of the mapper's child sort (K2V2Tab, unc_device.cuh): k-mers in the order of their FM ranges,
// consecutive k-mers whose ranges overlap (the get_base_range quirk) merged into one group.  T = K2V2Tab.
// Returns false when the merged groups hold more k-mers than the table has room for (no real index does).
template <typename R, typename T>
static inline bool hix_k2v2_tab(const R *kmer_range, T &t) {
    memset(&t, 0, sizeof(t));
    std::vector<uint32_t> ord(1024);
    for (uint32_t k = 0; k < 1024; k++) ord[k] = k;
    auto empty = [&](uint32_t k) { return kmer_range[k].x > kmer_range[k].y; };
    std::stable_sort(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) {
        if (kmer_range[a].x != kmer_range[b].x) return kmer_range[a].x < kmer_range[b].x;
        if (empty(a) != empty(b)) return empty(a);      // empty ranges first
        return a < b;
    });
    uint32_t n_groups = 0, n_merged = 0;
    for (uint32_t i = 0; i < 1024;) {
        uint32_t j = i + 1;
        if (!empty(ord[i])) {
            uint64_t hi = kmer_range[ord[i]].y;
            while (j < 1024 && !empty(ord[j]) && kmer_range[ord[j]].x <= hi) { hi = std::max<uint64_t>(hi, kmer_range[ord[j]].y); j++; }
        }
        const uint32_t g = n_groups++, members = j - i;
        const uint16_t slot = (uint16_t) (((g & 31u) << 5) | (g >> 5));
        t.gkmer[g] = (uint16_t) ord[i];
        if (members > 1) {
            if (n_merged + members > sizeof(t.mk) / sizeof(t.mk[0]) || members > 255) return false;
            t.gmeta[g] = (uint16_t) ((n_merged << 8) | members);
            for (uint32_t m = 0; m < members; m++) t.mk[n_merged + m] = (uint16_t) ord[i + m];
            n_merged += members;
        }
        for (uint32_t m = 0; m < members; m++) { t.kslot[ord[i + m]] = slot; t.ksub[ord[i + m]] = (uint8_t) m; }
        i = j;
    }
    return true;
}
