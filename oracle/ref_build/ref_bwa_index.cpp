// oracle/_ref/libref_bwa_index.so: the reference's own BwaIndex<k5> (src/bwa_index.hpp) and k-mer helpers (src/bp.hpp)
// behind a C interface: sa, get_neighbor, get_kmer_range, range_to_fms, get_kmers, translate_loc and the kmer_* helpers.
//
// TEST INFRASTRUCTURE ONLY.  Built by oracle/bwa_index.mk where the reference tree lies under /root/reference, against
// oracle/_ref/libuncalled_ref.so (which holds bwa and range.cpp compiled from the reference's own sources).  Nothing of
// the reference is copied here; this file only calls it.  Its own definitions are hidden (-fvisibility=hidden), so the
// BwaIndex template instantiated here cannot interpose on anything in the library.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

// pacseq_ is private; the shim frees it (the reference's destroy() does not)
#define private public
#include "bwa_index.hpp"
#undef private

#define EXPORT extern "C" __attribute__((visibility("default")))
typedef BwaIndex<KmerLen::k5> Idx;

EXPORT void *ref_bwa_open(const char *prefix) { return new Idx(prefix, true); }

EXPORT void ref_bwa_free(void *h) {
    Idx *x = (Idx *) h;
    x->destroy();
    free(x->pacseq_);
    delete x;
}

EXPORT uint64_t ref_bwa_size(void *h) { return ((Idx *) h)->size(); }

EXPORT void ref_bwa_sa(void *h, uint64_t n, const uint64_t *rows, uint64_t *out) {
    for (uint64_t i = 0; i < n; i++) out[i] = ((Idx *) h)->sa(rows[i]);
}

EXPORT void ref_bwa_neighbor(void *h, uint64_t n, const uint64_t *st, const uint64_t *en, const uint8_t *base, uint64_t *os,
                             uint64_t *oe) {
    for (uint64_t i = 0; i < n; i++) {
        Range r = ((Idx *) h)->get_neighbor(Range(st[i], en[i]), base[i]);
        os[i] = r.start_; oe[i] = r.end_;
    }
}

EXPORT void ref_bwa_kmer_ranges(void *h, uint64_t *st, uint64_t *en) {
    for (uint16_t k = 0; k < 1024; k++) {
        Range r = ((Idx *) h)->get_kmer_range(k);
        st[k] = r.start_; en[k] = r.end_;
    }
}

// first / second: room for end - start each
EXPORT void ref_bwa_range_to_fms(void *h, const char *name, uint64_t start, uint64_t end, uint64_t *first, uint64_t *second) {
    auto p = ((Idx *) h)->range_to_fms(name, start, end);
    std::copy(p.first.begin(), p.first.end(), first);
    std::copy(p.second.begin(), p.second.end(), second);
}

// out: room for max(0, en - st - 4); kmers_revcomp of the same k-mers into rev when rev is not null.  Returns the count.
EXPORT uint64_t ref_bwa_get_kmers(void *h, uint64_t st, uint64_t en, uint16_t *out, uint16_t *rev) {
    std::vector<u16> k = ((Idx *) h)->get_kmers(st, en);
    std::copy(k.begin(), k.end(), out);
    if (rev) {
        std::vector<u16> r = kmers_revcomp<KmerLen::k5>(k);
        std::copy(r.begin(), r.end(), rev);
    }
    return k.size();
}

// name: room for cap bytes.  Returns the contig length, 0 when sa_loc lies in no contig (name and loc untouched).
EXPORT uint64_t ref_bwa_translate_loc(void *h, uint64_t sa_loc, char *name, uint64_t cap, uint64_t *loc) {
    std::string nm;
    u64 l = 0;
    const u64 len = ((Idx *) h)->translate_loc(sa_loc, nm, l);
    if (len) { strncpy(name, nm.c_str(), cap - 1); name[cap - 1] = 0; *loc = l; }
    return len;
}

// the k = 5 helpers for every k-mer: comp, revcomp, head, base(i) x 5, neighbor(b) x 4, str_to_kmer(kmer_to_str)
EXPORT void ref_kmer_helpers(uint16_t *comp, uint16_t *revcomp, uint8_t *head, uint8_t *base5, uint16_t *nb4, uint16_t *roundtrip,
                             char *str6) {
    for (u16 k = 0; k < 1024; k++) {
        comp[k] = kmer_comp<KmerLen::k5>(k);
        revcomp[k] = kmer_revcomp<KmerLen::k5>(k);
        head[k] = kmer_head<KmerLen::k5>(k);
        for (u8 i = 0; i < 5; i++) base5[5 * k + i] = kmer_base<KmerLen::k5>(k, i);
        for (u8 b = 0; b < 4; b++) nb4[4 * k + b] = kmer_neighbor<KmerLen::k5>(k, b);
        std::string s = kmer_to_str<KmerLen::k5>(k);
        memcpy(str6 + 6 * k, s.c_str(), 6);
        roundtrip[k] = str_to_kmer<KmerLen::k5>(s, 0);
    }
}

EXPORT uint16_t ref_str_to_kmer(const char *s, uint64_t offset) { return str_to_kmer<KmerLen::k5>(std::string(s), offset); }
EXPORT uint16_t ref_kmer_count() { return kmer_count<KmerLen::k5>(); }
