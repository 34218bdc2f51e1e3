// unc_dtw_align.cuh -- the stages between a read's raw signal and its DTW against a reference span: the loop body of the
// reference's dtw_test driver (src/dtw_test.cpp:94-175) after event detection, which is K1 (unc_k1.cuh) run over the whole
// signal with an event row as long as the signal.
//
//   (b) mask     EventProfiler::get_full_mask (src/event_profiler.hpp:129-151) over the read's events, tail loop included,
//                and the compaction of the unmasked means, in place.  Serial per read: one thread per read.
//   (c) k-mers   BwaIndex::get_kmers (src/bwa_index.hpp:234-255, seq_to_kmers src/bp.hpp:126-146) over the device copy
//                of the .pac, kmers_revcomp (src/bp.hpp:83-99) for the - strand.  One thread per k-mer.
//   (d) target   read_mean / read_stdv from the template model's k-mer means (src/dtw_test.cpp:106-115): a float running
//                sum, then a float sum of double squares.  Serial per read, in the reference's order.
//   (e) normalise  Normalizer(read_mean, read_stdv) + set_signal + pop() (src/normalizer.cpp:22-44,105-129): the offline
//                normaliser of K1 (unc_norm_scale_shift) with the read's own target.  In place, one thread per read.
//
// The sweep is k_dtw (unc_dtw.cuh) over these device-resident means and k-mers.
#pragma once
#include "unc_device.cuh"
#include "unc_k1.cuh"
#include "unc_stream.cuh"

#define UNC_ALIGN_MAX_MEANS 50000u   /* dtw_test.cpp:156: "Takes up too much space" */

struct DevAlignRead {
    u64 kmer_off;                    // into DevAlign::kmers
    u64 pac_st;                      // .pac coordinate of the span's first base
    u32 n_kmers;                     // span length - 4
    u32 fwd;
};

struct DevAlign {
    float *events;                   // K1's rows (read r at r * ev_stride): raw event means in, kept normalised means out
    u32 ev_stride;
    const u32 *n_events;             // K1's event counts
    u32 *n_kept;                     // (b): unmasked events
    const DevAlignRead *q;
    u32 n;
    const u8 *pac;                   // 2-bit packed forward strand, 4 bases per byte, first base in the high bits
    const float *lv_mean;            // template model means, k-mer order of src/model_r94.inl
    u16 *kmers;
    float *tgt;                      // (d): (read_mean, read_stdv) per read
};

// (b) one read: get_full_mask's loop, each mask entry decided as EventProfiler::add_event pushes it
UNC_DEV void unc_align_mask(const DevAlign &A, u32 r) {
    float *ev = A.events + (size_t) r * A.ev_stride;
    const u32 ne = A.n_events[r];
    DevChanSig c;
    unc_evprof_reset(c);
    u32 m = 0, kept = 0;                                  // mask entries so far, kept means so far
    for (u32 i = 0; i < ne; i++) {
        const bool ready = unc_evprof_add(c, ev[i]);
        if (c.p_is_full) {                                // mask.push_back(to_mask_ == 0) for event m
            if (ready) ev[kept++] = c.next_mean;           // next_mean is ev[m]; kept <= m <= i, so the write is behind the reads
            m++;
        }
    }
    for (; m < ne; m++) {                                 // the tail loop (:142-149)
        if (c.to_mask == 0) ev[kept++] = ev[m];
        else c.to_mask--;
    }
    A.n_kept[r] = kept;
}

// (c) k-mer i of read r: bases [pac_st + i, pac_st + i + 5), first base most significant; reversed and complemented on -
UNC_DEV u16 unc_align_kmer(const DevAlign &A, const DevAlignRead &q, u32 i) {
    const u32 j = q.fwd ? i : q.n_kmers - 1u - i;
    u32 k = 0;
    for (u32 b = 0; b < 5u; b++) {
        const u64 p = q.pac_st + j + b;
        k = (k << 2) | ((A.pac[p >> 2] >> (((3u ^ (u32) p) & 3u) << 1)) & 3u);
    }
    if (q.fwd) return (u16) k;
    // kmer_revcomp: complement, reverse the 2-bit groups
    u32 rc = 0, x = k ^ 0x3FFu;
    for (u32 b = 0; b < 5u; b++) { rc = (rc << 2) | (x & 3u); x >>= 2; }
    return (u16) rc;
}

// (d) one read
UNC_DEV void unc_align_target(const DevAlign &A, u32 r) {
    const DevAlignRead q = A.q[r];
    const u16 *km = A.kmers + q.kmer_off;
    float mean = 0.0f;
    for (u32 i = 0; i < q.n_kmers; i++) mean = f_add(mean, A.lv_mean[km[i]]);
    mean = f_div(mean, (float) q.n_kmers);                           // float /= size_t
    float var = 0.0f;
    for (u32 i = 0; i < q.n_kmers; i++) {
        const double d = (double) f_sub(A.lv_mean[km[i]], mean);      // pow(float, 2): a double square, exact
        var = (float) d_add((double) var, d_mul(d, d));               // float += double
    }
    A.tgt[2 * r] = mean;
    A.tgt[2 * r + 1] = f_sqrt(f_div(var, (float) q.n_kmers));
}

// (e) one read
UNC_DEV void unc_align_norm(const DevAlign &A, u32 r) {
    const u32 n = A.n_kept[r];
    if (n == 0) return;
    float *ev = A.events + (size_t) r * A.ev_stride;
    float scale, shift;
    unc_norm_scale_shift(ev, n, A.tgt[2 * r], A.tgt[2 * r + 1], &scale, &shift);
    for (u32 i = 0; i < n; i++) ev[i] = f_add(f_mul(scale, ev[i]), shift);
}

// What the driver does with a read after (e) (dtw_test.cpp:156-159), and what the product does where the reference's
// behaviour is undefined: 0 = align, else the reason for skipping it.
enum { UNC_ALIGN_OK = 0, UNC_ALIGN_TOO_MANY_MEANS = 1, UNC_ALIGN_NO_EVENTS = 2, UNC_ALIGN_TOO_LARGE = 3 };
static inline int unc_align_verdict(uint32_t n_kept) {
    if (n_kept == 0) return UNC_ALIGN_NO_EVENTS;
    if (n_kept > UNC_ALIGN_MAX_MEANS) return UNC_ALIGN_TOO_MANY_MEANS;
    return UNC_ALIGN_OK;
}
