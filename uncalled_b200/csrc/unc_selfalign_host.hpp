// unc_selfalign_host.hpp -- host half of `self_align` (reference src/self_align_ref.cpp:34-91): WHICH
// reference positions are sampled.  The reference calls srand(0) and keeps position i of every sequence
// iff rand() % sample_dist == 0, one draw per position, sequences in .ann order; the sample set is
// therefore a function of glibc's rand().  GlibcRand restates that generator (glibc stdlib/random_r.c:
// TYPE_3, degree 31, separation 3 -- r[i] = r[i-31] + r[i-3], output >> 1, 310 outputs discarded after
// seeding with the 16807 Lehmer sequence) so that the sample set does not depend on the C library the
// product is linked against and the call leaves the process-global rand() state alone.
// Pure C++ (no CUDA): also compiled into the emulator library; tests compare it with libc's rand().
#pragma once
#include <stdint.h>
#include <vector>

struct GlibcRand {
    int32_t r[31];
    int f, b;
    explicit GlibcRand(unsigned seed = 1) { reseed(seed); }
    void reseed(unsigned seed) {
        if (seed == 0) seed = 1;                             // srandom_r: "we must make sure the seed is not 0"
        r[0] = (int32_t) seed;
        int32_t word = (int32_t) seed;
        for (int i = 1; i < 31; i++) {                       // word = 16807 * word % 2147483647 without overflow
            long hi = word / 127773, lo = word % 127773;
            long w = 16807 * lo - 2836 * hi;
            if (w < 0) w += 2147483647;
            r[i] = word = (int32_t) w;
        }
        f = 3; b = 0;
        for (int i = 0; i < 310; i++) next();
    }
    int next() {
        uint32_t v = (uint32_t) r[f] + (uint32_t) r[b];
        r[f] = (int32_t) v;
        if (++f == 31) f = 0;
        if (++b == 31) b = 0;
        return (int) (v >> 1);
    }
};

// Sampled start positions: pos[i] = index into the packed reference (.pac) of the path's first base,
// lim[i] = end (exclusive) of the sequence it lies in.  Sequences are laid out back to back (st += len).
static inline void unc_selfalign_sample(const std::vector<uint32_t> &seq_lens, uint32_t sample_dist,
                                        std::vector<uint32_t> &pos, std::vector<uint32_t> &lim) {
    GlibcRand rng(0);                                        // srand(0)
    uint64_t st = 0;
    for (uint32_t len : seq_lens) {
        for (uint64_t i = 0; i < len; i++) {
            if ((uint32_t) rng.next() % sample_dist != 0) continue;
            pos.push_back((uint32_t) (st + i));
            lim.push_back((uint32_t) (st + len));
        }
        st += len;
    }
}

// find-repeats: the .pac end (exclusive) of every sequence, sequences laid out back to back as above.  Zero-length
// sequences give repeated ends, which the device's search for the first end above a position skips.
static inline std::vector<uint32_t> unc_repeats_ends(const std::vector<uint32_t> &seq_lens) {
    std::vector<uint32_t> ends;
    uint64_t st = 0;
    for (uint32_t len : seq_lens) ends.push_back((uint32_t) (st += len));
    return ends;
}
