// unc_warp.cuh -- the thin warp-primitive layer the device code is written against.
//
// Under nvcc these are the sm_90a warp intrinsics.  Under -DUNC_EMUL (host build used by
// tests/test_emul_*.py) they are provided by tests/emul/warp_emul.hpp, a 32-fiber lockstep
// emulator, so that the *same* kernel source is exercised on a CPU-only box.  The emulator
// is a test vehicle for the device code, not a product path: libunc_b200.so never contains it.
#pragma once
#include <stdint.h>

#ifdef UNC_EMUL
#include "warp_emul.hpp"
#else
#include <cuda_runtime.h>
#define UNC_DEV __device__ __forceinline__
#define UNC_DEV_NOINLINE __device__ __noinline__
#define UNC_FULL 0xffffffffu

UNC_DEV int w_lane() { return (int) (threadIdx.x & 31); }
UNC_DEV int c_tid() { return (int) threadIdx.x; }
UNC_DEV int c_nthreads() { return (int) blockDim.x; }
UNC_DEV void c_sync() { __syncthreads(); }
// named barrier `id` (1..15) over `count` threads (a multiple of 32): bar.sync id, count
UNC_DEV void c_sync_sub(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
UNC_DEV void c_arrive_sub(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }
UNC_DEV void c_fence() { __threadfence_block(); }
#ifndef K2_SPIN_NS
#define K2_SPIN_NS 40
#endif
UNC_DEV void w_spin() { if (K2_SPIN_NS) __nanosleep(K2_SPIN_NS); }
UNC_DEV void w_sync() { __syncwarp(); }
UNC_DEV uint32_t w_ballot(int p) { return __ballot_sync(UNC_FULL, p); }
UNC_DEV uint32_t w_shfl(uint32_t v, int src) { return __shfl_sync(UNC_FULL, v, src); }
UNC_DEV float w_shflf(float v, int src) { return __shfl_sync(UNC_FULL, v, src); }
UNC_DEV uint32_t w_shfl_up(uint32_t v, int d) { return __shfl_up_sync(UNC_FULL, v, d); }
UNC_DEV uint32_t w_shfl_down(uint32_t v, int d) { return __shfl_down_sync(UNC_FULL, v, d); }
UNC_DEV uint32_t w_match(uint32_t v) { return __match_any_sync(UNC_FULL, v); }
UNC_DEV uint32_t d_atomic_add(uint32_t *p, uint32_t v) { return atomicAdd(p, v); }
UNC_DEV uint32_t d_atomic_or(uint32_t *p, uint32_t v) { return atomicOr(p, v); }
// 16-byte compare-and-swap on global memory (sm_90: ATOMG.E.CAS.128); p 16-byte aligned
UNC_DEV unsigned __int128 d_atomic_cas128(unsigned __int128 *p, unsigned __int128 cmp, unsigned __int128 v) {
    return atomicCAS(p, cmp, v);
}
UNC_DEV uint32_t s_atomic_add(uint32_t *p, uint32_t v) { return atomicAdd(p, v); }
UNC_DEV uint32_t s_atomic_or(uint32_t *p, uint32_t v) { return atomicOr(p, v); }
UNC_DEV uint32_t s_atomic_max(uint32_t *p, uint32_t v) { return atomicMax(p, v); }
UNC_DEV int d_popc(uint32_t v) { return __popc(v); }
UNC_DEV int d_popcll(uint64_t v) { return __popcll(v); }
UNC_DEV int d_clz(uint32_t v) { return __clz((int) v); }
UNC_DEV int d_ffs(uint32_t v) { return __ffs((int) v); }
UNC_DEV int d_clzll(uint64_t v) { return __clzll((long long) v); }
UNC_DEV int d_ctzll(uint64_t v) { return __ffsll((long long) v) - 1; }
// IEEE round-to-nearest, never contracted into FMA (the reference build has no FMA)
UNC_DEV float f_mul(float a, float b) { return __fmul_rn(a, b); }
UNC_DEV float f_add(float a, float b) { return __fadd_rn(a, b); }
UNC_DEV float f_sub(float a, float b) { return __fsub_rn(a, b); }
UNC_DEV float f_div(float a, float b) { return __fdiv_rn(a, b); }
UNC_DEV float f_sqrt(float a) { return __fsqrt_rn(a); }
UNC_DEV double d_mul(double a, double b) { return __dmul_rn(a, b); }
UNC_DEV double d_add(double a, double b) { return __dadd_rn(a, b); }
UNC_DEV double d_sub(double a, double b) { return __dsub_rn(a, b); }
UNC_DEV double d_div(double a, double b) { return __ddiv_rn(a, b); }
UNC_DEV double d_sqrt(double a) { return __dsqrt_rn(a); }
// x86-64 float -> u32 conversion as gcc emits it (cvttss2si to 64 bit, low half kept)
UNC_DEV uint32_t f_to_u32_x86(float v) { return (uint32_t) (long long) v; }
UNC_DEV uint64_t f_to_u64(float v) { return (uint64_t) v; }
template <typename T> UNC_DEV T d_ldg(const T *p) { return __ldg(p); }
// hint: bring the line holding *p towards the SM (no register is held while it is in flight)
UNC_DEV void d_prefetch(const void *p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
// single 128-bit volatile shared-memory accesses (one transaction: payload + flag together)
UNC_DEV uint4 s_load_v4(const uint4 *p) {
    uint4 v;
    unsigned a = (unsigned) __cvta_generic_to_shared(p);
    asm volatile("ld.volatile.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}
UNC_DEV void s_store_v4(uint4 *p, uint4 v) {
    unsigned a = (unsigned) __cvta_generic_to_shared(p);
    asm volatile("st.volatile.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
UNC_DEV uint64_t s_load_u64(const uint64_t *p) {
    uint64_t v;
    unsigned a = (unsigned) __cvta_generic_to_shared(p);
    asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(v) : "r"(a) : "memory");
    return v;
}
UNC_DEV void s_store_u64(uint64_t *p, uint64_t v) {
    unsigned a = (unsigned) __cvta_generic_to_shared(p);
    asm volatile("st.volatile.shared.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory");
}
UNC_DEV float u2f(uint32_t v) { return __uint_as_float(v); }
UNC_DEV uint32_t f2u(float v) { return __float_as_uint(v); }
// explicit fused multiply-add (used only where the reference result is reproduced through an exactly
// rounded division sequence, never as a contraction of a*b+c)
UNC_DEV double d_fma(double a, double b, double c) { return __fma_rn(a, b, c); }
UNC_DEV float f_fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
UNC_DEV double u2d(uint64_t v) { return __longlong_as_double((long long) v); }
UNC_DEV uint64_t d2u(double v) { return (uint64_t) __double_as_longlong(v); }
// ---- bulk asynchronous copy global -> shared (TMA, cp.async.bulk) completing on an mbarrier
UNC_DEV void t_bar_init(uint64_t *bar) {
    unsigned a = (unsigned) __cvta_generic_to_shared(bar);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(a) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// orders this thread's earlier generic-proxy accesses to shared memory before later async-proxy ones
UNC_DEV void t_fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// one thread: arm the barrier with `bytes` and start the copy (dst, src 16-byte aligned, bytes % 16 == 0)
UNC_DEV void t_bulk_load(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    unsigned b = (unsigned) __cvta_generic_to_shared(bar), d = (unsigned) __cvta_generic_to_shared(dst);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(d), "l"(src), "r"(bytes), "r"(b) : "memory");
}
// per-thread asynchronous 16-byte copies global -> shared (cp.async, LDGSTS): no registers held
UNC_DEV void a_copy16(void *dst, const void *src) {
    unsigned d = (unsigned) __cvta_generic_to_shared(dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(src) : "memory");
}
UNC_DEV void a_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
UNC_DEV void a_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
UNC_DEV void t_bar_wait(uint64_t *bar, uint32_t parity) {
    unsigned b = (unsigned) __cvta_generic_to_shared(bar);
    asm volatile("{\n.reg .pred p;\nWAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}"
                 ::"r"(b), "r"(parity) : "memory");
}
#endif

UNC_DEV uint32_t w_lanemask_lt() { return (1u << w_lane()) - 1u; }

// exclusive prefix sum over the warp; *total receives the warp sum (uniform)
UNC_DEV uint32_t w_exscan(uint32_t v, uint32_t *total) {
    uint32_t x = v;
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t y = w_shfl_up(x, d);
        if (w_lane() >= d) x += y;
    }
    *total = w_shfl(x, 31);
    return x - v;
}

UNC_DEV uint64_t w_shfl64(uint64_t v, int src) {
    return ((uint64_t) w_shfl((uint32_t) (v >> 32), src) << 32) | w_shfl((uint32_t) v, src);
}
UNC_DEV uint64_t w_shfl_up64(uint64_t v, int d) {
    return ((uint64_t) w_shfl_up((uint32_t) (v >> 32), d) << 32) | w_shfl_up((uint32_t) v, d);
}

UNC_DEV uint32_t w_max(uint32_t v) {
    for (int d = 16; d > 0; d >>= 1) {
        uint32_t y = w_shfl(v, w_lane() ^ d);
        v = y > v ? y : v;
    }
    return v;
}
