/*
 * TEST INFRASTRUCTURE -- tests/simt/cuda_runtime.h
 *
 * A stand-in for <cuda_runtime.h> that lets the product's DEVICE code (the .cuh files under zxc_b200/csrc) compile with
 * g++ and run on the CPU, one emulated warp = 32 fibers in one OS thread (simt_rt.h).  Every warp-level
 * primitive (__shfl*_sync, __ballot_sync, __syncwarp, ...) is a rendezvous of the lanes its mask names: a lane
 * that reaches one parks, the scheduler resumes the other lanes in a (seeded) random order until every lane of
 * the mask has arrived at the same primitive with the same mask, computes the group's results over the mask
 * and lets it continue; disjoint groups (partial masks) complete independently.  Between two rendezvous the lanes run one
 * after another in that random order, so code that needs an ordering the source does not ask for with a
 * __syncwarp() shows up as a mismatch -- and a lane that skips a rendezvous the others take deadlocks
 * loudly.  Nothing here is linked into libzxc.so; the tests use it to check the kernels' logic against
 * the reference without a GPU.
 */
#pragma once
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __noinline__
#define __shared__
#define __align__(x) __attribute__((aligned(x)))
#define __launch_bounds__(...)
#define __restrict__

struct uint2 { uint32_t x, y; };
struct alignas(16) uint4 { uint32_t x, y, z, w; };
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }
struct dim3 { unsigned x, y, z; };

#include "simt_rt.h"

#define threadIdx (simt::cur().tid)
#define blockIdx (simt::cur().bid)
#define blockDim (simt::cur().bdim)
static const dim3 gridDim = {1, 1, 1}; /* the harnesses launch the warps of one grid-stride loop as a grid of one block */

/* ---- warp primitives: the mask names the lanes that take part (simt_rt.cc run_warp) ---- */
static inline void __syncwarp(unsigned mask = 0xFFFFFFFFu) { simt::rendezvous(simt::OP_SYNC, 0, 0, mask); }
static inline unsigned __ballot_sync(unsigned m, int pred) { return (unsigned)simt::rendezvous(simt::OP_BALLOT, pred != 0, 0, m); }
static inline int __any_sync(unsigned m, int pred) { return simt::rendezvous(simt::OP_BALLOT, pred != 0, 0, m) != 0; }
static inline int __all_sync(unsigned m, int pred) { return (unsigned)simt::rendezvous(simt::OP_BALLOT, pred != 0, 0, m) == m; }
static inline unsigned __reduce_max_sync(unsigned m, unsigned v) { return (unsigned)simt::rendezvous(simt::OP_MAX, v, 0, m); }
static inline unsigned __reduce_min_sync(unsigned m, unsigned v) { return (unsigned)simt::rendezvous(simt::OP_MIN, v, 0, m); }
static inline unsigned __reduce_add_sync(unsigned m, unsigned v) { return (unsigned)simt::rendezvous(simt::OP_ADD, v, 0, m); }
static inline unsigned __reduce_or_sync(unsigned m, unsigned v) { return (unsigned)simt::rendezvous(simt::OP_OR, v, 0, m); }
static inline unsigned __match_any_sync(unsigned m, unsigned long long v) { return (unsigned)simt::rendezvous(simt::OP_MATCH, v, 0, m); }

template <class T> static inline T simt_shfl(int op, unsigned mask, T v, unsigned arg) {
    static_assert(sizeof(T) <= 8, "shuffle of at most 64 bits");
    uint64_t raw = 0;
    memcpy(&raw, &v, sizeof(T));
    raw = simt::rendezvous(op, raw, arg, mask);
    T r;
    memcpy(&r, &raw, sizeof(T));
    return r;
}
template <class T> static inline T __shfl_sync(unsigned m, T v, int src, int width = 32) { (void)width; return simt_shfl(simt::OP_SHFL_IDX, m, v, (unsigned)src & 31u); }
template <class T> static inline T __shfl_up_sync(unsigned m, T v, unsigned d, int width = 32) { (void)width; return simt_shfl(simt::OP_SHFL_UP, m, v, d); }
template <class T> static inline T __shfl_down_sync(unsigned m, T v, unsigned d, int width = 32) { (void)width; return simt_shfl(simt::OP_SHFL_DOWN, m, v, d); }
template <class T> static inline T __shfl_xor_sync(unsigned m, T v, int x, int width = 32) { (void)width; return simt_shfl(simt::OP_SHFL_XOR, m, v, (unsigned)x); }

/* ---- scalar intrinsics ---- */
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline int __ffsll(long long v) { return __builtin_ffsll(v); }
static inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
static inline int __clzll(long long v) { return v ? __builtin_clzll((unsigned long long)v) : 64; }
static inline unsigned __brev(unsigned v) {
    v = ((v >> 1) & 0x55555555u) | ((v & 0x55555555u) << 1);
    v = ((v >> 2) & 0x33333333u) | ((v & 0x33333333u) << 2);
    v = ((v >> 4) & 0x0F0F0F0Fu) | ((v & 0x0F0F0F0Fu) << 4);
    return __builtin_bswap32(v);
}
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned s) { /* ((hi:lo) >> (s & 31)) low word */
    s &= 31u;
    return s ? (lo >> s) | (hi << (32u - s)) : lo;
}
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned s) { /* ((hi:lo) << (s & 31)) high word */
    s &= 31u;
    return s ? (hi << s) | (lo >> (32u - s)) : hi;
}
static inline unsigned long long __umul64hi(unsigned long long a, unsigned long long b) { return (unsigned long long)(((unsigned __int128)a * b) >> 64); }
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((uint64_t)a * b) >> 32); }
static inline float __fdividef(float a, float b) { return a / b; }
static inline unsigned __float2uint_rz(float f) { return f <= 0.f ? 0u : (unsigned)f; }
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned s) {
    const uint64_t v = ((uint64_t)b << 32) | a;
    unsigned r = 0;
    for (int i = 0; i < 4; i++) {
        const unsigned sel = (s >> (4 * i)) & 0xF;
        unsigned byte = (unsigned)(v >> (8 * (sel & 7))) & 0xFF;
        if (sel & 8) byte = (byte & 0x80) ? 0xFF : 0;
        r |= byte << (8 * i);
    }
    return r;
}
template <class T> static inline T min(T a, T b) { return b < a ? b : a; }
template <class T> static inline T max(T a, T b) { return a < b ? b : a; }
static inline unsigned min(unsigned a, int b) { return min(a, (unsigned)b); }
static inline unsigned max(unsigned a, int b) { return max(a, (unsigned)b); }
static inline unsigned min(int a, unsigned b) { return min((unsigned)a, b); }
static inline unsigned max(int a, unsigned b) { return max((unsigned)a, b); }

/* ---- atomics: lanes of one emulated warp never run concurrently, warps of one process neither ---- */
template <class T> static inline T atomicAdd(T* p, T v) { const T o = *p; *p = o + v; return o; }
template <class T> static inline T atomicMin(T* p, T v) { const T o = *p; if (v < o) *p = v; return o; }
template <class T> static inline T atomicMax(T* p, T v) { const T o = *p; if (v > o) *p = v; return o; }
template <class T> static inline T atomicOr(T* p, T v) { const T o = *p; *p = o | v; return o; }
template <class T> static inline T atomicAnd(T* p, T v) { const T o = *p; *p = o & v; return o; }
template <class T> static inline T atomicExch(T* p, T v) { const T o = *p; *p = v; return o; }
template <class T> static inline T atomicCAS(T* p, T c, T v) { const T o = *p; if (o == c) *p = v; return o; }
static inline long long clock64() { return 0; }
static inline void __threadfence() {}
static inline void __threadfence_block() {}
