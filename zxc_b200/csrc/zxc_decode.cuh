/*
 * zxc_decode.cuh -- sm_90a block-decode kernels (device code only).
 *
 * One warp per independent block (SURVEY.md section 8 rows D1-D9); lane = sequence,
 * 32 sequences per batch:
 *   1. token / offset unpack               (GLO zxc_decompress.c:626-694, GHI :701-727)
 *   2. escape resolution over the extras   (varint, :51-88): every value of the section is computed once per block
 *      by a segment-map scan; a lane takes the value(s) whose ordinal (ballot + popc) is its own
 *   3. warp prefix sums -> literal source offset and output offset per lane
 *   4. bounds / offset validation; first failing lane == first failing sequence
 *   5. two copy passes -- every literal run, then every match whose source ends at or below the batch's first output
 *      byte (short items per lane, long ones as balanced 16-byte chunks over the warp) -- and the matches that read
 *      the batch's own output one after the other in sequence order
 *   6. the output is staged in a per-warp shared-memory ring and leaves the SM as coalesced
 *      16-byte stores (512 B per warp instruction); match sources come from the ring when they
 *      are recent and from global memory (L2) once flushed.
 * The block format and the presence of a dictionary are template parameters (decode_lz_block<UNITS, GHI, HAS_DICT, LEAN>).
 * The LEAN kernel instance decodes only RAW blocks and GLO blocks with raw or RLE literals and raw tokens, and defers
 * every other block to the general instance (decode_job).  Without a dictionary it reads a batch's tokens, offsets and
 * first 32 escape values from a per-warp look-ahead slot behind the ring, filled by cp.async while the batch before it copies (ZXC_LOOKAHEAD).
 * zxc_decode_stage.cuh holds the opt-in TMA flavour (sections staged by cp.async.bulk, ring flushed by bulk stores).
 * Overlapping matches (off < ml) use the period-`off` index instead of the reference's shuffle
 * tables (:197-413).  Output is written exactly (no wild-copy overshoot): none of the
 * reference's PAD / TAIL_PAD slack is needed on the destination; the wire-level 32-byte
 * literal slack rule stays normative (:1003).
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "zxc_b200.h"
#include "zxc_error.h"

typedef uint8_t u8;
typedef uint32_t u32;
typedef uint64_t u64;
typedef int32_t i32;

#define FULL 0xFFFFFFFFu
/* small steps of the sequence-centric body, switchable at build time for A/B measurements; every setting is bit-exact */
#ifndef ZXC_FASTMOD
#define ZXC_FASTMOD 1 /* period replication without integer division */
#endif
#ifndef ZXC_TAIL_SMEM
#define ZXC_TAIL_SMEM 1 /* shared-space byte copies in the sequence-order tail */
#endif
#ifndef ZXC_ALIGNED_LD
#define ZXC_ALIGNED_LD 1 /* one 16 / 32-bit load per offset / GHI word when the section is aligned */
#endif
#ifndef ZXC_HINTS
#define ZXC_HINTS 0 /* branch hints on the cold paths */
#endif
#if ZXC_HINTS
#define ZXC_RARE(x) __builtin_expect(!!(x), 0)
#else
#define ZXC_RARE(x) (x)
#endif
#ifndef ZXC_STAT
#define ZXC_STAT(i, v) /* tests/simt counts events here (lane 0 only); nothing in the product build */
#endif
#ifndef WARPS_PER_CTA
#define WARPS_PER_CTA 4
#endif
#define CTA_THREADS (WARPS_PER_CTA * 32)
#ifndef RING_BYTES
#define RING_BYTES 4096u          /* per-warp output ring (power of two, multiple of 512) */
#endif
#define RING_LIMIT (RING_BYTES - 576u) /* largest output span one batch may add */
#ifndef CTAS_PER_SM
#define CTAS_PER_SM 7u            /* register-limited (72 regs x 128 threads); 112 KB of rings, rest is L1 */
#endif
#ifndef LEAN_CTAS_PER_SM
#define LEAN_CTAS_PER_SM 8u /* the lean instance's own launch bounds: 64 registers without spills (DESIGN.md section 9) */
#endif
#ifndef LEAN_SMEM_PAD
#define LEAN_SMEM_PAD 0u /* development: extra dynamic shared memory per lean CTA, to move the carve-out step alone */
#endif

#define BT_RAW 0
#define BT_GLO 1
#define BT_GHI 2
#define BT_EOF 255

#define FLAG_VERIFY 1u
#define FLAG_UNITS_ON 4u
#define FLAG_UNITS_OFF 8u
#define FLAG_DEFERRED 2u /* only jobs whose status says D2_DEFER (left over by the lean instance) */
#define D2_DEFER_STATUS ((i32)0x80000000)

struct DecodeParams {
    const u8* src;
    u8* dst;
    const zxc_b200_job_t* jobs;
    i32* status;
    const u8* dict;
    const u8* dict_huf;
    u8* scratch;
    unsigned long long* counter;
    u32 n_jobs;
    u32 dict_size;
    u32 scratch_stride;
    u32 flags;
    u32 block_cap; /* largest decoded block size of this launch: sizes the per-warp scratch regions */
    u32* defer_list;  /* job indices the lean instance left to a FLAG_DEFERRED launch ... */
    u32* defer_count; /* ... how many; more than defer_cap means "scan the status array instead" */
    u32 defer_cap;
};

/* this warp's scratch, past the 256-byte lead-in where word loads may start */
__host__ __device__ __forceinline__ u8* warp_scratch(const DecodeParams& P, u32 gwarp) {
    return P.scratch + (size_t)gwarp * P.scratch_stride + 256;
}

/* ------------------------------------------------------------------------- */
/* small device helpers                                                      */
/* ------------------------------------------------------------------------- */
__device__ __forceinline__ u32 ld16(const u8* p) { return (u32)p[0] | ((u32)p[1] << 8); }
__device__ __forceinline__ u32 ld32(const u8* p) {
    return (u32)p[0] | ((u32)p[1] << 8) | ((u32)p[2] << 16) | ((u32)p[3] << 24);
}
__device__ __forceinline__ u64 ld64(const u8* p) { return (u64)ld32(p) | ((u64)ld32(p + 4) << 32); }

__device__ __forceinline__ u32 warp_incl_scan(u32 v, u32 lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const u32 t = __shfl_up_sync(FULL, v, d);
        if (lane >= (u32)d) v += t;
    }
    return v;
}

/* Explicit shared-memory stores.  With the ring as an ordinary pointer ptxas re-derives the CTA's shared window base
 * (S2R SR_CgaCtaId, MOV, LEA, IADD) in front of every predicated STS of the copy helpers instead of holding it in a
 * register -- four extra instructions per store.  A 32-bit shared address made opaque once per block cannot be
 * re-derived, so it stays in a register (or one LDL away).  The host versions serve the CPU emulator (tests/simt). */
#ifdef __CUDACC__
__device__ __forceinline__ u32 smem_addr(const void* p) {
    u32 a = (u32)__cvta_generic_to_shared(p);
    asm volatile("" : "+r"(a));
    return a;
}
template <int OFF> __device__ __forceinline__ void sts32(u32 a, u32 v) {
    asm volatile("st.shared.u32 [%0+%2], %1;" ::"r"(a), "r"(v), "n"(OFF) : "memory");
}
template <int OFF> __device__ __forceinline__ void sts16(u32 a, u32 v) {
    asm volatile("st.shared.u16 [%0+%2], %1;" ::"r"(a), "h"((unsigned short)v), "n"(OFF) : "memory");
}
template <int OFF> __device__ __forceinline__ void sts8(u32 a, u32 v) {
    asm volatile("st.shared.u8 [%0+%2], %1;" ::"r"(a), "r"(v), "n"(OFF) : "memory");
}
/* v, hidden from the compiler's value tracking: what is derived from it is computed where it is used instead of being
 * hoisted out of the loop and held in registers across it */
__device__ __forceinline__ u32 opaque(u32 v) {
    asm volatile("" : "+r"(v));
    return v;
}
/* generic pointer of shared address a, derived anew at every call */
__device__ __forceinline__ u8* ring_at(u32 a) { return reinterpret_cast<u8*>(__cvta_shared_to_generic((size_t)opaque(a))); }
/* the warp's index in the grid, read from the special registers anew at every call */
__device__ __forceinline__ u32 grid_warp_now() {
    u32 t, c;
    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
    asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(c));
    return c * WARPS_PER_CTA + (t >> 5);
}
#else
extern u8 smem[];
static inline u32 smem_addr(const void* p) { return (u32)(reinterpret_cast<const u8*>(p) - smem); }
static inline u32 opaque(u32 v) { return v; }
static inline u8* ring_at(u32 a) { return smem + a; }
static inline u32 grid_warp_now() { return blockIdx.x * WARPS_PER_CTA + (threadIdx.x >> 5); }
template <int OFF> static inline void sts32(u32 a, u32 v) { memcpy(smem + a + OFF, &v, 4); }
template <int OFF> static inline void sts16(u32 a, u32 v) { const unsigned short h = (unsigned short)v; memcpy(smem + a + OFF, &h, 2); }
template <int OFF> static inline void sts8(u32 a, u32 v) { smem[a + OFF] = (u8)v; }
#endif

/* L1 prefetch of the 128-byte line that holds p: a hint that never faults and returns nothing, so no instruction
 * waits on it.  The emulator has no caches. */
#ifdef __CUDACC__
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
#else
static inline void prefetch_l1(const void*) {}
#endif

/* Development flavour (make NVEXTRA=-DZXC_TRACE=1 OUT=<elsewhere>): lane 0 of every warp adds clock64() deltas per
 * phase of the sequence-centric body, and event counts, to its row of zxc_trace_acc; zxc_b200_trace_read() returns
 * the rows (profiles/trace_decode.py).  In the product build the hooks expand to nothing. */
#if ZXC_TRACE
#define TRACE_SLOTS 16
#define TRACE_ROWS 8192
enum {
    TR_UNPACK, TR_SCAN, TR_LIT, TR_MATCH, TR_TAIL, TR_FLUSH, TR_START, TR_END, TR_GIANT, TR_CLAIM,
    TR_BATCHES, TR_BLOCKS, TR_M_RING, TR_M_GLOBAL, TR_M_DICT, TR_M_SEQ
};
__device__ unsigned long long zxc_trace_acc[TRACE_ROWS * TRACE_SLOTS];
__device__ __forceinline__ void trace_add(u32 slot, unsigned long long v, u32 lane) {
    const u32 row = blockIdx.x * WARPS_PER_CTA + (threadIdx.x >> 5);
    if (lane == 0 && row < TRACE_ROWS) atomicAdd(&zxc_trace_acc[row * TRACE_SLOTS + slot], v);
}
#define ZXC_TRACE_DECL long long tr_t = clock64()
#define ZXC_TRACE_MARK(slot, lane)                               \
    do {                                                         \
        const long long tr_n = clock64();                        \
        trace_add(slot, (unsigned long long)(tr_n - tr_t), lane); \
        tr_t = tr_n;                                             \
    } while (0)
#define ZXC_TRACE_ADD(slot, v, lane) trace_add(slot, (unsigned long long)(v), lane)
#else
#define ZXC_TRACE_DECL
#define ZXC_TRACE_MARK(slot, lane)
#define ZXC_TRACE_ADD(slot, v, lane)
#endif

#include "zxc_decode_stage.cuh"
#define WARP_SMEM_BYTES (RING_BYTES + STAGE_BYTES) /* a warp's output ring, its staging area right behind */
#define DECODE_SMEM_BYTES (WARPS_PER_CTA * WARP_SMEM_BYTES)

/* The lean instance without a dictionary stages the next batch's tokens, offsets and escape values into a per-warp look-ahead slot right
 * behind the ring by cp.async, one batch ahead (DESIGN.md section 3a step 8).  -DZXC_LOOKAHEAD=0 builds it without
 * the slot, for A/B timing; every other instance is the same either way. */
#ifndef ZXC_LOOKAHEAD
#define ZXC_LOOKAHEAD (!ZXC_STAGE)
#endif
#if ZXC_LOOKAHEAD && ZXC_STAGE
#error "ZXC_LOOKAHEAD and ZXC_STAGE both stage the token and offset sections: build with one of them"
#endif
#define LA_SLOT_BYTES (ZXC_LOOKAHEAD ? 256u : 0u)
#define LA_OFF 48u  /* slot bytes [0, 48): token words; [48, 128): offset words */
#define LA_ESC 128u /* [128, 256): the batch's first 32 escape values */
#define LEAN_WARP_SMEM_BYTES (WARP_SMEM_BYTES + LA_SLOT_BYTES)
/* dynamic shared memory of the lean launch without a dictionary; the one with a dictionary has no slot */
#define LEAN_SMEM_BYTES (WARPS_PER_CTA * LEAN_WARP_SMEM_BYTES + LEAN_SMEM_PAD)
/* which instance carries the slot: the lean one without a dictionary (with one it measured slower, DESIGN.md 3d) */
template <bool HAS_DICT, bool LEAN> __host__ __device__ constexpr bool la_on() {
    return LEAN && !HAS_DICT && ZXC_LOOKAHEAD != 0;
}

/* 4-byte global -> shared copy that holds no register until it lands; cp_async_wait_all() waits for this thread's */
#ifdef __CUDACC__
__device__ __forceinline__ void cp_async4(u32 sdst, const void* gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(sdst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void cp_async_check_idle() {}
#else
/* CPU emulator (tests/simt): a copy fills its destination with a poison pattern when it is issued and moves the data
 * only at the issuing lane's wait, the latest moment the hardware may take.  A read before that lane's wait -- a
 * missing wait, or a missing __syncwarp() between the other lanes' waits and the read -- sees the poison. */
struct SimtCpAsync {
    u32 s;
    const u8* g;
};
inline SimtCpAsync simt_cp_pending[32][8];
inline u32 simt_cp_n[32];
static inline void simt_cp_fail(const char* what) {
    fprintf(stderr, "simt cp.async check failed: %s\n", what);
    abort();
}
static inline void cp_async4(u32 sdst, const void* gsrc) {
    const int l = simt::g_warp->current;
    if ((sdst & 3u) || (reinterpret_cast<uintptr_t>(gsrc) & 3u)) simt_cp_fail("4-byte copy not 4-byte aligned");
    if (simt_cp_n[l] >= 8) simt_cp_fail("more copies in flight than a lane issues per batch");
    memset(smem + sdst, 0xE7, 4);
    simt_cp_pending[l][simt_cp_n[l]++] = SimtCpAsync{sdst, static_cast<const u8*>(gsrc)};
}
static inline void cp_async_wait_all() {
    const int l = simt::g_warp->current;
    for (u32 k = 0; k < simt_cp_n[l]; k++) memcpy(smem + simt_cp_pending[l][k].s, simt_cp_pending[l][k].g, 4);
    simt_cp_n[l] = 0;
}
/* a block starts with no copy of this lane in flight: the previous one waited for all it issued */
static inline void cp_async_check_idle() {
    if (simt_cp_n[simt::g_warp->current]) simt_cp_fail("a copy was still in flight when the previous block ended");
}
#endif

#include "zxc_huffman.cuh"

/* per-warp scratch layout (bytes), a function of the launch's block_cap */
__host__ __device__ __forceinline__ u32 scr_lit_cap(u32 bs) { return (bs + 255u) & ~255u; }
__host__ __device__ __forceinline__ u32 scr_tok_cap(u32 bs) { return (bs / 4u + 64u + 255u) & ~255u; }
/* rank words of the PivCo decode, worst case: HUF_MAXLEN (11) bitmap levels over every literal + one per node */
__host__ __device__ __forceinline__ u32 scr_cum_cap(u32 bs) {
    return (11u * (scr_lit_cap(bs) / 8u) + 4u * 512u + 255u) & ~255u;
}
__host__ __device__ __forceinline__ u32 scr_stride(u32 bs) {
    return 256u + scr_lit_cap(bs) + scr_tok_cap(bs) + (u32)HUF_WORK_BYTES + scr_cum_cap(bs);
}

/* warp-wide byte copy, global -> global, non-overlapping */
__device__ __forceinline__ void warp_copy(u8* d, const u8* s, u32 n, u32 lane) {
    u32 k = lane;
    for (; k + 96 < n; k += 128) {
        const u8 a = s[k], b = s[k + 32], c = s[k + 64], e = s[k + 96];
        d[k] = a;
        d[k + 32] = b;
        d[k + 64] = c;
        d[k + 96] = e;
    }
    for (; k < n; k += 32) d[k] = s[k];
}

/* prefix varint with the reference's exact failure behaviour (zxc_decompress.c:51-88):
 * value 0 and the cursor jams to `end`, except at/after end where it stays. */
__device__ __forceinline__ u32 read_varint(const u8* e, u32& pos, u32 end) {
    if (pos >= end) return 0;
    const u32 b0 = e[pos];
    if (b0 < 0x80) {
        pos += 1;
        return b0;
    }
    if (b0 < 0xC0) {
        if (pos + 1 >= end) {
            pos = end;
            return 0;
        }
        const u32 v = (b0 & 0x3F) | ((u32)e[pos + 1] << 6);
        pos += 2;
        return v;
    }
    if (b0 < 0xE0) {
        if (pos + 2 >= end) {
            pos = end;
            return 0;
        }
        const u32 v = (b0 & 0x1F) | ((u32)e[pos + 1] << 5) | ((u32)e[pos + 2] << 13);
        pos += 3;
        return v;
    }
    pos = end;
    return 0;
}

/* cursor after one varint, advancing exactly as read_varint would */
__device__ __forceinline__ u32 varint_advance(const u8* e, u32 pos, u32 end) {
    if (pos >= end) return pos;
    const u32 b0 = e[pos];
    const u32 nxt = pos + 1u + (b0 >> 7) + ((b0 & 0xC0u) == 0xC0u);
    return (b0 >= 0xE0u || nxt > end) ? end : nxt;
}

/* ------------------------------------------------------------------------- */
/* rapidhash V3 folded to 32 bits, warp-cooperative (vendors/rapidhash.h).    */
/* Lanes 0..6 own the seven stripe accumulators; the tail is warp-uniform.    */
/* ------------------------------------------------------------------------- */
__device__ __forceinline__ u64 mul_fold(u64 a, u64 b) { return (a * b) ^ __umul64hi(a, b); }

__device__ u32 warp_checksum(const u8* p, u32 len, u32 lane) {
    const u64 S0 = 0x2d358dccaa6c78a5ull, S1 = 0x8bb84b93962eacc9ull, S2 = 0x4b33a62ed433d4a3ull,
              S3 = 0x4d5a2da51de1aa47ull, S4 = 0xa0761d6478bd642full, S5 = 0xe7037ed1a0b428dbull,
              S6 = 0x90ed1765281c388cull, S7 = 0xaaaaaaaaaaaaaaaaull;
    u64 seed = 0;
    seed ^= mul_fold(seed ^ S2, S1);
    u64 a = 0, b = 0;
    u32 rem = len;
    if (len <= 16) {
        if (len >= 8) {
            seed ^= len;
            a = ld64(p);
            b = ld64(p + len - 8);
        } else if (len >= 4) {
            seed ^= len;
            a = ld32(p);
            b = ld32(p + len - 4);
        } else if (len > 0) {
            a = ((u64)p[0] << 45) | p[len - 1];
            b = p[len >> 1];
        }
    } else {
        if (len > 112) {
            const u64 sk = lane == 0 ? S0 : lane == 1 ? S1 : lane == 2 ? S2 : lane == 3 ? S3
                         : lane == 4 ? S4 : lane == 5 ? S5 : S6;
            u64 acc = seed;
            const u32 stripes = (len - 1) / 112; /* while (rem > 112) */
            if (lane < 7) {
                const u8* q = p + 16 * lane;
                for (u32 s = 0; s < stripes; s++, q += 112) acc = mul_fold(ld64(q) ^ sk, ld64(q + 8) ^ acc);
            }
            u64 x = (lane < 7) ? acc : 0;
#pragma unroll
            for (int d = 4; d >= 1; d >>= 1) x ^= __shfl_xor_sync(FULL, x, d);
            seed = __shfl_sync(FULL, x, 0); /* lanes 0..7 xor-reduced: accumulators 0..6 */
            p += (size_t)stripes * 112;
            rem -= stripes * 112;
        }
        const u64 ts[6] = {S2, S2, S1, S1, S2, S1};
#pragma unroll
        for (u32 k = 0; k < 6; k++)
            if (rem > 16u * (k + 1)) seed = mul_fold(ld64(p + 16 * k) ^ ts[k], ld64(p + 16 * k + 8) ^ seed);
        a = ld64(p + rem - 16) ^ rem;
        b = ld64(p + rem - 8);
    }
    a ^= S1;
    b ^= seed;
    const u64 lo = a * b, hi = __umul64hi(a, b);
    const u64 h = mul_fold(lo ^ S7, hi ^ S1 ^ rem);
    return (u32)(h ^ (h >> 32));
}

/* ------------------------------------------------------------------------- */
/* RLE literal section -> scratch (zxc_decompress.c:906-978)                  */
/* ------------------------------------------------------------------------- */
__device__ int rle_expand(const u8* r, u32 rsz, u8* w, u32 wsz, u32 lane) {
    u32 rp = 0, wp = 0;
    while (rp < rsz && wp < wsz) {
        const u32 t = r[rp++];
        if (!(t & 0x80)) {
            const u32 len = t + 1;
            if (wsz - wp < len || rsz - rp < len) return ZXC_ERROR_CORRUPT_DATA;
            for (u32 k = lane; k < len; k += 32) w[wp + k] = r[rp + k];
            wp += len;
            rp += len;
        } else {
            const u32 len = (t & 0x7F) + 4;
            if (wsz - wp < len || rp >= rsz) return ZXC_ERROR_CORRUPT_DATA;
            const u8 v = r[rp++];
            for (u32 k = lane; k < len; k += 32) w[wp + k] = v;
            wp += len;
        }
    }
    return wp == wsz ? ZXC_OK : ZXC_ERROR_CORRUPT_DATA;
}

/* ------------------------------------------------------------------------- */
/* section layout of a GLO / GHI payload (zxc_common.c:773-832 +              */
/* zxc_decompress.c:859-1023, :1241-1269), checks in the reference's order    */
/* ------------------------------------------------------------------------- */
struct Sections {
    const u8* lit;
    const u8* tok;  /* GLO tokens or GHI sequence words */
    const u8* offs; /* GLO offsets */
    const u8* ext;
    u32 ext_end;
    u32 n_lit_avail;
    u32 n_seq;
    u32 enc_off;
};

/* LEAN: the caller has deferred every block with Huffman literals or tokens, so the PivCo decoder is not compiled in;
 * the token section always starts at S.lit + S.n_lit_avail (the decode loop holds no pointer of its own for it) */
template <bool LEAN>
__device__ int parse_sections(const u8* pay, u32 comp, bool ghi, u32 cap, const u8* dict_huf, u8* scratch,
                              u32 block_cap, u32 lane, Sections& S) {
    /* scratch points at this warp's literal buffer; token buffer, Huffman work area follow */
    const u32 scratch_cap = scr_lit_cap(block_cap);
    u8* tok_buf = scratch + scratch_cap;
    HufWork* hw = reinterpret_cast<HufWork*>(tok_buf + scr_tok_cap(block_cap));
    u32* cum = reinterpret_cast<u32*>(reinterpret_cast<u8*>(hw) + HUF_WORK_BYTES);
    const u32 cum_words = scr_cum_cap(block_cap) / 4u;
    if (comp < 12) return ZXC_ERROR_BAD_HEADER;
    const u32 n_seq = ld32(pay), n_lit = ld32(pay + 4);
    const u32 enc_lit = pay[8], enc_tok = pay[9], enc_off = pay[11];
    S.n_seq = n_seq;
    S.enc_off = enc_off;
    S.offs = 0;
    if (!ghi) {
        const u32 desc = (enc_lit != 0 ? 4u : 0u) + (enc_tok == 2 ? 4u : 0u);
        if (comp < 12 + desc) return ZXC_ERROR_BAD_HEADER;
        u32 lit_comp = n_lit, tok_comp = n_seq;
        const u8* dp = pay + 12;
        if (enc_lit != 0) {
            lit_comp = ld32(dp);
            dp += 4;
        }
        if (enc_tok == 2) tok_comp = ld32(dp);
        if (enc_off > 1) return ZXC_ERROR_CORRUPT_DATA;
        const u8* p_data = pay + 12 + desc;
        const u32 avail = comp - 12 - desc;
        if (!LEAN && (enc_lit == 2 || enc_lit == 3)) {
            if (lit_comp > avail) return ZXC_ERROR_CORRUPT_DATA;
            if (n_lit != 0) {
                if (n_lit > cap) return ZXC_ERROR_DST_TOO_SMALL;
                if (enc_lit == 3 && !dict_huf) return ZXC_ERROR_DICT_REQUIRED;
                if (n_lit > scratch_cap) return ZXC_ERROR_CORRUPT_DATA; /* lit_buffer_cap, :774 */
                int rc;
                if (enc_lit == 2) {
                    if (lit_comp < 128) return ZXC_ERROR_CORRUPT_DATA;
                    rc = pivco_decode(p_data, p_data + 128, lit_comp - 128, scratch, n_lit, hw, cum, cum_words, lane);
                } else {
                    rc = pivco_decode(dict_huf, p_data, lit_comp, scratch, n_lit, hw, cum, cum_words, lane);
                }
                if (rc != ZXC_OK) return rc;
                __syncwarp();
                S.lit = scratch;
                S.n_lit_avail = n_lit;
            } else {
                S.lit = p_data;
                S.n_lit_avail = 0;
            }
        } else if (enc_lit == 1) {
            if (n_lit > 0) {
                if (n_lit > cap) return ZXC_ERROR_DST_TOO_SMALL;
                if (n_lit > scratch_cap) return ZXC_ERROR_CORRUPT_DATA; /* lit_buffer_cap, :914 */
                if (lit_comp > avail) return ZXC_ERROR_CORRUPT_DATA;
                const int rc = rle_expand(p_data, lit_comp, scratch, n_lit, lane);
                if (rc != ZXC_OK) return rc;
                __syncwarp();
                S.lit = scratch;
                S.n_lit_avail = n_lit;
            } else {
                S.lit = p_data;
                S.n_lit_avail = 0;
            }
        } else if (enc_lit == 0) {
            S.lit = p_data;
            S.n_lit_avail = lit_comp;
        } else {
            return ZXC_ERROR_CORRUPT_DATA;
        }
        const u64 sz_off = enc_off ? (u64)n_seq : (u64)n_seq * 2;
        const u64 consumed = (u64)lit_comp + tok_comp + sz_off;
        if (consumed > avail) return ZXC_ERROR_CORRUPT_DATA;
        if (avail - lit_comp < 32) return ZXC_ERROR_CORRUPT_DATA;
        if (enc_tok != 0 && enc_tok != 2) return ZXC_ERROR_CORRUPT_DATA;
        S.tok = p_data + lit_comp;
        S.offs = S.tok + tok_comp;
        if (LEAN && S.lit == scratch) {
            /* RLE literals expanded into the scratch: the tokens and offsets are copied right behind them, short of the
             * escape-value table; a section that does not fit there (never a valid block) goes to the general instance */
            const u32 ts = tok_comp + (u32)sz_off;
            if ((u64)n_lit + ts > scratch_cap + scr_tok_cap(block_cap) + (u32)HUF_WORK_BYTES) return D2_DEFER_STATUS;
            warp_copy(scratch + n_lit, S.tok, ts, lane);
            __syncwarp();
            S.tok = scratch + n_lit;
        } else if (LEAN && S.n_lit_avail == 0) {
            S.lit = S.tok; /* RLE section that expands to nothing */
        }
        if (!LEAN && enc_tok == 2) { /* level 7: Huffman-coded tokens (:1019-1022) */
            /* the reference's token buffer holds block_cap / 5 + 16 sequences (zxc_cctx_max_seq) and its PivCo decoder
             * rejects an empty section; scr_tok_cap(block_cap) >= that + 32 */
            if (n_seq == 0 || n_seq > block_cap / 5u + 16u || tok_comp < 128) return ZXC_ERROR_CORRUPT_DATA;
            const int rc = pivco_decode(S.tok, S.tok + 128, tok_comp - 128, tok_buf, n_seq, hw, cum, cum_words, lane);
            if (rc != ZXC_OK) return rc;
            __syncwarp();
            S.tok = tok_buf;
        }
        S.ext = S.offs + (u32)sz_off;
        S.ext_end = avail - (u32)consumed;
    } else {
        if (enc_lit != 0 || enc_tok != 0) return ZXC_ERROR_CORRUPT_DATA;
        const u32 avail = comp - 12;
        const u64 consumed = (u64)n_lit + (u64)n_seq * 4;
        if (consumed > avail) return ZXC_ERROR_CORRUPT_DATA;
        if (avail - n_lit < 32) return ZXC_ERROR_CORRUPT_DATA;
        S.lit = pay + 12;
        S.n_lit_avail = n_lit;
        S.tok = S.lit + n_lit;
        S.ext = S.tok + (size_t)n_seq * 4;
        S.ext_end = avail - (u32)consumed;
    }
    return ZXC_OK;
}

#include "zxc_decode_units.cuh"

/* ------------------------------------------------------------------------- */
/* output window: ring (recent) + global (flushed) + dictionary (negative)    */
/* ------------------------------------------------------------------------- */
struct Window {
    u8* ring;        /* this warp's RING_BYTES of shared memory, 16-byte aligned */
    u8* out;         /* block output in global memory */
    const u8* dict;  /* dictionary content or NULL */
    u32 dict_size;
    i32 near_lo;     /* positions >= near_lo are valid in the ring */
};

__device__ __forceinline__ u8 window_byte(const Window& w, i32 pos) {
    if (pos >= w.near_lo) return w.ring[(u32)pos & (RING_BYTES - 1)];
    return pos >= 0 ? w.out[pos] : w.dict[(i32)w.dict_size + pos];
}
__device__ __forceinline__ u8 far_byte(const Window& w, i32 pos) {
    return pos >= 0 ? w.out[pos] : w.dict[(i32)w.dict_size + pos];
}

/* flush ring bytes [F, target) to global; 16-byte stores once (out + F) is 16-aligned */
__device__ __forceinline__ void ring_flush(const Window& w, u32& F, u32 target, u32 lane, bool al16) {
    const u32 mask = RING_BYTES - 1;
    if (target <= F) return; /* after a giant sequence F may sit above the 512-byte floor of O */
    if (al16) {
        const u32 head_end = min(target, (F + 15u) & ~15u);
        if (F < head_end) {
            const u32 p = F + lane;
            if (p < head_end) w.out[p] = w.ring[p & mask];
            F = head_end;
        }
#if ZXC_BULK_FLUSH
        /* every whole 16-byte unit by the bulk-copy engine: one or two copies (the ring wraps) issued by lane 0; the
         * warp's writes to the ring are ordered before them by the caller's __syncwarp() and the proxy fence.  The
         * copies complete under flush_wait(), which the caller runs before the ring is written or the flushed output
         * is read again. */
        const u32 nb = (target - F) & ~15u;
        if (nb) {
            if (lane == 0) {
                const u32 r = F & mask, first = min(nb, RING_BYTES - r);
                st_store_fence();
                st_store(w.out + F, smem_addr(w.ring) + r, first);
                if (first < nb) st_store(w.out + F + first, smem_addr(w.ring), nb - first);
                st_store_commit();
            }
            F += nb;
        }
#else
        while (target - F >= 512u) {
            const uint4 v = *reinterpret_cast<const uint4*>(w.ring + ((F + 16u * lane) & mask));
            *reinterpret_cast<uint4*>(w.out + F + 16u * lane) = v;
            F += 512u;
        }
        const u32 units = (target - F) >> 4;
        if (lane < units) {
            const uint4 v = *reinterpret_cast<const uint4*>(w.ring + ((F + 16u * lane) & mask));
            *reinterpret_cast<uint4*>(w.out + F + 16u * lane) = v;
        }
        F += units << 4;
#endif
    }
    for (u32 p = F + lane; p < target; p += 32) w.out[p] = w.ring[p & mask];
    F = target;
}

/* the bulk copies of ring_flush have read the ring and their output is visible to the warp */
__device__ __forceinline__ void flush_wait(u32 lane) {
#if ZXC_BULK_FLUSH
    if (lane == 0) st_store_wait();
    __syncwarp();
#else
    (void)lane;
#endif
}

/* whole-warp match copy of n bytes into the ring at d from distance off */
__device__ __forceinline__ void warp_match_to_ring(const Window& w, u32 d, u32 off, u32 n, u32 lane) {
    const u32 mask = RING_BYTES - 1;
    ZXC_STAT(16, d < off); /* byte copies that start in the dictionary */
    if (off >= 32) {
        /* chunk c only reads bytes below its own start: earlier chunks are complete */
        for (u32 c = 0; c < n; c += 32) {
            const u32 k = c + lane;
            if (k < n) w.ring[(d + k) & mask] = window_byte(w, (i32)(d + k) - (i32)off);
            __syncwarp();
        }
    } else {
        /* period-`off` replication of the complete window [d-off, d): lane r holds window byte r, byte k of the match
         * is window byte k mod off -- fetched by shuffle, the residue stepped by 32 mod off (no division per byte) */
        const u32 mine = lane < off ? (u32)window_byte(w, (i32)d - (i32)off + (i32)lane) : 0u;
        ZXC_STAT(15, 1); /* period replications */
#if ZXC_FASTMOD
        /* x mod off for x <= 32, off < 32 without the integer division: with a reciprocal good to a few ulp the float
         * quotient is at most one too small at exact multiples and never too large (between multiples the true quotient
         * keeps a margin of 1 / off from the next integer), so one subtraction repairs it */
        const float inv = __fdividef(1.0f, (float)off);
        u32 step = 32u - (u32)(32.0f * inv) * off;
        if (step >= off) step -= off;
        u32 r = lane - (u32)((float)lane * inv) * off;
        if (r >= off) r -= off;
#else
        const u32 step = 32u % off;
        u32 r = lane % off;
#endif
        for (u32 c = 0; c < n; c += 32) {
            const u32 b = __shfl_sync(FULL, mine, r);
            if (c + lane < n) w.ring[(d + c + lane) & mask] = (u8)b;
            r += step;
            if (r >= off) r -= off;
        }
    }
}

/* whole-warp match copy global -> global (giant sequences that bypass the ring) */
__device__ __forceinline__ void warp_match_global(const Window& w, u32 d, u32 off, u32 n, u32 lane) {
    if (off >= 32) {
        for (u32 c = 0; c < n; c += 32) {
            const u32 k = c + lane;
            if (k < n) w.out[d + k] = far_byte(w, (i32)(d + k) - (i32)off);
            __syncwarp();
        }
    } else {
        for (u32 k = lane; k < n; k += 32) w.out[d + k] = far_byte(w, (i32)d - (i32)off + (i32)(k % off));
    }
}

/* ------------------------------------------------------------------------- */
/* per-lane copy of n bytes (n <= 4*NWORDS - 4) into the ring, branch-free: the  */
/* NWORDS + 1 aligned source words that cover the item are loaded once, shifted  */
/* onto the destination grid in registers, and the partial words at either end   */
/* leave as byte / halfword stores of those registers (a neighbouring lane owns  */
/* the other bytes of such a word, so no read-modify-write).  `sp` is a generic   */
/* pointer (ring or global); the caller guarantees no ring wrap on either side;   */
/* reads up to 6 bytes before sp and 7 past sp + n.                               */
/* ------------------------------------------------------------------------- */
/* whole words K .. N-1 of a per-lane copy: word k is stored when k < kt (constant offsets, unrolled at compile time) */
template <int K, int N>
__device__ __forceinline__ void store_ladder(u32 d0, const u32* D, u32 kt) {
    if constexpr (K < N) {
        if ((u32)K < kt) sts32<4 * K>(d0, D[K]);
        store_ladder<K + 1, N>(d0, D, kt);
    }
}

template <int NWORDS>
__device__ __forceinline__ void lane_copy_words2(u32 ring_s, u32 dpos, const u8* sp, u32 n, bool on) {
    if (on) {
        const u32 da = dpos & 3u;
        const u32 e = da + n;              /* end of the item, in bytes from the start of destination word 0 */
        const u32 kt = e >> 2;             /* words below kt are whole (word 0 only if da == 0) ... */
        const u32 tb = e & 3u;             /* ... word kt holds the last tb bytes */
        const u8* bp = sp - da;
        const u32 m = (u32)(reinterpret_cast<uintptr_t>(bp)) & 3u;
        const u32* wp = reinterpret_cast<const u32*>(bp - m);
        const u32 sh = m * 8u;
        const u32 nsrc = kt + (tb ? 1u : 0u) + (m ? 1u : 0u);
        u32 W[NWORDS + 1];
#pragma unroll
        for (int k = 0; k <= NWORDS; k++) W[k] = (u32)k < nsrc ? wp[k] : 0u;
        u32 D[NWORDS];
#pragma unroll
        for (int k = 0; k < NWORDS; k++) D[k] = __funnelshift_r(W[k], W[k + 1], sh);
        const u32 d0 = ring_s + (dpos & (RING_BYTES - 1)) - da; /* destination word 0 */
        /* whole words */
        if (da == 0 && kt > 0) sts32<0>(d0, D[0]);
        store_ladder<1, NWORDS>(d0, D, kt);
        /* head of word 0: bytes [da, min(4, e)) when da != 0, as a byte mask */
        {
            const u32 e0 = e < 4u ? e : 4u;
            const u32 bm = da ? ((0xFu << da) & (0xFu >> (4u - e0))) : 0u;
            if (bm & 2u) sts8<1>(d0, D[0] >> 8);
            if ((bm & 0xCu) == 0xCu) sts16<2>(d0, D[0] >> 16);
            if ((bm & 0xCu) == 0x4u) sts8<2>(d0, D[0] >> 16);
            if ((bm & 0xCu) == 0x8u) sts8<3>(d0, D[0] >> 24);
        }
        /* tail: the first tb bytes of word kt (word 0 with da != 0 was the head's business) */
        {
            u32 tv = D[0];
#pragma unroll
            for (int k = 1; k < NWORDS; k++)
                if (kt == (u32)k) tv = D[k];
            const u32 tm = (kt > 0u || da == 0u) ? tb : 0u;
            const u32 dt = d0 + 4u * kt;
            if (tm == 1u) sts8<0>(dt, tv);
            if (tm >= 2u) sts16<0>(dt, tv);
            if (tm == 3u) sts8<2>(dt, tv >> 16);
        }
    }
}

/* ------------------------------------------------------------------------- */
/* long items of one pass, all at once: every aligned run of four                 */
/* whole destination words of every item is one lane's work, so a pass moves up   */
/* to 512 bytes per step and -- what matters -- pays ONE memory round trip per    */
/* step (round 1 moved 32 bytes of an item per round trip, four items at a time: */
/* its loop had to order each step's loads behind the previous step's stores),    */
/* and two thirds of the corpus' bytes sit in items longer than 64 bytes that     */
/* come from global memory.  Items of one call are mutually independent and do not overlap  */
/* themselves (distance >= length), so no chunk reads what another one writes;    */
/* the aligned words a chunk loads may reach 3 bytes into a neighbour's           */
/* destination, those bytes are shifted out.  Owners hold (dpos, source, n).      */
/* ------------------------------------------------------------------------- */
__device__ __forceinline__ void balanced_copy_words(u32 ring_s, u32 m_items, u32 my_d, const u8* my_sp, u32 my_n,
                                                    u32 lane) {
    const bool own = (m_items >> lane) & 1u;
    const u32 o_da = my_d & 3u;
    const u32 o_ff = o_da ? 1u : 0u;
    const u32 o_lfe = (o_da + my_n) >> 2;
    const u32 o_tb = (o_da + my_n) & 3u;
    const u32 o_dbyte = ring_s + (my_d & (RING_BYTES - 1));
    /* edge bytes by the owner: the head of destination word 0, the tail of word lfe (items here are > 20 bytes) */
    if (own && o_da) {
        sts8<0>(o_dbyte, my_sp[0]);
        if (o_da < 3) sts8<1>(o_dbyte, my_sp[1]);
        if (o_da < 2) sts8<2>(o_dbyte, my_sp[2]);
    }
    if (own && o_tb) {
        const u32 t0 = my_n - o_tb;
        sts8<0>(o_dbyte + t0, my_sp[t0]);
        if (o_tb > 1) sts8<1>(o_dbyte + t0, my_sp[t0 + 1]);
        if (o_tb > 2) sts8<2>(o_dbyte + t0, my_sp[t0 + 2]);
    }
    const u32 c = own ? (o_lfe - o_ff + 3u) >> 2 : 0u; /* chunks of four whole words */
    const u32 incl = warp_incl_scan(c, lane);
    const u32 total = __shfl_sync(FULL, incl, 31);
    const u32 excl = incl - c;
    const u32 pk = (my_d & (RING_BYTES - 1)) | (my_n << 16); /* ring offset < 64 Ki, n <= RING_LIMIT */
    const unsigned long long my_sp64 = reinterpret_cast<unsigned long long>(my_sp);
    for (u32 base = 0; base < total; base += 32) {
        ZXC_STAT(8, 1); /* balanced steps */
        const u32 q = base + lane;
        const bool act = q < total;
        u32 lo = 0, hi = 31; /* owner = first lane whose inclusive count exceeds q */
#pragma unroll
        for (int it = 0; it < 5; it++) {
            const u32 mid = (lo + hi) >> 1;
            const u32 v = __shfl_sync(FULL, incl, mid);
            if (v > q) hi = mid;
            else lo = mid + 1;
        }
        const u32 j = lo & 31u;
        const u32 k = q - __shfl_sync(FULL, excl, j);
        const u32 pj = __shfl_sync(FULL, pk, j);
        const u8* sp = reinterpret_cast<const u8*>(__shfl_sync(FULL, my_sp64, j));
        if (act) {
            const u32 da = pj & 3u;
            const u32 n = pj >> 16;
            const u32 lfe = (da + n) >> 2;
            const u32 w0 = (da ? 1u : 0u) + 4u * k;
            const u8* bp = sp - da;
            const u32 m = (u32)(reinterpret_cast<uintptr_t>(bp)) & 3u;
            const u32* wp = reinterpret_cast<const u32*>(bp - m) + w0;
            const u32 dw = ring_s + (pj & 0xFFFFu) - da + 4u * w0;
            const u32 sh = m * 8u;
            const u32 left = lfe - w0;            /* whole words from w0 on, >= 1 */
            const u32 nsrc = left + (m ? 1u : 0u);
            u32 W[5];
#pragma unroll
            for (int i = 0; i < 5; i++) W[i] = (u32)i < nsrc ? wp[i] : 0u;
            sts32<0>(dw, __funnelshift_r(W[0], W[1], sh));
            if (1 < left) sts32<4>(dw, __funnelshift_r(W[1], W[2], sh));
            if (2 < left) sts32<8>(dw, __funnelshift_r(W[2], W[3], sh));
            if (3 < left) sts32<12>(dw, __funnelshift_r(W[3], W[4], sh));
        }
    }
}

#ifndef ZXC_NW
#define ZXC_NW 8 /* destination words a per-lane copy may touch: items up to 4 * ZXC_NW - 4 bytes are "short" (6: -3.6 %, 10: +0.1 %) */
#endif
#define LIT_SHORT (4u * ZXC_NW - 4u)
#define MATCH_SHORT (4u * ZXC_NW - 4u)

/* ------------------------------------------------------------------------- */
/* GLO / GHI block body.  Returns decoded bytes or a negative zxc_error_t.    */
/* ------------------------------------------------------------------------- */
/* GHI and HAS_DICT are compile-time: the loop below sits at the kernel's register limit, and every branch and live
 * value it does not carry (the other block format's unpack, the dictionary pointer and its source classification)
 * is code the instruction cache does not hold and a register that is not spilled.  LEAN: see decode_job. */
/* the escape-value table: the rank-table area of a warp's scratch, idle once the sections are parsed */
__device__ __forceinline__ u32* esc_table(u8* scratch, u32 block_cap) {
    return reinterpret_cast<u32*>(scratch + scr_lit_cap(block_cap) + scr_tok_cap(block_cap) + (u32)HUF_WORK_BYTES);
}

/* LEAN look-ahead slot (slot_s: LA_SLOT_BYTES of shared memory behind the warp's ring).  Lane l copies slot word l --
 * a word of the aligned words that cover the tokens of the batch that starts at sequence nb for l < 12, of its
 * offsets above -- each with one 4-byte cp.async.  tk: the token section, the offsets right behind it.  The words lie
 * in the sections but for at most 3 bytes either side, which are inside the payload (or the scratch the RLE path
 * copied the sections to); nothing is copied when no batch follows. */
__device__ __forceinline__ void la_issue_words(u32 slot_s, const u8* tk, u32 n_seq, u32 enc_off, u32 nb, u32 lane) {
    if (nb < n_seq) {
        const u32 nt = min(32u, n_seq - nb), ow = enc_off ? 1u : 2u;
        const bool t = lane < LA_OFF / 4u;
        const u8* s = t ? tk + nb : tk + n_seq + ow * nb; /* the batch's first token / offset byte */
        const u32 n = t ? nt : ow * nt;
        const u32 x = (u32)reinterpret_cast<uintptr_t>(s) & 3u;
        const u32 k = t ? lane : lane - LA_OFF / 4u;
        if (4u * k < x + n) cp_async4(slot_s + 4u * lane, s - x + 4u * k);
    }
}
/* ... and escape value ob + l of the block's table, when there is one */
__device__ __forceinline__ void la_issue_esc(u32 slot_s, u32 n_val, u32 ob, u32 lane, const DecodeParams& P) {
    if (ob + lane < n_val)
        cp_async4(slot_s + LA_ESC + 4u * lane, esc_table(warp_scratch(P, grid_warp_now()), P.block_cap) + ob + lane);
}
/* escape value k of a batch whose first ordinal is ob: from the slot for the first 32, else from the table; 0 past
 * the last varint, as the reference reads (:51-88) */
__device__ __forceinline__ u32 la_esc(u32 slot_s, u32 k, u32 ob, u32 n_val, const DecodeParams& P) {
    if (k >= n_val) return 0u;
    if (k - ob < 32u) return lds32(slot_s + LA_ESC + 4u * (k - ob));
    return esc_table(warp_scratch(P, grid_warp_now()), P.block_cap)[k];
}

template <bool UNITS, bool GHI, bool HAS_DICT, bool LEAN>
__device__ int decode_lz_block(const u8* pay, u32 comp, u8* out, u32 cap, const u8* dict_in,
                               u32 dict_size_in, const u8* dict_huf, u8* scratch, u32 scratch_cap, u8* ring,
                               u32 lane, const DecodeParams& P) {
    constexpr bool ghi = GHI;
    const u8* dict = HAS_DICT ? dict_in : (const u8*)0;
    const u32 dict_size = HAS_DICT ? dict_size_in : 0u;
    ZXC_TRACE_DECL;
    ZXC_TRACE_ADD(TR_BLOCKS, 1, lane);
    Sections S;
    const int prc = parse_sections<LEAN>(pay, comp, ghi, cap, dict_huf, scratch, scratch_cap, lane, S);
    if (prc != ZXC_OK) return prc;
    const u8* lit = S.lit;
    const u8* tok = S.tok;
    const u8* offs = S.offs;
    const u8* ext = S.ext;
    const u32 ext_end = S.ext_end, n_lit_avail = S.n_lit_avail, n_seq = S.n_seq, enc_off = S.enc_off;

    /* Output-centric body (zxc_decode_units.cuh): only in the <UNITS = true> instance, which the launch picks on request
     * (ZXC_B200_UNITS=1); the sequence-centric body below is the faster one on every workload measured (DESIGN.md). */
    if (UNITS && cap <= 65536u) { /* its tables go where the scratch is idle */
        u8* tok_buf = scratch + scr_lit_cap(scratch_cap);
        u8* hw_area = tok_buf + scr_tok_cap(scratch_cap);
        const bool scratch_busy = (lit == scratch) || (tok == tok_buf);
        u8* tab = scratch_busy ? hw_area : scratch;
        const u32 tab_bytes = scratch_busy ? (u32)HUF_WORK_BYTES + scr_cum_cap(scratch_cap)
                                           : scr_stride(scratch_cap) - 256u;
        const int r = decode_lz_units(lit, n_lit_avail, tok, offs, ext, ext_end, n_seq, enc_off, ghi, out, cap, dict,
                                      dict_size, tab, tab_bytes, lane);
        if (r != UW_NOT_TAKEN) return r;
    }

    const u32 mask = RING_BYTES - 1;
    const u32 esc = ghi ? 255u : 15u;
    const u32 lt_mask = (1u << lane) - 1u;
    const bool al16 = (reinterpret_cast<uintptr_t>(out) & 15u) == 0;
    Window w;
    w.ring = ring;
    w.out = out;
    w.dict = dict;
    w.dict_size = dict_size;
    w.near_lo = 0;
    const u32 ring_s = smem_addr(ring);
    (void)ring_s;
    /* LEAN: the batch loop reads its tokens, offsets and first escape values from the look-ahead slot, where the
     * previous batch (or the block start) had them copied */
    constexpr bool LA = la_on<HAS_DICT, LEAN>();
    const u32 slot_s = ring_s + WARP_SMEM_BYTES;
    (void)slot_s;
    /* LEAN: the window's ring pointer is re-derived from ring_s in front of each rare path that uses it */
#define W_RING()                                     \
    do {                                             \
        if constexpr (LEAN) w.ring = ring_at(ring_s); \
    } while (0)
    u32 O = 0, L = 0, F = 0, epos = 0, ring_lo = 0;

    /* Escape values for the whole block up front (segment-map scan over the extras section, zxc_decode2_core.h):
     * a batch then reads its values by ordinal instead of walking the varint chain lane-uniformly.  The values
     * live in the rank-table area of the scratch, idle once the sections are parsed; a section too long for it
     * keeps the per-batch walk. */
    u32* vals = esc_table(scratch, scratch_cap);
    /* LEAN: an extras section too long for the table goes to the general instance (nothing is written yet), so the
     * batch loop below carries neither the varint cursor nor its walk; without extras every escape reads 0 from the
     * empty table, as the reference reads 0 past the section's end */
    if constexpr (LEAN) {
        if (4ull * ext_end > scr_cum_cap(scratch_cap)) return D2_DEFER_STATUS;
    }
    if constexpr (LA) { /* batch 0's tokens and offsets travel during the extras scan, its escape values after it */
        cp_async_check_idle();
        la_issue_words(slot_s, tok, n_seq, enc_off, 0u, lane);
    }
    const bool use_vals = LEAN || (ext_end != 0u && 4ull * ext_end <= scr_cum_cap(scratch_cap));
    u32 n_val = 0, ord_base = 0;
    if (use_vals && (!LEAN || ext_end != 0u)) {
        const u32 seg = max(4u, (ext_end + 31u) / 32u);
        const u32 nseg = (ext_end + seg - 1u) / seg;
        const u32 lo = lane * seg, hi = min(ext_end, lo + seg);
        u64 inc = lane < nseg ? z2_seg_map(ext, lo, hi, ext_end) : Z2_MAP_ID;
#pragma unroll
        for (int dd = 1; dd < 32; dd <<= 1) {
            const u64 o = __shfl_up_sync(FULL, inc, dd);
            if (lane >= (u32)dd) inc = z2_map_compose(o, inc);
        }
        u64 excl = __shfl_up_sync(FULL, inc, 1);
        if (lane == 0) excl = Z2_MAP_ID;
        n_val = z2_map_cnt(__shfl_sync(FULL, inc, 31), 0);
        if (lane < nseg) {
            const u32 ent = z2_map_exit(excl, 0);
            if (ent != 3u) z2_seg_values(ext, lo, hi, ext_end, ent, z2_map_cnt(excl, 0), vals);
        }
        __syncwarp();
    }
    if constexpr (LA) la_issue_esc(slot_s, n_val, 0u, lane, P);

#if ZXC_STAGE
    /* the token / offset sections (and raw literals) come through shared memory (zxc_decode_stage.cuh); Huffman-decoded
     * tokens and expanded literals sit in the scratch and are read from there */
    const u32 stage_s = smem_addr(ring) + RING_BYTES;
    TokStream::open(stage_s, tok, (ghi ? 4u : 1u) * n_seq, pay + comp, tok >= pay && tok < pay + comp);
    OffStream::open(stage_s, ghi ? tok : offs, ghi ? 0u : (enc_off ? 1u : 2u) * n_seq, pay + comp, !ghi);
#if ZXC_STAGE_LIT
    LitStream::open(stage_s, lit, n_lit_avail, pay + comp, lit >= pay && lit < pay + comp);
#define ST_LIT_CLOSE() LitStream::close(stage_s)
#else
#define ST_LIT_CLOSE() do { } while (0)
#endif
#define ST_CLOSE()                   \
    do {                             \
        TokStream::close(stage_s);   \
        OffStream::close(stage_s);   \
        ST_LIT_CLOSE();              \
    } while (0)
#else
#define ST_CLOSE() do { } while (0)
#define ST_LIT_CLOSE() do { } while (0)
#endif

    ZXC_TRACE_MARK(TR_START, lane);

    u32 base = 0;
    while (base < n_seq) {
        /* ---- unpack tokens and offsets ---- */
        const u32 i = base + lane;
        const bool valid = i < n_seq;
        u32 ll = 0, ml = 0, off = 1;
        /* LEAN without a dictionary: the first 512 bytes of literals from the cursor on (a batch reads 290 on the bench
         * corpus) are requested into L1 now, so that they arrive while the tokens and offsets do and the literal pass
         * finds them there; clamped to the literal section.  (With a dictionary both prefetches measured slower.) */
        if (LEAN && !HAS_DICT && lane < 4u && L + 128u * lane < n_lit_avail) prefetch_l1(lit + L + 128u * lane);
        if constexpr (LA) { /* a lane's wait covers its own copies; the warp reads every lane's */
            cp_async_wait_all();
            __syncwarp();
        }
#if ZXC_STAGE
        const u32 tok_w = ghi ? 4u : 1u, off_w = enc_off ? 1u : 2u;
        const u32 tx0 = (u32)(reinterpret_cast<uintptr_t>(tok) & 15u), ox0 = (u32)(reinterpret_cast<uintptr_t>(offs) & 15u);
        const u32 i_end = min(base + 32u, n_seq);
        const StWindow st_t = TokStream::need(stage_s, tok, tx0 + tok_w * base, tx0 + tok_w * i_end, 0u, lane);
        const StWindow st_o = OffStream::need(stage_s, offs, ox0 + off_w * base, ox0 + off_w * i_end, 0u, lane);
        const bool t_st = tx0 + tok_w * i_end <= st_t.hi, o_st = !ghi && ox0 + off_w * i_end <= st_o.hi;
#endif
        if (valid) {
            u32 a, b = 0;
#if ZXC_STAGE
            if (!ghi) {
                a = t_st ? lds8(st_t.ring_s + ((tx0 + i) & (ST_RING - 1u))) : (u32)tok[i];
                if (!o_st) {
                    b = enc_off ? (u32)offs[i] : ld16(offs + 2 * (size_t)i);
                } else if (enc_off) {
                    b = lds8(st_o.ring_s + ((ox0 + i) & (ST_RING - 1u)));
                } else {
                    const u32 x = ox0 + 2u * i;
                    b = (ox0 & 1u) ? (lds8(st_o.ring_s + (x & (ST_RING - 1u))) |
                                      (lds8(st_o.ring_s + ((x + 1u) & (ST_RING - 1u))) << 8))
                                   : lds16(st_o.ring_s + (x & (ST_RING - 1u)));
                }
            } else if (t_st) {
                const u32 x = tx0 + 4u * i;
                if (tx0 & 3u) {
                    a = lds8(st_t.ring_s + (x & (ST_RING - 1u))) | (lds8(st_t.ring_s + ((x + 1u) & (ST_RING - 1u))) << 8) |
                        (lds8(st_t.ring_s + ((x + 2u) & (ST_RING - 1u))) << 16) |
                        (lds8(st_t.ring_s + ((x + 3u) & (ST_RING - 1u))) << 24);
                } else {
                    a = lds32(st_t.ring_s + (x & (ST_RING - 1u)));
                }
            } else {
                a = ld32(tok + 4 * (size_t)i);
            }
#else
            if (!ghi) {
                /* LEAN: raw literals, raw tokens and offsets lie one behind the other in the payload, so the loop holds one
                 * pointer for all three and forms the others from it where they are read */
                const u8* tk = tok;
                if constexpr (LEAN) tk = lit + opaque(n_lit_avail);
                if constexpr (LA) {
                    /* the slot holds the aligned words from the one that holds the batch's first token (offset) on */
                    a = lds8(slot_s + ((u32)reinterpret_cast<uintptr_t>(tk + base) & 3u) + lane);
                    const u32 ox = (u32)reinterpret_cast<uintptr_t>(tk + n_seq + (enc_off ? base : 2u * base)) & 3u;
                    const u32 oa = slot_s + LA_OFF + ox + (enc_off ? lane : 2u * lane);
                    if (enc_off) b = lds8(oa);
                    else if (ox & 1u) b = lds8(oa) | (lds8(oa + 1u) << 8);
                    else b = lds16(oa);
                } else {
                    a = tk[i];
#if ZXC_ALIGNED_LD
                    if (LEAN) {
                        const u32 oi = n_seq + (enc_off ? i : 2u * i);
                        if (enc_off) b = (u32)tk[oi];
                        else if ((reinterpret_cast<uintptr_t>(tk) + n_seq) & 1u) b = ld16(tk + oi);
                        else b = (u32)*reinterpret_cast<const unsigned short*>(tk + oi);
                    } else if (enc_off) b = (u32)offs[i];
                    else if (reinterpret_cast<uintptr_t>(offs) & 1u) b = ld16(offs + 2 * (size_t)i);
                    else b = (u32)reinterpret_cast<const unsigned short*>(offs)[i];
#else
                    b = enc_off ? (u32)offs[i] : ld16(offs + 2 * (size_t)i);
#endif
                }
            } else {
#if ZXC_ALIGNED_LD
                a = (reinterpret_cast<uintptr_t>(tok) & 3u) ? ld32(tok + 4 * (size_t)i) : reinterpret_cast<const u32*>(tok)[i];
#else
                a = ld32(tok + 4 * (size_t)i);
#endif
            }
#endif
            if (!ghi) {
                ll = a >> 4;
                ml = a & 15;
                off = b + 1;
            } else {
                ll = a >> 24;
                ml = (a >> 16) & 0xFF;
                off = (a & 0xFFFF) + 1;
            }
        }
        /* ---- escapes: one uniform walk over the batch's varints ---- */
        const bool e_ll = valid && ll == esc, e_ml = valid && ml == esc;
        const u32 m_ll = __ballot_sync(FULL, e_ll), m_ml = __ballot_sync(FULL, e_ml);
        ZXC_TRACE_MARK(TR_UNPACK, lane);
        u32 k_esc = 0, epos_end = epos;
        if ((m_ll | m_ml) && use_vals) {
            /* LEAN: the table's address is formed here from the launch parameters, not held across the loop */
            const u32* vt = vals;
            if constexpr (LEAN) vt = esc_table(warp_scratch(P, grid_warp_now()), P.block_cap);
            u32 k = ord_base + __popc(m_ll & lt_mask) + __popc(m_ml & lt_mask);
            if constexpr (LA) { /* the table is read only for ordinals past the staged 32 */
                if (e_ll) {
                    ll += la_esc(slot_s, k, ord_base, n_val, P);
                    k++;
                }
                if (e_ml) ml += la_esc(slot_s, k, ord_base, n_val, P);
            } else {
                if (e_ll) {
                    ll += k < n_val ? vt[k] : 0u; /* past the last varint the reference reads 0 (:51-88) */
                    k++;
                }
                if (e_ml) ml += k < n_val ? vt[k] : 0u;
            }
        } else if (ZXC_RARE((m_ll | m_ml) != 0)) {
            const u32 ord_ll = __popc(m_ll & lt_mask) + __popc(m_ml & lt_mask);
            k_esc = __popc(m_ll) + __popc(m_ml);
            u32 my_pos = ext_end; /* cursor where this lane's first varint starts */
            for (u32 s = 0; s < k_esc; s++) {
                if (s == ord_ll) my_pos = epos_end;
                epos_end = varint_advance(ext, epos_end, ext_end);
            }
            if (e_ll) ll += read_varint(ext, my_pos, ext_end);
            if (e_ml) ml += read_varint(ext, my_pos, ext_end);
        }
        /* ---- prefix sums and fit ---- */
        if (valid) ml += 5;
        const u32 tot = ll + ml;
        const u32 s_ll = warp_incl_scan(ll, lane);
        const u32 s_tot = warp_incl_scan(tot, lane);

        /* ---- how many leading sequences fit the ring this round ---- */
        const u32 nvalid = min(32u, n_seq - base);
        const u32 m = __popc(__ballot_sync(FULL, valid && s_tot <= RING_LIMIT));
        const u32 lit_start = L + s_ll - ll;
        const u32 out_start = O + s_tot - tot;
        const u32 mdst = out_start + ll;

        if (ZXC_RARE(m == 0)) {
            /* ---- giant sequence (lane 0): bypass the ring, global -> global ---- */
            const u32 g_ll = __shfl_sync(FULL, ll, 0), g_ml = __shfl_sync(FULL, ml, 0),
                      g_off = __shfl_sync(FULL, off, 0);
            ZXC_STAT(9, 1); /* giant sequences */
            if (L + g_ll > n_lit_avail || (u64)O + g_ll + g_ml > cap) {
                ST_CLOSE();
                return ZXC_ERROR_OVERFLOW;
            }
            if (O + g_ll + dict_size < g_off) {
                ST_CLOSE();
                return ZXC_ERROR_BAD_OFFSET;
            }
            __syncwarp();
            W_RING();
            ring_flush(w, F, O, lane, al16);
            __syncwarp();
            flush_wait(lane);
            warp_copy(out + O, lit + L, g_ll, lane);
            __syncwarp();
            warp_match_global(w, O + g_ll, g_off, g_ml, lane);
            __syncwarp();
            O += g_ll + g_ml;
            L += g_ll;
            F = O;
            /* re-seed the ring with the last 64 bytes so short sources that straddle O resolve */
            ring_lo = O >= 64 ? O - 64 : 0;
            for (u32 p = ring_lo + lane; p < O; p += 32) w.ring[p & mask] = out[p];
            __syncwarp();
            const u32 q = ((m_ll & 1u) ? 1u : 0u) + ((m_ml & 1u) ? 1u : 0u);
            ord_base += q;
            if (!use_vals)
                for (u32 s = 0; s < q; s++) epos = varint_advance(ext, epos, ext_end); /* rare: re-walk */
            base += 1;
            if constexpr (LA) {
                la_issue_words(slot_s, lit + opaque(n_lit_avail), n_seq, enc_off, base, lane);
                la_issue_esc(slot_s, n_val, ord_base, lane, P);
            }
            ZXC_TRACE_MARK(TR_GIANT, lane);
            continue;
        }

        ZXC_STAT(10, m < nvalid);              /* partial batches */
        ZXC_STAT(11, m < nvalid && !use_vals); /* ... that re-walk the varint cursor */
        /* ---- validation ---- */
        const bool act = lane < m;
        const bool ovf = act && (lit_start + ll > n_lit_avail || out_start + tot > cap);
        const bool bad = act && (mdst + dict_size < off);
        const u32 m_err = __ballot_sync(FULL, ovf || bad);
        if (ZXC_RARE(m_err != 0)) {
            ZXC_STAT(19, 1); /* verdicts raised by a batch */
            const int code = ovf ? ZXC_ERROR_OVERFLOW : ZXC_ERROR_BAD_OFFSET;
            ST_CLOSE();
            return __shfl_sync(FULL, code, __ffs(m_err) - 1);
        }
        const u32 T = __shfl_sync(FULL, s_tot, m - 1), TL = __shfl_sync(FULL, s_ll, m - 1);
        if constexpr (LA) {
            /* the next batch starts at sequence base + m, with the escape ordinal after this batch's: its words are
             * copied into the slot while this batch copies (the slot's reads are behind the ballot above) */
            const u32 below = m < 32u ? (1u << m) - 1u : FULL;
            ord_base += __popc(m_ll & below) + __popc(m_ml & below);
            base += m;
            la_issue_words(slot_s, lit + opaque(n_lit_avail), n_seq, enc_off, base, lane);
            la_issue_esc(slot_s, n_val, ord_base, lane, P);
        }
#if ZXC_STAGE && ZXC_STAGE_LIT
        const u32 lx0 = (u32)(reinterpret_cast<uintptr_t>(lit) & 15u);
        const StWindow lw = LitStream::need(stage_s, lit, lx0 + L, lx0 + L + TL, 8u, lane);
#endif
        {
            const i32 a = (i32)(O + T) - (i32)RING_BYTES + 32;
            w.near_lo = a > (i32)ring_lo ? a : (i32)ring_lo;
        }

        flush_wait(lane); /* the previous flush has left the ring and reached the output */
        /* ---- copy passes: pass 0 = every literal run (independent of all matches), then match
         * rounds: a match is ready once its source ends below the lowest pending match destination.
         * One body serves all passes so the hot loop stays inside the instruction cache. ---- */
        /* ---- classify matches ---- */
        const i32 src_lo = (i32)mdst - (i32)off;
        const i32 src_end = min((i32)mdst, src_lo + (i32)ml);
        /* word copies need: no ring wrap on the destination, and a source that is entirely in the
         * ring (no wrap) or entirely flushed to global memory */
        const bool near = src_lo >= w.near_lo;
        const u32 si = (u32)src_lo & mask;
        /* a source that lies inside the dictionary, 8 bytes clear of either end (the aligned word loads reach that far),
         * is a global source like any other */
        const bool in_dict = src_lo + (i32)ml + 8 <= 0 && (i32)dict_size + src_lo >= 8;
        const bool m_word_ok = ((mdst & mask) + ml + 4 <= RING_BYTES) &&
                               (near ? (si >= 8 && si + ml + 8 <= RING_BYTES)
                                     : (in_dict || (src_lo >= 8 && src_lo + (i32)ml + 4 <= w.near_lo)));
        const bool m_lane_ok = m_word_ok && ml <= MATCH_SHORT && off >= ml;
        const bool m_grp_ok = m_word_ok && !m_lane_ok && off >= ml; /* chunks of one item run side by side */
        auto match_src = [&]() -> const u8* {
            return near ? (LEAN ? ring_at(ring_s + si) : ring + si)
                        : (src_lo < 0 ? dict + ((i32)dict_size + src_lo) : out + src_lo);
        };
        /* LEAN: the source pointer is formed in the match pass, so no 64-bit value of it lives through the literal pass */
        const u8* m_sp = LEAN ? nullptr : match_src();
        const bool l_word_ok = (out_start & mask) + ll + 4 <= RING_BYTES;

        /* ---- dependencies ---- */
        /* A match whose source ends at or below O -- the first output byte of this batch -- reads nothing the batch
         * writes: such matches (94 % of them on the bench corpus) go side by side in one pass after the literals.  The
         * others go one after the other in sequence order behind that pass, each copied by the whole warp (lane = byte):
         * sequential order is the reference's order, so no dependency analysis is needed, and a chain of 32 dependent
         * matches costs 32 short steps instead of 32 passes. */
        const bool m_free = src_end <= (i32)O;
        if (LEAN && !HAS_DICT && act && m_free && !near && src_lo >= 0) {
            /* LEAN without a dictionary: the first and last source line of every free match outside the ring, requested
             * into L1 now so that they arrive while the literal pass waits on its own loads and the match pass finds
             * them there instead of paying a second round trip.  Both lie in output already written (below O). */
            const u8* ps = out + src_lo;
            const u8* pe = ps + ml - 1u;
            prefetch_l1(ps);
            if ((reinterpret_cast<uintptr_t>(ps) ^ reinterpret_cast<uintptr_t>(pe)) >> 7) prefetch_l1(pe);
        }
        ZXC_TRACE_ADD(TR_M_RING, __popc(__ballot_sync(FULL, act && near)), lane);
        ZXC_TRACE_ADD(TR_M_GLOBAL, __popc(__ballot_sync(FULL, act && !near && src_lo >= 0)), lane);
        ZXC_TRACE_ADD(TR_M_DICT, __popc(__ballot_sync(FULL, act && !near && src_lo < 0)), lane);
        ZXC_TRACE_ADD(TR_M_SEQ, __popc(__ballot_sync(FULL, act && !m_free)), lane);
        ZXC_TRACE_ADD(TR_BATCHES, 1, lane);
        ZXC_TRACE_MARK(TR_SCAN, lane);
        /* ---- pass loop ---- */
        ZXC_STAT(0, 1);            /* batches */
        ZXC_STAT(1, m);            /* sequences */
        bool lit_pass = true;
#pragma unroll 1
        for (;;) {
            bool ready, lok, gok;
            u32 it_d, it_n;
            const u8* it_sp;
            if (lit_pass) {
                ready = act && ll > 0;
                it_d = out_start;
                it_n = ll;
                it_sp = lit + lit_start;
#if ZXC_STAGE && ZXC_STAGE_LIT
                {
                    const u8* sp_s = lit_ptr(lw, lx0 + lit_start, ll);
                    if (sp_s) it_sp = sp_s;
                    ZXC_STAT(13, __popc(__ballot_sync(FULL, ready && sp_s != 0))); /* literal runs read from the ring */
                    ZXC_STAT(14, __popc(__ballot_sync(FULL, ready)));
                }
#endif
                lok = l_word_ok && ll <= LIT_SHORT;
                gok = l_word_ok && ll > LIT_SHORT;
            } else {
                ready = act && m_free;
                it_d = mdst;
                it_n = ml;
                it_sp = LEAN ? match_src() : m_sp;
                lok = m_lane_ok;
                gok = m_grp_ok;
            }
            lane_copy_words2<ZXC_NW>(ring_s, it_d, it_sp, it_n, ready && lok);
            const u32 m_grp = __ballot_sync(FULL, ready && gok);
            ZXC_STAT(2, 1);                                           /* passes */
            ZXC_STAT(3, __popc(__ballot_sync(FULL, ready && lok)));   /* per-lane items */
            ZXC_STAT(4, __popc(m_grp));                               /* long items */
            ZXC_STAT(5, m_grp != 0);                                  /* long-copy calls */
            ZXC_STAT(6, __popc(__ballot_sync(FULL, ready && !lok && !gok))); /* slow items */
            ZXC_STAT(7, __ballot_sync(FULL, ready && lok) != 0);      /* passes with a per-lane item */
            ZXC_STAT(17, __popc(__ballot_sync(FULL, !lit_pass && ready && (lok || gok) && src_lo < 0)));  /* dictionary words */
            ZXC_STAT(18, __popc(__ballot_sync(FULL, !lit_pass && ready && !lok && !gok)));  /* match byte path */
            ZXC_STAT(20, __popc(__ballot_sync(FULL, !lit_pass && ready && (lok || gok) && near))); /* ring words */
            ZXC_STAT(21, __popc(__ballot_sync(FULL, !lit_pass && ready && (lok || gok) && !near && src_lo >= 0))); /* global words */
            if (m_grp) balanced_copy_words(ring_s, m_grp, it_d, it_sp, it_n, lane);
            u32 m_slow = __ballot_sync(FULL, ready && !lok && !gok);
            while (ZXC_RARE(m_slow != 0)) { /* ring wrap, close overlap, dictionary, straddling sources: byte paths */
                const int j = __ffs(m_slow) - 1;
                m_slow &= m_slow - 1;
                const u32 d = __shfl_sync(FULL, it_d, j), n = __shfl_sync(FULL, it_n, j);
                const u32 aux = __shfl_sync(FULL, lit_pass ? lit_start : off, j);
                W_RING();
                if (lit_pass) {
                    for (u32 k = lane; k < n; k += 32) w.ring[(d + k) & mask] = lit[aux + k];
                } else {
                    warp_match_to_ring(w, d, aux, n, lane);
                }
            }
            __syncwarp();
            ZXC_TRACE_MARK(lit_pass ? TR_LIT : TR_MATCH, lane);
            if (!lit_pass) break;
            lit_pass = false;
        }
        {
            u32 rest = __ballot_sync(FULL, act && !m_free);
            const u32 my_pk = ml | ((near && off >= ml) ? 0x80000000u : 0u);
            ZXC_STAT(12, __popc(rest)); /* matches that go in sequence order */
            while (rest) {
                const int j = __ffs(rest) - 1;
                rest &= rest - 1;
                const u32 d = __shfl_sync(FULL, mdst, j), pk = __shfl_sync(FULL, my_pk, j);
                const u32 n = pk & 0x7FFFFFFFu;
                if (pk >> 31) { /* the whole source is in the ring and the match does not overlap itself */
                    const u32 sl = __shfl_sync(FULL, (u32)src_lo, j);
#if ZXC_TAIL_SMEM
                    for (u32 k = lane; k < n; k += 32) sts8<0>(ring_s + ((d + k) & mask), lds8(ring_s + ((sl + k) & mask)));
#else
                    for (u32 k = lane; k < n; k += 32) ring[(d + k) & mask] = ring[(sl + k) & mask];
#endif
                } else {
                    W_RING();
                    warp_match_to_ring(w, d, __shfl_sync(FULL, off, j), n, lane);
                }
                __syncwarp();
            }
        }
        ZXC_TRACE_MARK(TR_TAIL, lane);

        /* ---- advance and flush ---- */
        O += T;
        L += TL;
        W_RING();
        ring_flush(w, F, O & ~511u, lane, al16);
        __syncwarp();
        ZXC_TRACE_MARK(TR_FLUSH, lane);

        if constexpr (LA) {
            /* advanced where the next batch's copies were issued */
        } else if (m < nvalid) {
            const u32 below = (1u << m) - 1u;
            const u32 q = __popc(m_ll & below) + __popc(m_ml & below);
            ord_base += q;
            if (!use_vals)
                for (u32 s = 0; s < q; s++) epos = varint_advance(ext, epos, ext_end); /* rare: re-walk */
            base += m;
        } else {
            ord_base += __popc(m_ll) + __popc(m_ml);
            epos = epos_end;
            base += 32;
        }
    }
    if constexpr (LA) cp_async_wait_all(); /* the copies issued for the batch after the last one land before the block ends */

    /* trailing literals (zxc_decompress.c:1198-1206) */
    ST_LIT_CLOSE();
    const u32 rem = n_lit_avail - L;
    if (rem > cap - O) return ZXC_ERROR_OVERFLOW;
    W_RING();
#undef W_RING
    ring_flush(w, F, O, lane, al16);
    __syncwarp();
    flush_wait(lane);
    warp_copy(out + O, lit + L, rem, lane);
    ZXC_TRACE_MARK(TR_END, lane);
    return (int)(O + rem);
}

/* zxc_decompress_chunk_wrapper_body (zxc_decompress.c:1646-1695) for one job.
 * LEAN: decode only what the bench-shaped frames are made of -- RAW blocks and GLO blocks with raw tokens and raw or
 * RLE literals, in a launch without checksum verification -- and return D2_DEFER_STATUS for every other job, before
 * anything is written to its output; the general instance decodes those.  The lean instance carries neither the PivCo
 * Huffman decoder, the checksum nor the GHI body (DESIGN.md section 3d). */
template <bool UNITS, bool HAS_DICT, bool LEAN = false>
__device__ int decode_job(const DecodeParams& P, const zxc_b200_job_t& job, u8* scratch, u8* ring, u32 lane) {
    const u8* blk = P.src + job.src_off;
    u8* out = P.dst + job.dst_off;
    if (job.src_len < 8) return LEAN ? D2_DEFER_STATUS : ZXC_ERROR_SRC_TOO_SMALL;
    const u32 type = blk[0];
    const u32 comp = ld32(blk + 3);
    const bool verify = (P.flags & FLAG_VERIFY) != 0;
    if (LEAN) {
        /* the 8-byte block header and, for GLO, bytes 8 (enc_lit) and 9 (enc_tok) of the 12-byte section header */
        const bool whole = !verify && (u64)job.src_len >= 8ull + comp;
        const bool take = whole && (type == BT_RAW || (type == BT_GLO && comp >= 12u && blk[8 + 9] == 0 && blk[8 + 8] <= 1));
        if (!take) return D2_DEFER_STATUS;
    }
    if ((u64)job.src_len < 8ull + comp + (verify ? 4u : 0u)) return ZXC_ERROR_SRC_TOO_SMALL;
    const u8* data = blk + 8;
    if constexpr (!LEAN) {
        if (verify && ld32(data + comp) != warp_checksum(data, comp, lane)) return ZXC_ERROR_BAD_CHECKSUM;
    }
    switch (type) {
        case BT_GLO:
            return decode_lz_block<UNITS, false, HAS_DICT, LEAN>(data, comp, out, job.dst_cap, P.dict, P.dict_size,
                                                                 P.dict_huf, scratch, P.block_cap, ring, lane, P);
        case BT_GHI:
            if constexpr (LEAN) return D2_DEFER_STATUS; /* not reached: deferred above */
            else return decode_lz_block<UNITS, true, HAS_DICT, false>(data, comp, out, job.dst_cap, P.dict, P.dict_size,
                                                                      P.dict_huf, scratch, P.block_cap, ring, lane, P);
        case BT_RAW:
            if (comp > job.dst_cap) return ZXC_ERROR_DST_TOO_SMALL;
            warp_copy(out, data, comp, lane);
            return (int)comp;
        case BT_EOF:
            return ZXC_ERROR_CORRUPT_DATA;
        default:
            return ZXC_ERROR_BAD_BLOCK_TYPE;
    }
}

/* LEAN: decode_job<LEAN>; each job it defers is marked D2_DEFER_STATUS and listed for a DEFERRED launch that follows.
 * The lean instance has its own CTAs per SM (LEAN_CTAS_PER_SM): 8 against the general one's 7, in 64 registers without
 * spills: it holds no 64-bit ring or token pointer across its loops (ring_at, opaque; DESIGN.md section 9). */
template <bool UNITS, bool DEFERRED, bool HAS_DICT, bool LEAN>
__global__ void __launch_bounds__(CTA_THREADS, LEAN ? LEAN_CTAS_PER_SM : CTAS_PER_SM) zxc_decode_kernel(const DecodeParams P) {
    extern __shared__ __align__(16) u8 smem[];
    const u32 lane = threadIdx.x & 31;
    const u32 wic = threadIdx.x >> 5;
    const u32 gwarp = blockIdx.x * WARPS_PER_CTA + wic;
    u8* scratch = warp_scratch(P, gwarp);
    u8* ring = smem + (size_t)wic * (la_on<HAS_DICT, LEAN>() ? LEAN_WARP_SMEM_BYTES : WARP_SMEM_BYTES); /* the slot behind */
#if ZXC_STAGE
    st_init(smem_addr(ring) + RING_BYTES, lane);
#endif
    if (DEFERRED) {
        const u32 n_def = *P.defer_count;
        if (n_def == 0) return;
        if (n_def <= P.defer_cap) { /* the listed jobs, one per claim */
            for (;;) {
                unsigned long long k = 0;
                if (lane == 0) k = atomicAdd(P.counter, 1ull);
                k = __shfl_sync(FULL, k, 0);
                if (k >= n_def) break;
                const u32 j = P.defer_list[k];
                const zxc_b200_job_t job = P.jobs[j];
                const int r = decode_job<UNITS, HAS_DICT, false>(P, job, scratch, ring, lane);
                flush_wait(lane); /* nothing of this block is still on its way out of the ring */
                __syncwarp();
                if (lane == 0) P.status[j] = r;
            }
            return;
        }
        /* list overflow: 32 status words per claim, the warp decodes the jobs still marked deferred */
        for (;;) {
            unsigned long long b = 0;
            if (lane == 0) b = atomicAdd(P.counter, 32ull);
            b = __shfl_sync(FULL, b, 0);
            if (b >= P.n_jobs) break;
            const unsigned long long jj = b + lane;
            u32 m = __ballot_sync(FULL, jj < P.n_jobs && P.status[jj] == D2_DEFER_STATUS);
            while (m) {
                const unsigned long long j = b + (u32)(__ffs(m) - 1);
                m &= m - 1;
                const zxc_b200_job_t job = P.jobs[j];
                const int r = decode_job<UNITS, HAS_DICT, false>(P, job, scratch, ring, lane);
                flush_wait(lane); /* nothing of this block is still on its way out of the ring */
                __syncwarp();
                if (lane == 0) P.status[j] = r;
            }
        }
        return;
    }
    /* LEAN: the job index in one register (claims end below n_jobs plus one per warp, far below 2^32 for any job table
     * that fits in device memory), the ring as its shared address */
    using JobIx = typename std::conditional<LEAN, u32, unsigned long long>::type;
    u32 ring_s = 0;
    if constexpr (LEAN) ring_s = smem_addr(ring);
    for (;;) {
        ZXC_TRACE_DECL;
        unsigned long long c = 0;
        if (lane == 0) c = atomicAdd(P.counter, 1ull);
        const JobIx j = __shfl_sync(FULL, (JobIx)c, 0);
        ZXC_TRACE_MARK(TR_CLAIM, lane);
        if (j >= P.n_jobs) break;
        const zxc_b200_job_t job = P.jobs[j];
        const int r = LEAN ? decode_job<UNITS, HAS_DICT, LEAN>(P, job, warp_scratch(P, grid_warp_now()), ring_at(ring_s), lane)
                           : decode_job<UNITS, HAS_DICT, LEAN>(P, job, scratch, ring, lane);
        flush_wait(lane); /* nothing of this block is still on its way out of the ring */
        __syncwarp();
        if (lane == 0) {
            P.status[j] = r;
            if (LEAN && r == D2_DEFER_STATUS) {
                const u32 slot = atomicAdd(P.defer_count, 1u);
                if (slot < P.defer_cap) P.defer_list[slot] = (u32)j;
            }
        }
    }
}

/* status reduce: first job whose result differs from its dst_cap */
__global__ void zxc_reduce_kernel(const i32* status, const zxc_b200_job_t* jobs, u32 n,
                                  unsigned long long* out /* [0]=first bad idx, [1]=sum */) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long bad = ~0ull, sum = 0;
    if (i < n) {
        const i32 s = status[i];
        if (s < 0 || (u32)s != jobs[i].dst_cap) bad = i;
        else sum = (u32)s;
    }
    for (int d = 16; d >= 1; d >>= 1) {
        const unsigned long long ob = __shfl_xor_sync(FULL, bad, d);
        bad = ob < bad ? ob : bad;
        sum += __shfl_xor_sync(FULL, sum, d);
    }
    if ((threadIdx.x & 31) == 0) {
        if (bad != ~0ull) atomicMin(&out[0], bad);
        if (sum) atomicAdd(&out[1], sum);
    }
}
