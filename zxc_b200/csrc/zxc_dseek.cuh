/*
 * zxc_dseek.cuh -- random access into a seekable frame in HBM (zxc_b200_seekable_device_decompress_ranges): a batch
 * of byte ranges planned, decoded and judged on the device, on the caller's stream.  Stream order:
 *
 *   zxc_dseek_tiles    per range: checks 1-5 of zxc_seekable_decompress_range, its block span, how many blocks it
 *                      covers whole (direct jobs) and in part (slot jobs, at most 2); the counts' scan within tiles of
 *                      ASM_TILE ranges and the tile sums
 *   zxc_dseek_scan     one CTA: the tile sums' scan, the first range whose direct jobs overflow the job table (it and
 *                      every later range get ZXC_ERROR_MEMORY), the real job counts and both decodes' work counters
 *   zxc_dseek_emit     one warp per range: its direct jobs (in place in d_dst) and slot jobs (into the slot area), both
 *                      tables right-aligned behind zeroed status words, as zxc_dplan_place does
 *   zxc_decode_kernel  (zxc_decode.cuh, unchanged) launch_decode(preset = 1) on the direct table, then on the slot table
 *   zxc_dseek_finish   one CTA per range: first failing block in block order (first_failure's rule), the slots'
 *                      sub-ranges into d_dst with 16-byte stores, and the range's result
 *
 * The frame's block table (comp_offsets, num_blocks + 1 entries) was uploaded once when the handle was opened; every
 * launch sequence is the same whatever the ranges hold.
 *
 * A frame in page-locked host memory (zxc_b200_seekable_device_open_host) takes the _host instances of the three plan
 * kernels and one more launch.  Each admitted range stages one span, the on-disk bytes of its blocks b0 .. b1, which
 * are contiguous in the frame:
 *
 *   zxc_dseek_tiles_host  also the span's staged size, scanned as a third quantity: the span at an offset congruent to
 *                         its host address mod 16, then DS_STAGE_PAD readable bytes, rounded up to 16
 *   zxc_dseek_scan_host   also the staged bytes' scan and the admitted ranges' staged total
 *   zxc_dseek_emit_host   job sources as staging offsets
 *   zxc_dseek_fetch       the admitted spans from mapped host memory into the staging area, as aligned 16-byte loads
 *                         over PCIe; then the decodes run on the staging area as they run on an HBM frame
 */
#pragma once
#include <cuda_runtime.h>

#include "zxc_assemble.cuh"
#include "zxc_b200.h"
#include "zxc_error.h"

#define DS_THREADS 256

/* the first bytes of the caller's scratch */
struct DSeekState {
    unsigned long long ctr[2][4]; /* the direct and the slot decode's work counters (launch_decode) */
    unsigned long long first_over; /* first range whose direct jobs do not fit the table (n_ranges: none) */
    unsigned long long d_real;     /* direct jobs of the ranges in front of it */
    unsigned long long s_real;     /* slot jobs of those ranges */
    unsigned long long p_real;     /* staged bytes of those ranges (a frame in host memory) */
};
#define DS_STATE_BYTES 256
static_assert(sizeof(DSeekState) <= DS_STATE_BYTES, "DSeekState fits its region");

/* zxc_dseek_tiles' record per range */
struct DSeekRec {
    unsigned long long ex_d; /* direct jobs of the tile's earlier ranges */
    unsigned int ex_s;       /* slot jobs of the tile's earlier ranges */
    int v;                   /* 1: to decode; else the range's result (0 or a check 1-5 code) */
    unsigned int nd, ns;     /* its direct and slot jobs */
    union {
        unsigned int pad[2];
        unsigned long long ex_p; /* staged bytes of the tile's earlier ranges (a frame in host memory) */
    };
};

struct DSeekArgs {
    const unsigned long long* offs; /* the handle's comp_offsets */
    const zxc_b200_range_t* ranges;
    u8* dst;
    u8* slots; /* 2 * n slots of slot_stride bytes */
    long long* results;
    DSeekState* st;
    DSeekRec* recs;
    unsigned long long* tiles; /* per tile: direct sum, slot sum; the scan turns them into exclusive prefixes */
    zxc_b200_job_t* djobs;     /* J entries */
    i32* dstatus;
    zxc_b200_job_t* sjobs; /* 2 * n entries */
    i32* sstatus;
    unsigned long long total, dst_capacity;
    unsigned int n, J, block_size, slot_stride;
    unsigned int need_dict; /* the frame names a dictionary and none is set */
    /* a frame in host memory (the _host instances and zxc_dseek_fetch) */
    const u8* hsrc;             /* the frame, at the device address of its page-locked host memory */
    u8* stage;                  /* the staging area, 16-byte aligned */
    unsigned long long* ptiles; /* per tile: staged bytes; the scan turns them into exclusive prefixes */
    unsigned long long src_size;
};

/* readable bytes behind each staged span: the decode kernels read up to 8 bytes past a block */
#define DS_STAGE_PAD 8u

/* expected_block_bytes */
__device__ __forceinline__ u32 ds_expected(const DSeekArgs& A, u64 b) {
    const u64 start = b * A.block_size;
    return A.total - start >= A.block_size ? A.block_size : (u32)(A.total - start);
}

/* a range's block span and which of its end blocks it covers only in part */
struct DSeekSpan {
    u64 b0, b1, lo; /* first and last block; lo = first direct block */
    u32 head, tail; /* b0 (head) / b1 (tail) decodes into a slot */
};
__device__ __forceinline__ DSeekSpan ds_span(const DSeekArgs& A, u64 offset, u64 len) {
    DSeekSpan s;
    const u64 bs = A.block_size, end = offset + len;
    s.b0 = offset / bs;
    s.b1 = (end - 1) / bs;
    s.head = offset != s.b0 * bs || end < s.b0 * bs + ds_expected(A, s.b0);
    s.tail = s.b1 != s.b0 && end < s.b1 * bs + ds_expected(A, s.b1);
    s.lo = s.b0 + s.head;
    return s;
}

/* checks 1-5 of zxc_seekable_decompress_range, in its order */
__device__ __forceinline__ int ds_check(const DSeekArgs& A, const zxc_b200_range_t& r) {
    if (r.len == 0) return 0;
    if (!A.dst) return ZXC_ERROR_NULL_INPUT;
    const u64 cap = r.dst_off > A.dst_capacity ? 0 : A.dst_capacity - r.dst_off;
    if (cap < r.len) return ZXC_ERROR_DST_TOO_SMALL;
    if (r.offset + r.len > A.total || r.offset + r.len < r.offset) return ZXC_ERROR_SRC_TOO_SMALL;
    if (A.need_dict) return ZXC_ERROR_DICT_REQUIRED;
    return 1;
}

/* where a staged span starts: the span [offs[b0], offs[b1 + 1]) of the frame at an offset congruent to its host address
 * mod 16, so that every copy of zxc_dseek_fetch is an aligned 16-byte copy */
__device__ __forceinline__ u32 ds_stage_skew(const DSeekArgs& A, u64 off) { return (u32)((uintptr_t)(A.hsrc + off) & 15u); }

/* a range's staged bytes: its span's skew, the span, DS_STAGE_PAD, rounded up to 16 */
__device__ __forceinline__ u64 ds_stage_bytes(const DSeekArgs& A, const DSeekSpan& s) {
    const u64 o0 = A.offs[s.b0], o1 = A.offs[s.b1 + 1];
    return (ds_stage_skew(A, o0) + (o1 - o0) + DS_STAGE_PAD + 15u) & ~(u64)15;
}

template <bool HOST>
__device__ __forceinline__ void ds_tiles(const DSeekArgs& A) {
    const u64 base = (u64)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    u32 nd[ASM_ITEMS], ns[ASM_ITEMS];
    int v[ASM_ITEMS];
    u64 np[ASM_ITEMS];
    u64 sd = 0, ss = 0, sp = 0;
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        nd[k] = ns[k] = 0;
        np[k] = 0;
        v[k] = 0;
        if (base + k < A.n) {
            const zxc_b200_range_t r = A.ranges[base + k];
            v[k] = ds_check(A, r);
            if (v[k] == 1) {
                const DSeekSpan s = ds_span(A, r.offset, r.len);
                nd[k] = (u32)(s.b1 + 1 - s.tail - s.lo);
                ns[k] = s.head + s.tail;
                if constexpr (HOST) np[k] = ds_stage_bytes(A, s);
            }
        }
        sd += nd[k];
        ss += ns[k];
        sp += np[k];
    }
    unsigned long long td, ts, tp = 0;
    u64 ed = asm_cta_excl(sd, &td);
    u64 es = asm_cta_excl(ss, &ts);
    u64 ep = 0;
    if constexpr (HOST) ep = asm_cta_excl(sp, &tp);
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        if (base + k < A.n) {
            DSeekRec R;
            R.ex_d = ed;
            R.ex_s = (u32)es;
            R.v = v[k];
            R.nd = nd[k];
            R.ns = ns[k];
            if constexpr (HOST) R.ex_p = ep;
            else R.pad[0] = R.pad[1] = 0;
            A.recs[base + k] = R;
        }
        ed += nd[k];
        es += ns[k];
        ep += np[k];
    }
    if (threadIdx.x == 0) {
        A.tiles[2 * blockIdx.x] = td;
        A.tiles[2 * blockIdx.x + 1] = ts;
        if constexpr (HOST) A.ptiles[blockIdx.x] = tp;
    }
}

__global__ void __launch_bounds__(ASM_THREADS) zxc_dseek_tiles(const DSeekArgs A) { ds_tiles<false>(A); }
/* the staged sizes take 16 more registers than 64 hold; a grid of one CTA per 2 048 ranges needs no occupancy */
__global__ void __launch_bounds__(ASM_THREADS, 1) zxc_dseek_tiles_host(const DSeekArgs A) { ds_tiles<true>(A); }

template <bool HOST>
__device__ __forceinline__ void ds_scan(const DSeekArgs& A) {
    __shared__ unsigned long long s_tile, s_first;
    DSeekState* S = A.st;
    const u32 n_tiles = (A.n + ASM_TILE - 1) / ASM_TILE;
    if (threadIdx.x == 0) s_tile = s_first = ~0ull;
    unsigned long long cd = 0, cs = 0, cp = 0;
    for (u32 b = 0; b < n_tiles; b += blockDim.x) {
        const u32 i = b + threadIdx.x;
        const unsigned long long vd = i < n_tiles ? A.tiles[2 * i] : 0, vs = i < n_tiles ? A.tiles[2 * i + 1] : 0;
        unsigned long long td, ts;
        const unsigned long long ed = cd + asm_cta_excl(vd, &td); /* its barriers also order s_tile */
        const unsigned long long es = cs + asm_cta_excl(vs, &ts);
        if constexpr (HOST) {
            const unsigned long long vp = i < n_tiles ? A.ptiles[i] : 0;
            unsigned long long tp;
            const unsigned long long ep = cp + asm_cta_excl(vp, &tp);
            if (i < n_tiles) A.ptiles[i] = ep;
            cp += tp;
        }
        if (i < n_tiles) {
            A.tiles[2 * i] = ed;
            A.tiles[2 * i + 1] = es;
            if (ed + vd > A.J) atomicMin(&s_tile, (unsigned long long)i);
        }
        cd += td;
        cs += ts;
    }
    __syncthreads();
    const u64 t = s_tile;
    if (t != ~0ull) { /* the first range of that tile whose direct jobs end past J */
        for (u64 i = t * ASM_TILE + threadIdx.x; i < A.n && i < (t + 1) * ASM_TILE; i += blockDim.x) {
            const DSeekRec R = A.recs[i];
            if (R.nd && A.tiles[2 * t] + R.ex_d + R.nd > A.J) atomicMin(&s_first, i);
        }
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    u64 f = A.n, d_real = cd, s_real = cs;
    if (t != ~0ull) {
        f = s_first;
        const DSeekRec R = A.recs[f];
        d_real = A.tiles[2 * t] + R.ex_d;
        s_real = A.tiles[2 * t + 1] + R.ex_s;
        if constexpr (HOST) cp = A.ptiles[t] + R.ex_p;
    }
    S->first_over = f;
    S->d_real = d_real;
    S->s_real = s_real;
    if constexpr (HOST) S->p_real = cp;
    /* counter 0 claims job indices from the first real job; counters 1 and 2 as in zxc_dplan_place */
    S->ctr[0][0] = A.J - d_real;
    S->ctr[1][0] = 2ull * A.n - s_real;
    S->ctr[0][1] = S->ctr[0][2] = S->ctr[1][1] = S->ctr[1][2] = 0;
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dseek_scan(const DSeekArgs A) { ds_scan<false>(A); }
__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dseek_scan_host(const DSeekArgs A) { ds_scan<true>(A); }

/* a staged range's first span byte in the staging area */
__device__ __forceinline__ u64 ds_stage_pos(const DSeekArgs& A, u64 i, const DSeekRec& R, const DSeekSpan& s) {
    return A.ptiles[i / ASM_TILE] + R.ex_p + ds_stage_skew(A, A.offs[s.b0]);
}

template <bool HOST>
__device__ __forceinline__ void ds_emit(const DSeekArgs& A) {
    const DSeekState* S = A.st;
    const u64 f = S->first_over, d_real = S->d_real, s_real = S->s_real;
    const u64 d_lead = A.J - d_real, s_lead = 2ull * A.n - s_real;
    const u64 tid = (u64)blockIdx.x * DS_THREADS + threadIdx.x, nthreads = (u64)gridDim.x * DS_THREADS;
    /* no stale deferral marks in front of the real jobs (the deferred launch may scan the status words from 0) */
    for (u64 k = tid; k < d_lead; k += nthreads) A.dstatus[k] = 0;
    for (u64 k = tid; k < s_lead; k += nthreads) A.sstatus[k] = 0;
    const u64 i = tid >> 5;
    const u32 lane = threadIdx.x & 31;
    if (i >= A.n || i >= f) return;
    const DSeekRec R = A.recs[i];
    if (R.v != 1) return;
    const zxc_b200_range_t r = A.ranges[i];
    const DSeekSpan s = ds_span(A, r.offset, r.len);
    const u64 t = i / ASM_TILE;
    const u64 pd = d_lead + A.tiles[2 * t] + R.ex_d;
    const u64 ps = s_lead + A.tiles[2 * t + 1] + R.ex_s;
    const u64 bs = A.block_size;
    /* a frame in HBM is read where it lies; a frame in host memory from the range's staged span */
    u64 rebase = 0;
    if constexpr (HOST) rebase = ds_stage_pos(A, i, R, s) - A.offs[s.b0];
    for (u32 k = lane; k < R.nd; k += 32) {
        const u64 b = s.lo + k;
        zxc_b200_job_t Jb;
        Jb.src_off = A.offs[b] + rebase;
        Jb.src_len = (u32)(A.offs[b + 1] - A.offs[b]);
        Jb.dst_off = r.dst_off + (b * bs - r.offset); /* covered whole: the block starts inside the range */
        Jb.dst_cap = ds_expected(A, b);
        A.djobs[pd + k] = Jb;
    }
    if (lane < R.ns) { /* the head slot comes first, in block order */
        const u64 b = (lane == 0 && s.head) ? s.b0 : s.b1;
        zxc_b200_job_t Jb;
        Jb.src_off = A.offs[b] + rebase;
        Jb.src_len = (u32)(A.offs[b + 1] - A.offs[b]);
        Jb.dst_off = (ps + lane) * A.slot_stride;
        Jb.dst_cap = ds_expected(A, b);
        A.sjobs[ps + lane] = Jb;
    }
}

__global__ void __launch_bounds__(DS_THREADS) zxc_dseek_emit(const DSeekArgs A) { ds_emit<false>(A); }
__global__ void __launch_bounds__(DS_THREADS) zxc_dseek_emit_host(const DSeekArgs A) { ds_emit<true>(A); }

/* The admitted ranges' staged spans, [0, p_real) of the staging area, copied from the frame in mapped host memory.
 * CTAs take tiles of DS_FETCH_TILE staged bytes, grid-stride; thread 0 finds the first and the last range a tile
 * touches by binary search over the scanned staged sizes, and a thread whose chunk lies in a tile of several ranges
 * searches between those two.  Each thread writes DS_FETCH_UNROLL 16-byte chunks, adjacent threads adjacent chunks,
 * with all its loads issued before its first store, so that enough reads are in flight to cover PCIe's latency.  A
 * span sits at an offset congruent to its host address mod 16, so every chunk is one aligned 16-byte load: the
 * frame's bytes next to the span come along at its two edges, and only where such a chunk would reach past the frame
 * are its span bytes read one at a time.  Chunks behind a span (its pad) are zeros. */
#define DS_FETCH_THREADS 256
#define DS_FETCH_UNROLL 4
#define DS_FETCH_TILE (DS_FETCH_THREADS * DS_FETCH_UNROLL * 16)

/* the last range in [lo, hi] whose staging starts at or before x, given that lo's does */
__device__ __forceinline__ u32 ds_stage_find(const DSeekArgs& A, u64 x, u32 lo, u32 hi) {
    while (lo < hi) {
        const u32 mid = lo + (hi - lo + 1) / 2;
        if (A.ptiles[mid / ASM_TILE] + A.recs[mid].ex_p <= x) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(DS_FETCH_THREADS) zxc_dseek_fetch(const DSeekArgs A) {
    __shared__ u32 s_lo, s_hi;
    const DSeekState* S = A.st;
    const u64 total = S->p_real;
    const u32 last = (u32)S->first_over - 1; /* every staged byte belongs to a range in front of first_over */
    for (u64 t0 = (u64)blockIdx.x * DS_FETCH_TILE; t0 < total; t0 += (u64)gridDim.x * DS_FETCH_TILE) {
        const u64 t1 = t0 + DS_FETCH_TILE < total ? t0 + DS_FETCH_TILE : total;
        __syncthreads(); /* the previous tile's readers of s_lo, s_hi are done */
        if (threadIdx.x == 0) {
            s_lo = ds_stage_find(A, t0, 0, last);
            s_hi = ds_stage_find(A, t1 - 1, s_lo, last);
        }
        __syncthreads();
        const u32 lo = s_lo, hi = s_hi;
        u32 ci = ~0u;      /* the range whose span the thread has in hand */
        u64 c_pos = 0;     /* its first span byte in the staging area */
        u64 c_len = 0;     /* its span's length */
        u64 c_src = 0;     /* its span's offset in the frame */
        uint4 v[DS_FETCH_UNROLL];
#pragma unroll
        for (u32 k = 0; k < DS_FETCH_UNROLL; k++) {
            v[k] = make_uint4(0u, 0u, 0u, 0u);
            const u64 c = t0 + (u64)(threadIdx.x + k * DS_FETCH_THREADS) * 16;
            if (c >= t1) continue;
            const u32 i = lo == hi ? lo : ds_stage_find(A, c, lo, hi);
            if (i != ci) {
                ci = i;
                const DSeekRec R = A.recs[i];
                const zxc_b200_range_t r = A.ranges[i];
                const DSeekSpan s = ds_span(A, r.offset, r.len);
                c_src = A.offs[s.b0];
                c_len = A.offs[s.b1 + 1] - c_src;
                c_pos = ds_stage_pos(A, i, R, s);
            }
            if (c + 16 <= c_pos || c >= c_pos + c_len) continue; /* the pad */
            const u64 h = c_src + c - c_pos;                     /* c_src >= 16 > c_pos - c: no wrap */
            if (h + 16 <= A.src_size) {
                v[k] = *(const uint4*)(A.hsrc + h);
            } else { /* the chunk reaches past the frame: the span's bytes alone */
                u8 b[16];
#pragma unroll
                for (u32 j = 0; j < 16; j++) b[j] = (c + j >= c_pos && c + j < c_pos + c_len) ? A.hsrc[h + j] : (u8)0;
                v[k] = make_uint4(b[0] | b[1] << 8 | b[2] << 16 | (u32)b[3] << 24, b[4] | b[5] << 8 | b[6] << 16 | (u32)b[7] << 24,
                                  b[8] | b[9] << 8 | b[10] << 16 | (u32)b[11] << 24,
                                  b[12] | b[13] << 8 | b[14] << 16 | (u32)b[15] << 24);
            }
        }
#pragma unroll
        for (u32 k = 0; k < DS_FETCH_UNROLL; k++) {
            const u64 c = t0 + (u64)(threadIdx.x + k * DS_FETCH_THREADS) * 16;
            if (c < t1) *(uint4*)(A.stage + c) = v[k];
        }
    }
}

/* first_failure's rule for one job: its own negative status, or CORRUPT_DATA for another size; 1 when it held */
__device__ __forceinline__ int ds_job_verdict(i32 st, u32 want) {
    if (st < 0) return st;
    return (u32)st != want ? ZXC_ERROR_CORRUPT_DATA : 1;
}

/* n bytes from a slot (16-byte aligned base, any offset) to d (any alignment), by the whole CTA: the bytes in front
 * of d's first 16-byte boundary and behind its last one one at a time, the rest as 16-byte stores built from aligned
 * 4-byte loads */
__device__ __forceinline__ void ds_copy(u8* d, const u8* s, u64 n) {
    const u64 head = ((16u - ((uintptr_t)d & 15u)) & 15u) < n ? ((16u - ((uintptr_t)d & 15u)) & 15u) : n;
    const u64 body = (n - head) & ~(u64)15;
    for (u64 k = threadIdx.x; k < head; k += blockDim.x) d[k] = s[k];
    for (u64 k = head + body + threadIdx.x; k < n; k += blockDim.x) d[k] = s[k];
    const u8* sb = s + head;
    const u32 sh = (u32)((uintptr_t)sb & 3u) * 8u;
    const u32* w = (const u32*)((uintptr_t)sb & ~(uintptr_t)3);
    uint4* o = (uint4*)(d + head);
    for (u64 c = threadIdx.x; c < body / 16; c += blockDim.x) {
        const u32* p = w + 4 * c;
        const u32 a0 = p[0], a1 = p[1], a2 = p[2], a3 = p[3], a4 = sh ? p[4] : 0u;
        uint4 v;
        v.x = __funnelshift_r(a0, a1, sh);
        v.y = __funnelshift_r(a1, a2, sh);
        v.z = __funnelshift_r(a2, a3, sh);
        v.w = __funnelshift_r(a3, a4, sh);
        o[c] = v;
    }
}

__global__ void __launch_bounds__(DS_THREADS) zxc_dseek_finish(const DSeekArgs A) {
    __shared__ unsigned long long s_bad;
    const DSeekState* S = A.st;
    const u64 i = blockIdx.x;
    const DSeekRec R = A.recs[i];
    if (R.v != 1) {
        if (threadIdx.x == 0) A.results[i] = R.v;
        return;
    }
    if (i >= S->first_over) {
        if (threadIdx.x == 0) A.results[i] = ZXC_ERROR_MEMORY;
        return;
    }
    const zxc_b200_range_t r = A.ranges[i];
    const DSeekSpan s = ds_span(A, r.offset, r.len);
    const u64 t = i / ASM_TILE;
    const u64 pd = A.J - S->d_real + A.tiles[2 * t] + R.ex_d;
    const u64 ps = 2ull * A.n - S->s_real + A.tiles[2 * t + 1] + R.ex_s;
    if (threadIdx.x == 0) s_bad = ~0ull;
    __syncthreads();
    for (u32 k = threadIdx.x; k < R.nd; k += blockDim.x)
        if (ds_job_verdict(A.dstatus[pd + k], A.djobs[pd + k].dst_cap) != 1) atomicMin(&s_bad, (unsigned long long)k);
    __syncthreads();
    /* block order: head slot, direct blocks, tail slot */
    int v = 1;
    if (s.head) v = ds_job_verdict(A.sstatus[ps], ds_expected(A, s.b0));
    if (v == 1 && s_bad != ~0ull) v = ds_job_verdict(A.dstatus[pd + s_bad], A.djobs[pd + s_bad].dst_cap);
    if (v == 1 && s.tail) v = ds_job_verdict(A.sstatus[ps + s.head], ds_expected(A, s.b1));
    if (v != 1) {
        if (threadIdx.x == 0) A.results[i] = v;
        return;
    }
    const u64 bs = A.block_size, end = r.offset + r.len;
    if (s.head) {
        const u64 b_end = s.b0 * bs + ds_expected(A, s.b0);
        ds_copy(A.dst + r.dst_off, A.slots + ps * A.slot_stride + (r.offset - s.b0 * bs),
                (end < b_end ? end : b_end) - r.offset);
    }
    if (s.tail)
        ds_copy(A.dst + r.dst_off + (s.b1 * bs - r.offset), A.slots + (ps + s.head) * A.slot_stride, end - s.b1 * bs);
    if (threadIdx.x == 0) A.results[i] = (long long)r.len;
}
