/*
 * zxc_blocks.cuh -- the block API in HBM: many frameless blocks compressed (zxc_b200_compress_blocks_device) or
 * decompressed (zxc_b200_decompress_blocks_device) in one stream-ordered call each, every item exactly what this
 * library's zxc_compress_block / zxc_decompress_block(_safe) gives it alone.
 *
 * Compress.  A block's bytes depend on its content, the level, the checksum flag and the dictionary, not on the block
 * size the encoder's per-warp scratch is laid out for (tests/test_blocks_device.py pins this on the reference), so one
 * encode launch takes items of any size up to the largest one's size class:
 *   zxc_blocks_ctiles    per item: zxc_compress_block's argument checks, its pool share and its size class; the shares
 *                        scanned within tiles of ASM_TILE items, and each tile's largest class
 *   zxc_blocks_cscan     one thread: the tiles' scan, and the first item i whose admission no longer fits the room:
 *                        (shares of items 0..i) + one encode slot laid out for the largest class among them > room.
 *                        It and every later item that passed the checks get ZXC_ERROR_MEMORY.  The encode slot size
 *                        (B: the admitted items' largest class) and the warps whose slot reaches into the used pool
 *   zxc_blocks_cgather   one warp per item: its input copy and staging slot in the pool, and the caller's bytes into
 *                        the 256-aligned copy with 64 zero bytes behind (what EncodeParams::src assumes)
 *   zxc_seed_kernel      (zxc_encode.cuh, unchanged) with a dictionary
 *   zxc_blocks_encode    one warp per claimed item: the unchanged encode_block with P.block_size = B, the item's own n
 *   zxc_blocks_cfinish   one warp per item: DST_TOO_SMALL when the block does not fit, else the copy into dst
 * An item's share of the pool is its input copy, r256(n + 64), and its staging slot, r256(n + 12): encode_block
 * writes at most 8 + n + 4 bytes for an n-byte input (a RAW block with its checksum; it picks RAW whenever the encoded
 * form would not be shorter than n, before writing a byte of it).  The W launched warps' encode slots end at the
 * room's end, slot g at room_end - (W - g) * wstride(B); warps whose slot would reach into the used pool exit.
 *
 * Decompress.  zxc_decompress_block decodes one job {src, dst, min(src_size, 2^32 - 1), dst_capacity} at block_cap =
 * zxf_block_size_ceil(dst_capacity); the decode kernels take block_cap as a launch parameter, so items are grouped by
 * that class into the batched frame decode's launch slots (dp_slot's numbering):
 *   zxc_blocks_dcount    per item: the argument checks and its class (MEMORY above the scratch's B); per tile and
 *                        slot, the items' places scanned in index order
 *   zxc_dbatch_slots     (zxc_dbatch.cuh) one CTA: per slot, the tiles' scan, its real jobs and its work counters
 *   zxc_blocks_dplace    per item: its job into its slot's window at device addresses over a zero base, right-aligned
 *                        in index order; zeroed status words in front of every window's real jobs
 *   zxc_decode_kernel    (zxc_decode.cuh, unchanged) one launch_decode per slot
 *   zxc_blocks_dfinish   per item: its job's status is its result
 */
#pragma once
#include <cuda_runtime.h>

#include "zxc_assemble.cuh"
#include "zxc_dbatch.cuh"
#include "zxc_encode.cuh"
#include "zxc_format.h"

#define BK_THREADS 256
#define BK_CLASSES (ZXC_BLOCK_SIZE_MAX_LOG2 - ZXC_BLOCK_SIZE_MIN_LOG2 + 1)

/* the size class of an n-byte block: zxf_block_size_ceil(n) = ZXC_BLOCK_SIZE_MIN << class */
__device__ __forceinline__ u32 bk_class(u64 n) {
    u32 c = 0;
    while (c + 1 < BK_CLASSES && ((u64)ZXC_BLOCK_SIZE_MIN << c) < n) c++;
    return c;
}

/* ---- compress ---- */
struct BlocksCState {
    unsigned long long counter;    /* the encode kernel's work counter */
    unsigned long long first_over; /* first item past the room (n: none) */
    unsigned long long skip;       /* encode warps whose slot reaches into the used pool: they exit */
    unsigned long long wstride;    /* the encode slot of class B */
    unsigned int bs;               /* B */
};
#define BK_STATE_BYTES 256
static_assert(sizeof(BlocksCState) <= BK_STATE_BYTES, "BlocksCState fits its region");

struct BlocksCItem {
    const u8* src;
    u8* dst;
    u8* in;    /* its input copy in the pool */
    u8* stage; /* its staging slot, right behind the copy */
    unsigned long long cap;
    unsigned long long ex; /* pool units in front of it within its tile */
    unsigned int n, share, cls, live, size;
};

struct BlocksCArgs {
    const zxc_b200_frame_t* items;
    long long* results;
    BlocksCState* st;
    BlocksCItem* I;
    unsigned long long* tiles; /* 2 x n_tiles: the shares' tile sums, then their exclusive scan; the largest class + 1 */
    u8* room;
    unsigned long long room_bytes;          /* a multiple of 256 */
    unsigned long long wstride[BK_CLASSES]; /* enc_layout(class size, level).total */
    unsigned int n, warps;
};

__global__ void __launch_bounds__(ASM_THREADS) zxc_blocks_ctiles(const BlocksCArgs A) {
    __shared__ unsigned int s_max;
    if (threadIdx.x == 0) s_max = 0;
    __syncthreads();
    const u64 first = (u64)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    u32 sh[ASM_ITEMS];
    u64 s = 0;
#pragma unroll
    for (u32 q = 0; q < ASM_ITEMS; q++) {
        sh[q] = 0;
        if (first + q >= A.n) continue;
        const zxc_b200_frame_t d = A.items[first + q];
        BlocksCItem& I = A.I[first + q];
        /* zxc_compress_block's argument checks, in its order */
        long long v = 1;
        if (!d.src || !d.dst || d.src_size == 0 || d.dst_capacity == 0) v = ZXC_ERROR_NULL_INPUT;
        else if (d.src_size > ZXC_BLOCK_SIZE_MAX) v = ZXC_ERROR_BAD_BLOCK_SIZE;
        u32 cls = 0;
        if (v == 1) {
            cls = bk_class(d.src_size);
            sh[q] = (u32)(((d.src_size + 64 + 255) / 256) + ((d.src_size + 12 + 255) / 256));
            atomicMax(&s_max, cls + 1);
        } else {
            A.results[first + q] = v;
        }
        I.src = (const u8*)d.src;
        I.dst = (u8*)d.dst;
        I.cap = d.dst_capacity;
        I.n = (u32)(v == 1 ? d.src_size : 0);
        I.share = sh[q];
        I.cls = cls;
        I.live = v == 1;
        s += sh[q];
    }
    unsigned long long total;
    u64 ex = asm_cta_excl(s, &total); /* its barriers also order s_max */
#pragma unroll
    for (u32 q = 0; q < ASM_ITEMS; q++) {
        if (first + q < A.n) A.I[first + q].ex = ex;
        ex += sh[q];
    }
    if (threadIdx.x == 0) {
        const u32 n_tiles = (A.n + ASM_TILE - 1) / ASM_TILE;
        A.tiles[blockIdx.x] = total;
        A.tiles[n_tiles + blockIdx.x] = s_max;
    }
}

/* one thread: admission is monotone in the index (the shares' sum and the largest class only grow), so the first item
 * past the room is found tile by tile, then item by item inside the first tile that ends past it */
__global__ void zxc_blocks_cscan(const BlocksCArgs A) {
    BlocksCState* S = A.st;
    const u32 n_tiles = (A.n + ASM_TILE - 1) / ASM_TILE;
    const auto over = [&](u64 units, u32 m) { return m && units * 256 + A.wstride[m - 1] > A.room_bytes; };
    u64 acc = 0;
    u32 m = 0, t_over = n_tiles; /* m: the largest class + 1 in front of t_over */
    for (u32 t = 0; t < n_tiles; t++) {
        const u64 v = A.tiles[t];
        const u32 tm = (u32)A.tiles[n_tiles + t];
        A.tiles[t] = acc;
        if (t_over == n_tiles) {
            if (over(acc + v, tm > m ? tm : m)) t_over = t;
            else if (tm > m) m = tm;
        }
        acc += v;
    }
    u64 f = A.n, used = acc;
    if (t_over != n_tiles) {
        u64 u = A.tiles[t_over];
        for (u64 i = (u64)t_over * ASM_TILE; i < A.n && i < (u64)(t_over + 1) * ASM_TILE; i++) {
            const BlocksCItem& I = A.I[i];
            if (!I.live) continue;
            const u32 mi = I.cls + 1 > m ? I.cls + 1 : m;
            if (over(u + I.share, mi)) {
                f = i;
                break;
            }
            u += I.share;
            m = mi;
        }
        used = u;
    }
    const u32 b = m ? m - 1 : 0;
    const u64 ws = A.wstride[b];
    const u64 fit = (A.room_bytes - used * 256) / ws;
    S->first_over = f;
    S->bs = ZXC_BLOCK_SIZE_MIN << b;
    S->wstride = ws;
    S->skip = fit < A.warps ? A.warps - fit : 0;
    S->counter = 0;
}

/* the caller's bytes of item i and the 64 zero bytes behind them: 16-byte vectors when the source is 16-byte aligned,
 * else bytes; nothing outside [src, src + src_size) is read */
__global__ void __launch_bounds__(BK_THREADS) zxc_blocks_cgather(const BlocksCArgs A) {
    const u32 lane = threadIdx.x & 31;
    const u64 warps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u64 first_over = A.st->first_over;
    for (u64 i = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < A.n; i += warps) {
        BlocksCItem& I = A.I[i];
        if (!I.live) continue;
        if (i >= first_over) {
            __syncwarp();
            if (lane == 0) {
                A.results[i] = ZXC_ERROR_MEMORY;
                I.live = 0;
            }
            continue;
        }
        const u32 n = I.n;
        u8* d = A.room + (A.tiles[i / ASM_TILE] + I.ex) * 256;
        const u8* s = I.src;
        if (((uintptr_t)s & 15) == 0) {
            const u32 n16 = n >> 4;
            for (u32 q = lane; q < n16; q += 32) reinterpret_cast<uint4*>(d)[q] = reinterpret_cast<const uint4*>(s)[q];
            for (u32 q = (n16 << 4) + lane; q < n; q += 32) d[q] = s[q];
        } else {
            for (u32 q = lane; q < n; q += 32) d[q] = s[q];
        }
        d[n + lane] = 0;
        d[n + 32 + lane] = 0;
        __syncwarp();
        if (lane == 0) {
            I.in = d;
            I.stage = d + (((u64)n + 64 + 255) & ~255ull);
        }
    }
}

/* zxc_encode_kernel over the items: item j from its input copy into its staging slot, each with its own n; the
 * per-warp scratch is laid out for B, which the scan chose on the device */
template <bool OPT>
__global__ void __launch_bounds__(ENC_CTA_THREADS, OPT ? ENC_OPT_MIN_CTAS : 0)
    zxc_blocks_encode(EncodeParams P, const BlocksCArgs A) {
    const u32 lane = threadIdx.x & 31;
    const u32 gwarp = blockIdx.x * ENC_WARPS_PER_CTA + (threadIdx.x >> 5);
    __shared__ u32 s_hist[OPT ? ENC_WARPS_PER_CTA : 1][256];
    u32* hist = s_hist[OPT ? (threadIdx.x >> 5) : 0];
    const BlocksCState* S = A.st;
    if (gwarp < S->skip) return; /* its slot would reach into the used pool */
    P.block_size = S->bs;
    u8* scratch = A.room + A.room_bytes - (size_t)(A.warps - gwarp) * S->wstride;
    for (;;) {
        unsigned long long j = 0;
        if (lane == 0) j = atomicAdd(P.counter, 1ull);
        j = __shfl_sync(FULL, j, 0);
        if (j >= A.n) break;
        if (!A.I[j].live) continue;
        const u32 w = encode_block<OPT>(P, A.I[j].in, A.I[j].n, A.I[j].stage, scratch, hist, lane);
        __syncwarp();
        if (lane == 0) A.I[j].size = w;
    }
}

__global__ void __launch_bounds__(BK_THREADS) zxc_blocks_cfinish(const BlocksCArgs A) {
    const u32 lane = threadIdx.x & 31;
    const u64 warps = ((u64)gridDim.x * blockDim.x) >> 5;
    for (u64 i = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < A.n; i += warps) {
        const BlocksCItem& I = A.I[i];
        if (!I.live) continue;
        const u32 w = I.size;
        if (w > I.cap) { /* dst stays untouched */
            if (lane == 0) A.results[i] = ZXC_ERROR_DST_TOO_SMALL;
            continue;
        }
        const u8* s = I.stage;
        u8* d = I.dst;
        if (((uintptr_t)d & 15) == 0) {
            const u32 n16 = w >> 4;
            for (u32 q = lane; q < n16; q += 32) reinterpret_cast<uint4*>(d)[q] = reinterpret_cast<const uint4*>(s)[q];
            for (u32 q = (n16 << 4) + lane; q < w; q += 32) d[q] = s[q];
        } else {
            for (u32 q = lane; q < w; q += 32) d[q] = s[q];
        }
        if (lane == 0) A.results[i] = w;
    }
}

/* ---- decompress ---- */
struct BlocksDItem {
    unsigned long long pos; /* zxc_blocks_dcount: its place among its tile's items of its slot; then its window index */
    unsigned int slot;      /* DP_SLOTS when it decodes nothing */
};

struct BlocksDArgs {
    const zxc_b200_frame_t* items;
    long long* results;
    DBatchState* st;
    BlocksDItem* I;
    unsigned long long* stiles; /* n_tiles x n_slots: the slots' item counts per tile, then their exclusive scan */
    zxc_b200_job_t* jobs;       /* n_slots windows of n */
    i32* status;                /* n_slots windows of n */
    unsigned long long cap_max; /* ZXC_BLOCK_SIZE_MAX + ZXF_TAIL_PAD, or ZXC_BLOCK_SIZE_MAX for the safe call */
    unsigned int n, n_slots, bs, verify;
};

__global__ void __launch_bounds__(ASM_THREADS) zxc_blocks_dcount(const BlocksDArgs A) {
    __shared__ unsigned int s_used;
    if (threadIdx.x == 0) s_used = 0;
    __syncthreads();
    const u64 first = (u64)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    u32 sl[ASM_ITEMS];
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        sl[k] = DP_SLOTS;
        if (first + k >= A.n) continue;
        const zxc_b200_frame_t d = A.items[first + k];
        /* zxc_decompress_block's argument checks, in its order, then this call's limit */
        long long v = 1;
        if (!d.src || !d.dst || d.src_size < ZXF_BLOCK_HDR || d.dst_capacity == 0) v = ZXC_ERROR_NULL_INPUT;
        else if (d.dst_capacity > A.cap_max) v = ZXC_ERROR_BAD_BLOCK_SIZE;
        else if (((u64)ZXC_BLOCK_SIZE_MIN << bk_class(d.dst_capacity)) > A.bs) v = ZXC_ERROR_MEMORY;
        if (v == 1) {
            sl[k] = bk_class(d.dst_capacity) * 2 + A.verify;
            atomicOr(&s_used, 1u << sl[k]);
        } else {
            A.results[first + k] = v;
        }
        A.I[first + k].slot = sl[k];
    }
    __syncthreads();
    const u32 used = s_used;
    for (u32 s = 0; s < A.n_slots; s++) {
        if (!(used >> s & 1u)) {
            if (threadIdx.x == 0) A.stiles[(u64)blockIdx.x * A.n_slots + s] = 0;
            continue;
        }
        u64 v = 0;
#pragma unroll
        for (u32 k = 0; k < ASM_ITEMS; k++) v += sl[k] == s;
        unsigned long long total;
        u64 ex = asm_cta_excl(v, &total);
#pragma unroll
        for (u32 k = 0; k < ASM_ITEMS; k++) {
            if (sl[k] == s) A.I[first + k].pos = ex++;
        }
        if (threadIdx.x == 0) A.stiles[(u64)blockIdx.x * A.n_slots + s] = total;
    }
}

__global__ void __launch_bounds__(BK_THREADS) zxc_blocks_dplace(const BlocksDArgs A) {
    const DBatchState* S = A.st;
    const u64 i = (u64)blockIdx.x * BK_THREADS + threadIdx.x;
    if (i >= A.n) return;
    /* no stale deferral marks in front of the real jobs (the deferred launch may scan the status words from 0) */
    for (u32 s = 0; s < A.n_slots; s++)
        if (S->real[s] && i < A.n - S->real[s]) A.status[(u64)s * A.n + i] = 0;
    BlocksDItem& I = A.I[i];
    const u32 s = I.slot;
    if (s >= DP_SLOTS) return;
    const zxc_b200_frame_t d = A.items[i];
    const u64 w = A.n - S->real[s] + A.stiles[(i / ASM_TILE) * A.n_slots + s] + I.pos;
    zxc_b200_job_t Jb;
    Jb.src_off = (u64)(uintptr_t)d.src;
    Jb.dst_off = (u64)(uintptr_t)d.dst;
    Jb.src_len = (u32)(d.src_size > 0xFFFFFFFFull ? 0xFFFFFFFFull : d.src_size);
    Jb.dst_cap = (u32)d.dst_capacity;
    A.jobs[(u64)s * A.n + w] = Jb;
    I.pos = w;
}

__global__ void __launch_bounds__(BK_THREADS) zxc_blocks_dfinish(const BlocksDArgs A) {
    const u64 i = (u64)blockIdx.x * BK_THREADS + threadIdx.x;
    if (i >= A.n) return;
    const BlocksDItem I = A.I[i];
    if (I.slot < DP_SLOTS) A.results[i] = A.status[(u64)I.slot * A.n + I.pos];
}
