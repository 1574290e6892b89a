/*
 * zxc_cbatch.cuh -- many independent buffers in HBM compressed into one frame each, in one stream-ordered call
 * (zxc_b200_compress_device_batch).  Every step is zxc_b200_compress_device's per-frame algorithm run over all frames
 * at once, with the blocks of every frame numbered in one global sequence j = 0 .. nb:
 *
 *   zxc_cbatch_tiles     per frame: the argument checks (NULL_INPUT, BAD_BLOCK_SIZE, DST_TOO_SMALL), its share of
 *                        the pool and its block count, both scanned within tiles of ASM_TILE frames
 *   zxc_cbatch_scan      one CTA: the tile sums' scans and the first frame whose share ends past the pool (it and
 *                        every later frame that passed the checks get ZXC_ERROR_MEMORY); nb; the work counter
 *   zxc_cbatch_place     per frame: its first global block (the lookup's search key) and its input copy's address
 *   zxc_cbatch_gather    one warp per block: the caller's bytes into the frame's 256-aligned input copy, and 64
 *                        zero bytes behind its last block (what EncodeParams::src assumes)
 *   zxc_seed_kernel      (zxc_encode.cuh, unchanged) with a dictionary
 *   zxc_encode_batch_kernel  one warp per claimed block: the unchanged encode_block into staging slot j
 *   zxc_cbatch_sums      per tile of ASM_TILE blocks: the on-disk sizes' sum
 *   zxc_cbatch_bscan     one CTA: the exclusive scan of those sums
 *   zxc_cbatch_offsets   per block: its offset in the scan of all on-disk sizes
 *   zxc_cbatch_fit       per frame: its body (the scan at its last block minus the scan at its first) and whether
 *                        header + body + trailer fit its capacity
 *   zxc_cbatch_blocks    per block: the absolute destination, the SEK entry and the global hash term of a frame
 *                        that fits; size 0 for one that does not and for the unused entries past nb, so the
 *                        compaction copies nothing there
 *   zxc_compact_kernel   (zxc_encode.cuh, unchanged) over a zero base: every block to its absolute address
 *   zxc_cbatch_finish    per frame: file header, EOF block, SEK header, footer and the result
 *
 * The room: the pool, then one encode slot.  A frame's share of the pool is in_i + nb_i * staging_stride / 256 units of
 * 256 bytes, in_i = r256(src_size_i + 64) / 256 (none for an empty frame).  Staging slot j lies at pool + j *
 * staging_stride, and frame i's input copy right behind the staging slots of all nb blocks, at 256 * IN_i past them
 * (IN_i: the sum of in_k over the frames in front of it).  The W launched warps' encode slots end at the room's end,
 * slot g at room_end - (W - g) * wstride, and the warps whose slot would reach into the pool's used part (the lowest g)
 * exit at once: a batch that leaves more of the pool free runs more warps, and one warp always fits.
 */
#pragma once
#include <cuda_runtime.h>

#include "zxc_assemble.cuh"
#include "zxc_encode.cuh"
#include "zxc_format.h"

#define CB_THREADS 256
#define CB_POOL_UNITS_MAX (1ull << 32) /* the pool counts at most 1 TiB, which keeps every scan far from overflow */

/* the first bytes of the caller's scratch */
struct CBatchState {
    unsigned long long counter;    /* the encode kernel's work counter */
    unsigned long long nb;         /* blocks of the frames in front of first_over */
    unsigned long long first_over; /* first frame past the pool (n: none) */
    unsigned long long skip;       /* encode warps whose slot reaches into the pool's used part: they exit */
};
#define CB_STATE_BYTES 256
static_assert(sizeof(CBatchState) <= CB_STATE_BYTES, "CBatchState fits its region");

struct CBatchFrame {
    const u8* src;
    u8* dst;
    u8* in;                      /* its input copy in the pool */
    unsigned long long src_size, cap, fixed;
    unsigned long long share;    /* pool units (clamped to pool + 1) */
    unsigned long long ex_share; /* within its tile, then (zxc_cbatch_place) over all frames */
    unsigned long long ex_nb;
    unsigned long long body, off0; /* body bytes; the scan of on-disk sizes at its first block */
    unsigned int nb;             /* blocks (clamped like share) */
    unsigned int live;           /* passed the checks and fits the pool: still to be written */
    unsigned int fits;
    unsigned int hash;           /* global hash, XOR-accumulated by zxc_cbatch_blocks */
};

/* host-computed, passed by value: the options and the bytes every frame shares */
struct CBatchArgs {
    const zxc_b200_frame_t* frames;
    long long* results;
    CBatchState* st;
    CBatchFrame* F;
    unsigned long long* first;  /* n: each frame's first global block (ascending: the lookup's search key) */
    unsigned long long* ftiles; /* 2 x n_tiles: the share and block tile sums, then their exclusive scans */
    unsigned long long* btiles; /* ceil(nb_max / ASM_TILE): the on-disk size tile sums, then their scan */
    unsigned long long* offs;   /* nb_max: the scan of on-disk sizes, then absolute destinations */
    u32* sizes;                 /* nb_max: on-disk sizes */
    u8* staging;                /* the pool's base */
    unsigned long long pool_units, wstride;
    unsigned int n, nb_max, warps, block_size, staging_stride, checksum, seekable;
    unsigned char header[16];
    unsigned char eof[8];
};

/* the frame that holds global block j < nb: the last frame with first <= j */
__device__ __forceinline__ u32 cb_frame_of(const CBatchArgs& A, u64 j) {
    u32 lo = 0, hi = A.n; /* first[lo] <= j < first[hi] */
    while (hi - lo > 1) {
        const u32 mid = lo + (hi - lo) / 2;
        if (A.first[mid] <= j) lo = mid;
        else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(ASM_THREADS) zxc_cbatch_tiles(const CBatchArgs A) {
    const u64 first = (u64)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    const u64 bs = A.block_size, k = A.staging_stride / 256;
    u64 sh[ASM_ITEMS], nb[ASM_ITEMS], s = 0, b = 0;
#pragma unroll
    for (u32 q = 0; q < ASM_ITEMS; q++) {
        sh[q] = nb[q] = 0;
        if (first + q < A.n) {
            const zxc_b200_frame_t d = A.frames[first + q];
            CBatchFrame& F = A.F[first + q];
            /* zxc_b200_compress_device's argument checks, in its order */
            long long v = 1;
            u64 nb64 = 0, fixed = 0;
            if (!d.dst || d.dst_capacity == 0 || (d.src_size > 0 && !d.src)) {
                v = ZXC_ERROR_NULL_INPUT;
            } else {
                nb64 = d.src_size / bs + (d.src_size % bs != 0);
                if (nb64 > 0xFFFFFFFFull - 2) {
                    v = ZXC_ERROR_BAD_BLOCK_SIZE;
                } else {
                    fixed = ZXC_FILE_HEADER_SIZE + ZXF_BLOCK_HDR + (A.seekable && nb64 ? ZXF_BLOCK_HDR + 4 * nb64 : 0) +
                            ZXC_FILE_FOOTER_SIZE;
                    if (d.dst_capacity < fixed) v = ZXC_ERROR_DST_TOO_SMALL;
                }
            }
            if (v == 1) {
                if (nb64) {
                    /* clamped past the pool: such a frame is past it either way */
                    const u64 lim = A.pool_units / k + 1;
                    nb[q] = nb64 < lim ? nb64 : lim;
                    const u64 in = (d.src_size + 64 + 255) / 256;
                    const u64 c = (in < A.pool_units ? in : A.pool_units) + nb[q] * k;
                    sh[q] = c <= A.pool_units ? c : A.pool_units + 1;
                }
            } else {
                A.results[first + q] = v;
            }
            F.src = (const u8*)d.src;
            F.dst = (u8*)d.dst;
            F.src_size = d.src_size;
            F.cap = d.dst_capacity;
            F.fixed = fixed;
            F.share = sh[q];
            F.nb = (u32)nb[q];
            F.live = v == 1;
            F.hash = 0;
        }
        s += sh[q];
        b += nb[q];
    }
    unsigned long long ts, tb;
    u64 es = asm_cta_excl(s, &ts);
    u64 eb = asm_cta_excl(b, &tb);
#pragma unroll
    for (u32 q = 0; q < ASM_ITEMS; q++) {
        if (first + q < A.n) {
            A.F[first + q].ex_share = es;
            A.F[first + q].ex_nb = eb;
        }
        es += sh[q];
        eb += nb[q];
    }
    if (threadIdx.x == 0) {
        const u32 n_tiles = (A.n + ASM_TILE - 1) / ASM_TILE;
        A.ftiles[blockIdx.x] = ts;
        A.ftiles[n_tiles + blockIdx.x] = tb;
    }
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_cbatch_scan(const CBatchArgs A) {
    __shared__ unsigned long long s_tile, s_first;
    CBatchState* S = A.st;
    const u32 n_tiles = (A.n + ASM_TILE - 1) / ASM_TILE;
    if (threadIdx.x == 0) s_tile = s_first = ~0ull;
    unsigned long long cs = 0, cb = 0;
    for (u32 b = 0; b < n_tiles; b += blockDim.x) {
        const u32 i = b + threadIdx.x;
        const unsigned long long vs = i < n_tiles ? A.ftiles[i] : 0, vb = i < n_tiles ? A.ftiles[n_tiles + i] : 0;
        unsigned long long ts, tb;
        const unsigned long long es = cs + asm_cta_excl(vs, &ts); /* its barriers also order s_tile */
        const unsigned long long eb = cb + asm_cta_excl(vb, &tb);
        if (i < n_tiles) {
            A.ftiles[i] = es;
            A.ftiles[n_tiles + i] = eb;
            if (es + vs > A.pool_units) atomicMin(&s_tile, (unsigned long long)i);
        }
        cs += ts;
        cb += tb;
    }
    __syncthreads();
    const u64 t = s_tile;
    if (t != ~0ull) { /* the first frame of that tile whose share ends past the pool */
        for (u64 i = t * ASM_TILE + threadIdx.x; i < A.n && i < (t + 1) * ASM_TILE; i += blockDim.x)
            if (A.ftiles[t] + A.F[i].ex_share + A.F[i].share > A.pool_units) atomicMin(&s_first, i);
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    const u64 f = t != ~0ull ? s_first : A.n;
    const u64 used = f < A.n ? A.ftiles[f / ASM_TILE] + A.F[f].ex_share : cs;
    const u64 room = (A.pool_units - used) * 256 / A.wstride + 1;
    S->first_over = f;
    S->nb = f < A.n ? A.ftiles[n_tiles + f / ASM_TILE] + A.F[f].ex_nb : cb;
    S->skip = room < A.warps ? A.warps - room : 0;
    S->counter = 0;
}

__global__ void __launch_bounds__(CB_THREADS) zxc_cbatch_place(const CBatchArgs A) {
    const u64 i = (u64)blockIdx.x * CB_THREADS + threadIdx.x;
    if (i >= A.n) return;
    const u32 n_tiles = (A.n + ASM_TILE - 1) / ASM_TILE;
    CBatchFrame* F = A.F + i;
    const u64 nbx = A.ftiles[n_tiles + i / ASM_TILE] + F->ex_nb;
    A.first[i] = nbx;
    if (!F->live) return;
    if (i >= A.st->first_over) {
        A.results[i] = ZXC_ERROR_MEMORY;
        F->live = 0;
        return;
    }
    const u64 ex = A.ftiles[i / ASM_TILE] + F->ex_share;
    const u64 in_before = ex - nbx * (A.staging_stride / 256); /* the input units of the frames in front of it */
    F->in = A.staging + A.st->nb * A.staging_stride + in_before * 256;
}

/* the caller's bytes of block j, and the zero bytes behind a frame's last block: 16-byte vectors when the source is
 * 16-byte aligned, else bytes; nothing outside [src, src + src_size) is read */
__global__ void __launch_bounds__(CB_THREADS) zxc_cbatch_gather(const CBatchArgs A) {
    const u32 lane = threadIdx.x & 31;
    const u64 warps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u64 nb = A.st->nb;
    for (u64 j = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < nb; j += warps) {
        const u32 f = cb_frame_of(A, j);
        const CBatchFrame& F = A.F[f];
        const u64 jl = j - A.first[f];
        const u64 off = jl * A.block_size;
        const u64 rem = F.src_size - off;
        const u32 n = rem < A.block_size ? (u32)rem : A.block_size;
        const u8* s = F.src + off;
        u8* d = F.in + off;
        if (((uintptr_t)s & 15) == 0) {
            const u32 n16 = n >> 4;
            for (u32 q = lane; q < n16; q += 32) reinterpret_cast<uint4*>(d)[q] = reinterpret_cast<const uint4*>(s)[q];
            for (u32 q = (n16 << 4) + lane; q < n; q += 32) d[q] = s[q];
        } else {
            for (u32 q = lane; q < n; q += 32) d[q] = s[q];
        }
        if (jl + 1 == F.nb) d[n + lane] = 0, d[n + 32 + lane] = 0;
    }
}

/* zxc_encode_kernel over the global block sequence: block j is block j - first[f] of frame f, read from its input
 * copy; the slot, the size and the per-warp scratch are indexed as there */
template <bool OPT>
__global__ void __launch_bounds__(ENC_CTA_THREADS, OPT ? ENC_OPT_MIN_CTAS : 0)
    zxc_encode_batch_kernel(const EncodeParams P, const CBatchArgs A) {
    const u32 lane = threadIdx.x & 31;
    const u32 gwarp = blockIdx.x * ENC_WARPS_PER_CTA + (threadIdx.x >> 5);
    __shared__ u32 s_hist[OPT ? ENC_WARPS_PER_CTA : 1][256];
    u32* hist = s_hist[OPT ? (threadIdx.x >> 5) : 0];
    if (gwarp < A.st->skip) return; /* its slot would reach into the pool's used part */
    u8* scratch = P.scratch + (size_t)gwarp * P.scratch_stride;
    for (;;) {
        unsigned long long j = 0;
        if (lane == 0) j = atomicAdd(P.counter, 1ull);
        j = __shfl_sync(FULL, j, 0);
        if (j >= A.st->nb) break; /* read per claim, so nothing of the batch stays live across encode_block */
        const u32 f = cb_frame_of(A, j);
        const unsigned long long off = (j - A.first[f]) * (unsigned long long)P.block_size;
        const unsigned long long rem = A.F[f].src_size - off;
        const u32 n = rem < P.block_size ? (u32)rem : P.block_size;
        const u32 w = encode_block<OPT>(P, A.F[f].in + off, n, P.staging + (size_t)j * P.staging_stride, scratch, hist,
                                        lane);
        __syncwarp();
        if (lane == 0) P.out_size[j] = w;
    }
}

/* zxc_asm_tile_sums over the first nb blocks */
__global__ void __launch_bounds__(ASM_THREADS) zxc_cbatch_sums(const CBatchArgs A) {
    const u64 nb = A.st->nb;
    if ((u64)blockIdx.x * ASM_TILE >= nb) return;
    const u64 base = (u64)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    u64 s = 0;
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++)
        if (base + k < nb) s += A.sizes[base + k];
    unsigned long long total;
    asm_cta_excl(s, &total);
    if (threadIdx.x == 0) A.btiles[blockIdx.x] = total;
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_cbatch_bscan(const CBatchArgs A) {
    const u64 n_tiles = (A.st->nb + ASM_TILE - 1) / ASM_TILE;
    unsigned long long carry = 0;
    for (u64 b = 0; b < n_tiles; b += blockDim.x) {
        const u64 i = b + threadIdx.x;
        const unsigned long long v = i < n_tiles ? A.btiles[i] : 0;
        unsigned long long total;
        const unsigned long long ex = asm_cta_excl(v, &total);
        if (i < n_tiles) A.btiles[i] = carry + ex;
        carry += total;
    }
}

__global__ void __launch_bounds__(ASM_THREADS) zxc_cbatch_offsets(const CBatchArgs A) {
    const u64 nb = A.st->nb;
    if ((u64)blockIdx.x * ASM_TILE >= nb) return;
    const u64 base = (u64)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    u32 sz[ASM_ITEMS];
    u64 s = 0;
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        sz[k] = base + k < nb ? A.sizes[base + k] : 0u;
        s += sz[k];
    }
    unsigned long long total;
    u64 off = A.btiles[blockIdx.x] + asm_cta_excl(s, &total);
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        if (base + k < nb) A.offs[base + k] = off;
        off += sz[k];
    }
}

__global__ void __launch_bounds__(CB_THREADS) zxc_cbatch_fit(const CBatchArgs A) {
    const u64 i = (u64)blockIdx.x * CB_THREADS + threadIdx.x;
    if (i >= A.n) return;
    CBatchFrame* F = A.F + i;
    if (!F->live) return;
    u64 body = 0, off0 = 0;
    if (F->nb) {
        const u64 j0 = A.first[i], j1 = j0 + F->nb - 1;
        off0 = A.offs[j0];
        body = A.offs[j1] + A.sizes[j1] - off0;
    }
    F->body = body;
    F->off0 = off0;
    F->fits = F->fixed + body <= F->cap;
}

/* zxc_asm_blocks per block of the batch; every entry in [nb, nb_max) gets size 0 for the compaction */
__global__ void __launch_bounds__(CB_THREADS) zxc_cbatch_blocks(const CBatchArgs A) {
    const u64 nb = A.st->nb;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < A.nb_max; j += stride) {
        if (j >= nb) {
            A.sizes[j] = 0;
            continue;
        }
        const u32 f = cb_frame_of(A, j);
        CBatchFrame* F = A.F + f;
        if (!F->fits) {
            A.sizes[j] = 0;
            continue;
        }
        const u64 jl = j - A.first[f];
        const u32 sz = A.sizes[j];
        u8* body = F->dst + ZXC_FILE_HEADER_SIZE;
        A.offs[j] = (unsigned long long)(uintptr_t)(body + (A.offs[j] - F->off0));
        if (A.seekable) asm_st32(body + F->body + 2 * ZXF_BLOCK_HDR + 4 * jl, sz);
        if (A.checksum) {
            const u8* c = A.staging + j * A.staging_stride + sz - 4;
            const u32 cj = (u32)c[0] | ((u32)c[1] << 8) | ((u32)c[2] << 16) | ((u32)c[3] << 24);
            const u32 r = (u32)((F->nb - 1 - jl) & 31u);
            const u32 h = r ? (cj << r) | (cj >> (32 - r)) : cj;
            if (h) atomicXor(&F->hash, h);
        }
    }
}

/* zxc_asm_finish per frame */
__global__ void __launch_bounds__(CB_THREADS) zxc_cbatch_finish(const CBatchArgs A) {
    const u64 i = (u64)blockIdx.x * CB_THREADS + threadIdx.x;
    if (i >= A.n) return;
    const CBatchFrame* F = A.F + i;
    if (!F->live) return;
    if (!F->fits) {
        A.results[i] = ZXC_ERROR_DST_TOO_SMALL;
        return;
    }
    u8* dst = F->dst;
#pragma unroll
    for (int k = 0; k < 16; k++) dst[k] = A.header[k];
    u8* p = dst + ZXC_FILE_HEADER_SIZE + F->body;
#pragma unroll
    for (int k = 0; k < 8; k++) p[k] = A.eof[k];
    p += ZXF_BLOCK_HDR;
    if (A.seekable && F->nb) {
        put_block_header(p, ZXF_BT_SEK, F->nb * ZXF_SEEK_ENTRY);
        p += ZXF_BLOCK_HDR + (u64)ZXF_SEEK_ENTRY * F->nb;
    }
#pragma unroll
    for (int k = 0; k < 8; k++) p[k] = (u8)(F->src_size >> (8 * k));
    asm_st32(p + 8, A.checksum ? F->hash : 0u);
    A.results[i] = (long long)(F->fixed + F->body);
}
