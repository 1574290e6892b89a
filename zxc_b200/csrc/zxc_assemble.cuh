/*
 * zxc_assemble.cuh -- frame assembly on the device (zxc_b200_compress_device).  The encode kernel leaves one
 * staging slot per block and the block's on-disk size; these kernels turn that into the frame in the caller's
 * buffer with no host round trip, in this stream order:
 *
 *   zxc_asm_tile_sums   sum of the on-disk sizes of each tile of ASM_TILE blocks
 *   zxc_asm_scan_tiles  one CTA: exclusive scan of the tile sums, body size, capacity verdict
 *   zxc_asm_blocks      per block: body offset, decode-plan entry, SEK entry and its term of the global hash;
 *                       when the frame does not fit it zeroes the sizes instead, so the compaction copies nothing
 *   zxc_compact_kernel  (zxc_encode.cuh, unchanged) the blocks into place behind the file header
 *   zxc_asm_finish      file header, EOF block, SEK header, footer with the global hash, and the result
 *
 * The bytes of the file header, the EOF and SEK block headers and the footer are written on the host by the
 * zxc_format.c helpers and arrive here as kernel parameters (AsmFrame), so the wire format stays in one place.
 *
 * Global hash: the host folds h = rotl(h, 1) ^ c_j over the block checksums in order (zxf_hash_combine), which
 * equals XOR_j rotl(c_j, (n - 1 - j) mod 32); every block contributes its term independently and the terms
 * meet in one atomicXor word.
 */
#pragma once
#include <cuda_runtime.h>

#include "zxc_b200.h"
#include "zxc_error.h"

#define ASM_THREADS 256
#define ASM_ITEMS 8
#define ASM_TILE (ASM_THREADS * ASM_ITEMS) /* blocks per CTA of zxc_asm_tile_sums / zxc_asm_blocks */
#define ASM_SCAN_THREADS 1024

/* the first bytes of the caller's scratch */
struct AsmState {
    unsigned long long counter; /* the encode kernel's work counter */
    unsigned long long body;    /* body bytes (zxc_asm_scan_tiles) */
    unsigned int hash;          /* global hash, XOR-accumulated by zxc_asm_blocks */
    unsigned int fits;          /* header + body + trailer <= dst_capacity */
};

/* host-computed bytes and sizes, passed by value */
struct AsmFrame {
    unsigned char header[16];
    unsigned char eof[8];
    unsigned char sek[8];    /* SEK block header, when `seekable` */
    unsigned char footer[12]; /* decoded size; the hash field is written here when `checksum` */
    unsigned long long src_size;
    unsigned long long dst_capacity;
    unsigned long long fixed; /* file header + trailer: every byte of the frame but the body */
    unsigned int n_blocks;
    unsigned int block_size;
    unsigned int staging_stride;
    unsigned int checksum;
    unsigned int seekable; /* a SEK table follows the EOF block (seekable frames with at least one block) */
};

__device__ __forceinline__ unsigned long long asm_warp_incl(unsigned long long v, unsigned int lane) {
    for (unsigned int d = 1; d < 32; d <<= 1) {
        const unsigned long long t = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if (lane >= d) v += t;
    }
    return v;
}

/* exclusive prefix sum of v over the CTA (blockDim.x a multiple of 32); *total = the CTA's sum.  Every thread
 * calls it; it may be called again right away (the trailing barrier frees the shared words). */
__device__ __forceinline__ unsigned long long asm_cta_excl(unsigned long long v, unsigned long long* total) {
    __shared__ unsigned long long s_warp[32];
    __shared__ unsigned long long s_total;
    const unsigned int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const unsigned long long inc = asm_warp_incl(v, lane);
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    if (w == 0) {
        const unsigned long long x = lane < nw ? s_warp[lane] : 0;
        const unsigned long long xi = asm_warp_incl(x, lane);
        if (lane < nw) s_warp[lane] = xi - x;
        if (lane == 31) s_total = xi;
    }
    __syncthreads();
    const unsigned long long r = s_warp[w] + inc - v;
    *total = s_total;
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(ASM_THREADS) zxc_asm_tile_sums(const unsigned int* sizes, unsigned int n,
                                                                 unsigned long long* tile_sum) {
    const unsigned long long base = (unsigned long long)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    unsigned long long s = 0;
#pragma unroll
    for (unsigned int k = 0; k < ASM_ITEMS; k++)
        if (base + k < n) s += sizes[base + k];
    unsigned long long total;
    asm_cta_excl(s, &total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_asm_scan_tiles(unsigned long long* tile_sum,
                                                                       unsigned int n_tiles, AsmState* st,
                                                                       const AsmFrame F) {
    unsigned long long carry = 0;
    for (unsigned int b = 0; b < n_tiles; b += blockDim.x) {
        const unsigned int i = b + threadIdx.x;
        const unsigned long long v = i < n_tiles ? tile_sum[i] : 0;
        unsigned long long total;
        const unsigned long long ex = asm_cta_excl(v, &total);
        if (i < n_tiles) tile_sum[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) {
        st->body = carry;
        st->fits = F.fixed + carry <= F.dst_capacity ? 1u : 0u;
        st->hash = 0;
    }
}

__device__ __forceinline__ void asm_st32(unsigned char* p, unsigned int v) {
    p[0] = (unsigned char)v;
    p[1] = (unsigned char)(v >> 8);
    p[2] = (unsigned char)(v >> 16);
    p[3] = (unsigned char)(v >> 24);
}

__global__ void __launch_bounds__(ASM_THREADS) zxc_asm_blocks(unsigned int* sizes, const unsigned char* staging,
                                                              const unsigned long long* tile_off,
                                                              unsigned long long* offs, AsmState* st,
                                                              zxc_b200_job_t* jobs, unsigned char* dst,
                                                              const AsmFrame F) {
    const unsigned int n = F.n_blocks;
    const unsigned long long base = (unsigned long long)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    unsigned int sz[ASM_ITEMS];
    unsigned long long s = 0;
#pragma unroll
    for (unsigned int k = 0; k < ASM_ITEMS; k++) {
        sz[k] = base + k < n ? sizes[base + k] : 0u;
        s += sz[k];
    }
    unsigned long long total;
    unsigned long long off = tile_off[blockIdx.x] + asm_cta_excl(s, &total);
    const bool fits = st->fits != 0;
    unsigned char* sek = dst + 16 + st->body + 16; /* behind the EOF block and the SEK block header */
    unsigned int h = 0;
#pragma unroll
    for (unsigned int k = 0; k < ASM_ITEMS; k++) {
        const unsigned long long j = base + k;
        if (j >= n) break;
        offs[j] = off;
        if (jobs) {
            const unsigned long long d0 = j * F.block_size;
            const unsigned long long left = F.src_size - d0;
            zxc_b200_job_t J;
            J.src_off = 16 + off;
            J.dst_off = d0;
            J.src_len = sz[k];
            J.dst_cap = left < F.block_size ? (unsigned int)left : F.block_size;
            jobs[j] = J;
        }
        if (fits) {
            if (F.seekable) asm_st32(sek + 4 * j, sz[k]);
            if (F.checksum) {
                const unsigned char* c = staging + j * F.staging_stride + sz[k] - 4;
                const unsigned int cj = (unsigned int)c[0] | ((unsigned int)c[1] << 8) | ((unsigned int)c[2] << 16) |
                                        ((unsigned int)c[3] << 24);
                const unsigned int r = (unsigned int)((n - 1 - j) & 31u);
                h ^= r ? (cj << r) | (cj >> (32 - r)) : cj;
            }
        } else {
            sizes[j] = 0; /* the compaction then copies nothing */
        }
        off += sz[k];
    }
    for (unsigned int d = 16; d; d >>= 1) h ^= __shfl_xor_sync(0xFFFFFFFFu, h, d);
    if ((threadIdx.x & 31) == 0 && h) atomicXor(&st->hash, h);
}

/* one thread: 44 bytes at most */
__global__ void zxc_asm_finish(unsigned char* dst, const AsmState* st, const AsmFrame F, long long* result) {
    const unsigned long long body = F.n_blocks ? st->body : 0;
    if (F.fixed + body > F.dst_capacity) {
        *result = ZXC_ERROR_DST_TOO_SMALL;
        return;
    }
#pragma unroll
    for (int k = 0; k < 16; k++) dst[k] = F.header[k];
    unsigned char* p = dst + 16 + body;
#pragma unroll
    for (int k = 0; k < 8; k++) p[k] = F.eof[k];
    p += 8;
    if (F.seekable) {
#pragma unroll
        for (int k = 0; k < 8; k++) p[k] = F.sek[k];
        p += 8 + 4ull * F.n_blocks;
    }
#pragma unroll
    for (int k = 0; k < 12; k++) p[k] = F.footer[k];
    if (F.checksum) asm_st32(p + 8, F.n_blocks ? st->hash : 0u);
    *result = (long long)(F.fixed + body);
}
