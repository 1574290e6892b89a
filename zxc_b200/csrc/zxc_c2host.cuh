/*
 * zxc_c2host.cuh -- compress a device buffer into a frame in page-locked host memory, window by window
 * (zxc_b200_compress_device_to_host).  Each round encodes W input bytes with the unchanged encode kernel and moves
 * the round's blocks straight into mapped host memory, so the device memory the call needs is bounded by W, not by
 * the input.  Stream order, per round:
 *
 *   (copy)              the window's input into the padded input region, device to device
 *   zxc_encode_kernel   the window's blocks into their staging slots
 *   zxc_asm_tile_sums   (zxc_assemble.cuh, unchanged) sum of each tile of ASM_TILE on-disk sizes
 *   zxc_c2h_scan        one CTA: exclusive scan of the tile sums; the round's body base and size, the running body
 *                       total and the running capacity verdict
 *   zxc_c2h_blocks      per block: window-relative body offset, SEK entry (into the scratch table, by global index)
 *                       and its term of the global hash (global index j of n blocks)
 *   zxc_c2h_write       the round's bytes into host memory as aligned 16-byte stores
 *
 * and after the last round zxc_c2h_finish writes the file header's first chunk, the carried tail, the EOF block, the
 * SEK header and table, the footer with the global hash, and the result.
 *
 * Host memory is written in aligned 16-byte chunks of the destination's address space.  A round writes every whole
 * chunk from the one holding its first body byte up to the one holding its last; that last chunk, when the round
 * does not end on a chunk boundary, is not stored but carried in the state, and the next round (or the finish)
 * stores it whole with the bytes that follow.  Chunk 0, which holds frame byte 0, is the finish's; when the
 * destination is misaligned it and the frame's last chunk are written with narrower stores, so nothing outside the
 * frame is touched.  A round whose running total no longer fits dst_capacity writes nothing, and neither does the
 * finish then: no byte outside h_dst[0 .. dst_capacity) is written in any case.
 */
#pragma once
#include <cuda_runtime.h>

#include "zxc_assemble.cuh"

#define C2H_THREADS 256

/* the first bytes of the caller's scratch */
struct C2hState {
    unsigned long long counter; /* the encode kernel's work counter */
    unsigned long long body;    /* body bytes of the rounds so far */
    unsigned long long wbase;   /* this round's first body byte */
    unsigned long long wtotal;  /* this round's body bytes */
    unsigned int hash;          /* global hash, XOR-accumulated by zxc_c2h_blocks */
    unsigned int over;          /* header + body so far + trailer > dst_capacity */
    /* carry[r & 1]: the frame bytes from the chunk holding body byte `body` (before round r) up to it */
    unsigned char carry[2][16];
};

typedef unsigned __int128 c2h_u128;

__device__ __forceinline__ c2h_u128 c2h_ld16(const unsigned char* p) {
    const uint4 v = *(const uint4*)p;
    return ((c2h_u128)(((unsigned long long)v.w << 32) | v.z) << 64) | (((unsigned long long)v.y << 32) | v.x);
}

/* The 16 bytes at aligned address a (an address in the mapped host range), of which only bytes [k0, k1) are
 * written: one 16-byte store when all of them are, else the widest aligned stores that cover [k0, k1). */
__device__ __forceinline__ void c2h_store(unsigned char* a, c2h_u128 v, unsigned int k0, unsigned int k1) {
    if (k0 == 0 && k1 == 16) {
        const unsigned long long lo = (unsigned long long)v, hi = (unsigned long long)(v >> 64);
        *(uint4*)a = make_uint4((unsigned int)lo, (unsigned int)(lo >> 32), (unsigned int)hi, (unsigned int)(hi >> 32));
        return;
    }
    unsigned int k = k0;
    while (k < k1) {
        const unsigned long long x = (unsigned long long)(v >> (8 * k));
        if ((k & 7) == 0 && k + 8 <= k1) {
            *(unsigned long long*)(a + k) = x;
            k += 8;
        } else if ((k & 3) == 0 && k + 4 <= k1) {
            *(unsigned int*)(a + k) = (unsigned int)x;
            k += 4;
        } else if ((k & 1) == 0 && k + 2 <= k1) {
            *(unsigned short*)(a + k) = (unsigned short)x;
            k += 2;
        } else {
            a[k] = (unsigned char)x;
            k += 1;
        }
    }
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_c2h_scan(unsigned long long* tile_sum, unsigned int n_tiles,
                                                                 C2hState* st, unsigned long long fixed,
                                                                 unsigned long long dst_capacity) {
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
        const unsigned long long base = st->body;
        st->wbase = base;
        st->wtotal = carry;
        st->body = base + carry;
        if (fixed + base + carry > dst_capacity) st->over = 1;
    }
}

/* j0: the round's first block, n: the frame's block count */
__global__ void __launch_bounds__(ASM_THREADS) zxc_c2h_blocks(const unsigned int* sizes, const unsigned char* staging,
                                                              const unsigned long long* tile_off,
                                                              unsigned long long* offs, C2hState* st,
                                                              unsigned int* sek, unsigned int wn, unsigned int j0,
                                                              unsigned int n, unsigned int staging_stride,
                                                              unsigned int checksum) {
    const unsigned long long base = (unsigned long long)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    unsigned int sz[ASM_ITEMS];
    unsigned long long s = 0;
#pragma unroll
    for (unsigned int k = 0; k < ASM_ITEMS; k++) {
        sz[k] = base + k < wn ? sizes[base + k] : 0u;
        s += sz[k];
    }
    unsigned long long total;
    unsigned long long off = tile_off[blockIdx.x] + asm_cta_excl(s, &total);
    unsigned int h = 0;
#pragma unroll
    for (unsigned int k = 0; k < ASM_ITEMS; k++) {
        const unsigned long long j = base + k;
        if (j >= wn) break;
        offs[j] = off;
        const unsigned int g = j0 + (unsigned int)j;
        if (sek) sek[g] = sz[k];
        if (checksum) {
            const unsigned char* c = staging + j * staging_stride + sz[k] - 4;
            const unsigned int cj = (unsigned int)c[0] | ((unsigned int)c[1] << 8) | ((unsigned int)c[2] << 16) |
                                    ((unsigned int)c[3] << 24);
            const unsigned int r = (n - 1 - g) & 31u;
            h ^= r ? (cj << r) | (cj >> (32 - r)) : cj;
        }
        off += sz[k];
    }
    for (unsigned int d = 16; d; d >>= 1) h ^= __shfl_xor_sync(0xFFFFFFFFu, h, d);
    if ((threadIdx.x & 31) == 0 && h) atomicXor(&st->hash, h);
}

/* The frame's file header, as kernel parameter bytes (the carry holds it too once a round has passed it) */
struct C2hHeader {
    unsigned char b[16];
};

/* Grid-stride over the round's chunks.  Chunk i holds frame bytes [q0 + 16 i, q0 + 16 i + 16), q0 being the first
 * byte of the chunk that holds body byte wbase.  Its bytes before the round's body come from the carry (and the file
 * header); the rest from the staging slots, each piece funnel-shifted out of the two aligned 16-byte loads it
 * straddles in its slot (slots are 256-aligned and end at least 16 bytes past their block, so those loads stay in
 * the slot).  The block of a byte is found by binary search over the round's scanned offsets. */
__global__ void __launch_bounds__(C2H_THREADS) zxc_c2h_write(unsigned char* hd, const unsigned char* staging,
                                                             unsigned int staging_stride,
                                                             const unsigned long long* offs, const unsigned int* sizes,
                                                             unsigned int wn, C2hState* st, const C2hHeader H,
                                                             unsigned int parity) {
    __shared__ unsigned char s_hdr[16]; /* read by byte index: a parameter array would go through a stack copy */
    if (threadIdx.x == 0) {
#pragma unroll
        for (unsigned int k = 0; k < 16; k++) s_hdr[k] = H.b[k];
    }
    __syncthreads();
    if (st->over) return;
    const unsigned long long a = 16 + st->wbase, q1 = a + st->wtotal;
    const unsigned long long hb = (unsigned long long)hd;
    const unsigned long long q0 = ((hb + a) & ~15ull) - hb;
    const unsigned long long nc = (q1 - q0 + 15) >> 4;
    const unsigned char* cin = st->carry[parity];
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < nc;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long p = q0 + 16 * i;
        const unsigned long long lim = p + 16 < q1 ? p + 16 : q1;
        c2h_u128 v = 0;
        unsigned long long cur = p;
        for (; cur < a && cur < lim; cur++) /* chunk 0 only: the carried bytes */
            v |= (c2h_u128)(cur < 16 ? s_hdr[cur] : cin[cur - q0]) << (8 * (cur - p));
        if (cur < lim) {
            const unsigned long long rel = cur - a;
            unsigned int lo = 0, hi = wn; /* the last block whose offset is <= rel */
            while (hi - lo > 1) {
                const unsigned int mid = (lo + hi) >> 1;
                if (offs[mid] <= rel) lo = mid;
                else hi = mid;
            }
            for (unsigned int j = lo; cur < lim; j++) {
                const unsigned long long bo = a + offs[j], be = bo + sizes[j];
                const unsigned long long e = be < lim ? be : lim;
                const unsigned int len = (unsigned int)(e - cur);
                const unsigned char* s = staging + (unsigned long long)j * staging_stride + (cur - bo);
                const unsigned int sh = (unsigned int)((unsigned long long)s & 15);
                const unsigned char* al = s - sh;
                c2h_u128 w = c2h_ld16(al) >> (8 * sh);
                if (sh + len > 16) w |= c2h_ld16(al + 16) << (128 - 8 * sh);
                if (len < 16) w &= ((c2h_u128)1 << (8 * len)) - 1;
                v |= w << (8 * (cur - p));
                cur = e;
            }
        }
        if (lim == p + 16) {
            c2h_store(hd + p, v, 0, 16);
        } else { /* the round's last, partial chunk: carried to the next round or the finish */
            unsigned char* cout = st->carry[parity ^ 1];
            for (unsigned int k = 0; k < 16; k++) cout[k] = (unsigned char)(v >> (8 * k));
        }
    }
}

/* What the finish writes, passed by value */
struct C2hFinish {
    unsigned char header[16];
    unsigned char eof[8];
    unsigned char sek[8];     /* SEK block header, when `seekable` */
    unsigned char footer[12]; /* decoded size; the hash field is written here when `checksum` */
    unsigned long long dst_capacity;
    unsigned long long fixed; /* file header + trailer */
    unsigned int n_blocks;
    unsigned int checksum;
    unsigned int seekable;
    unsigned int parity; /* rounds & 1: the carry the last round left */
};

/* Grid-stride over chunk 0 (frame bytes from 0 up to the first chunk boundary past byte 0) and the chunks from the
 * carried tail to the frame's end; thread 0 of CTA 0 writes the result.  Nothing but the result when the frame does
 * not fit dst_capacity. */
__global__ void __launch_bounds__(C2H_THREADS) zxc_c2h_finish(unsigned char* hd, const unsigned char* sek_table,
                                                              const C2hState* st, const C2hFinish F,
                                                              long long* result) {
    /* the fixed bytes, read by byte index: header | EOF | SEK header | footer */
    __shared__ unsigned char s_fix[44];
    if (threadIdx.x == 0) {
#pragma unroll
        for (unsigned int k = 0; k < 16; k++) s_fix[k] = F.header[k];
#pragma unroll
        for (unsigned int k = 0; k < 8; k++) s_fix[16 + k] = F.eof[k];
#pragma unroll
        for (unsigned int k = 0; k < 8; k++) s_fix[24 + k] = F.sek[k];
#pragma unroll
        for (unsigned int k = 0; k < 12; k++) s_fix[32 + k] = F.footer[k];
    }
    __syncthreads();
    const unsigned long long body = st->body;
    const unsigned long long end = F.fixed + body;
    const bool fits = !st->over && end <= F.dst_capacity;
    if (blockIdx.x == 0 && threadIdx.x == 0) *result = fits ? (long long)end : (long long)ZXC_ERROR_DST_TOO_SMALL;
    if (!fits) return;
    const long long hb = (long long)(unsigned long long)hd;
    const long long c0 = (hb & ~15ll) - hb;                      /* chunk 0's first byte: -15 .. 0 */
    const long long a = 16 + (long long)body;                     /* the trailer's first byte */
    const long long qt = ((hb + a) & ~15ll) - hb;                 /* the carried tail's first byte */
    const unsigned long long nt = ((unsigned long long)end - qt + 15) >> 4;
    const unsigned char* cin = st->carry[F.parity];
    const long long sek_end = F.seekable ? 8 + 4ll * F.n_blocks : 0; /* SEK header and table, behind the EOF block */
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < nt + 1;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const long long p = i == 0 ? c0 : qt + 16 * (long long)(i - 1);
        const unsigned int k0 = p < 0 ? (unsigned int)-p : 0u;
        const unsigned int k1 = p + 16 <= (long long)end ? 16u : (unsigned int)((long long)end - p);
        c2h_u128 v = 0;
        for (unsigned int k = k0; k < k1; k++) {
            const long long q = p + k;
            unsigned int b;
            if (q < 16) {
                b = s_fix[q];
            } else if (q < a) {
                b = cin[q - qt];
            } else {
                const long long t = q - a;
                if (t < 8) {
                    b = s_fix[16 + t];
                } else if (t < 8 + sek_end) {
                    const long long u = t - 8;
                    b = u < 8 ? s_fix[24 + u] : sek_table[u - 8];
                } else {
                    const long long f = t - 8 - sek_end;
                    b = F.checksum && f >= 8 ? (st->hash >> (8 * (f - 8))) & 0xFFu : s_fix[32 + f];
                }
            }
            v |= (c2h_u128)b << (8 * k);
        }
        c2h_store(hd + p, v, k0, k1);
    }
}
