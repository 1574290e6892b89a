/*
 * zxc_pstream_device.cuh -- the kernels of the push streams in HBM (zxc_b200_cstream_device / _dstream_device,
 * driven by zxc_pstream.c through the zxg_ps_* calls of zxc_gpu.cu).
 *
 *   zxc_ps_walk       one thread: the dstream's batch walk from in->pos -- each block's 8-byte header, its on-disk
 *                     length and its checksum trailer -- stopping where the host walk of ds_decode_batch stops
 *   zxc_ps_trailers   the cstream's per-block checksum trailers, read from the encode's staging slots next to their
 *                     sizes, so that one copy brings both back
 *   zxc_ps_gather     the copies a call makes into `out`, as one launch over a table of pieces
 *
 * Bytes of `in` are read byte by byte (dp_block_header, ld32): chunks may have any alignment and nothing outside
 * in->src[0 .. size) is read.
 */
#pragma once
#include <cuda_runtime.h>

#include "zxc_dplan.cuh"
#include "zxc_gpu.h"

/* one entry of the walk: a data block whose bytes are all in the chunk (len > 0), or the header the walk stopped at
 * (len 0: EOF, a header the state machine rejects, or a block that runs past the chunk) */
static_assert(sizeof(zxg_psblk_t) == 24, "zxg_psblk_t layout");

__global__ void zxc_ps_walk(const u8* __restrict__ s, const u64 size, const u32 max_blocks, const u64 bound,
                            const u32 has_checksum, zxg_psblk_t* __restrict__ out, u32* __restrict__ n_out) {
    if (threadIdx.x != 0) return;
    const u32 trailer = has_checksum ? ZXF_BLOCK_CKS : 0u;
    u64 p = 0;
    u32 n = 0;
    while (n <= max_blocks && size - p >= ZXF_BLOCK_HDR) {
        zxg_psblk_t e;
        e.off = p;
        e.hdr = ld64(s + p);
        e.len = 0;
        e.trailer = 0;
        u32 type, comp;
        const bool ok = dp_block_header(s + p, &type, &comp);
        const u64 need = (u64)comp + trailer;
        /* ds_block_header's verdicts: a bad header, EOF, or a size above the bound end the walk; so does a block that
         * is not whole in the chunk, and the block after the batch's last */
        const bool whole = ok && type != ZXF_BT_EOF && need <= bound && size - p - ZXF_BLOCK_HDR >= need && n < max_blocks;
        if (whole) {
            e.len = (u32)(ZXF_BLOCK_HDR + need);
            if (trailer && need >= ZXF_BLOCK_CKS) e.trailer = ld32(s + p + ZXF_BLOCK_HDR + need - ZXF_BLOCK_CKS);
        }
        out[n++] = e;
        if (!whole) break;
        p += e.len;
    }
    *n_out = n;
}

/* trail[i] = the last 4 bytes of encoded block i (its checksum trailer when checksums are on) */
__global__ void zxc_ps_trailers(const u8* __restrict__ stage, const u32 sstride, const u32* __restrict__ sizes,
                                u32* __restrict__ trail, const u32 n) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u32 c = sizes[i];
    trail[i] = c >= ZXF_BLOCK_CKS ? ld32(stage + (size_t)i * sstride + c - ZXF_BLOCK_CKS) : 0u;
}

/* One CTA per piece (grid-stride): 16-byte vectors when source and destination share their alignment, else bytes.
 * Pieces are at most ZXG_PS_PIECE bytes, cut on the host, so that a few large blocks still spread over the SMs. */
__global__ void __launch_bounds__(256) zxc_ps_gather(const zxg_psseg_t* __restrict__ segs, const u32 n) {
    for (u32 k = blockIdx.x; k < n; k += gridDim.x) {
        const zxg_psseg_t g = segs[k];
        const u8* src = (const u8*)g.src;
        u8* dst = (u8*)g.dst;
        u64 len = g.len;
        if (((g.src ^ g.dst) & 15u) == 0) {
            const u64 head = ((16u - (g.dst & 15u)) & 15u) < len ? ((16u - (g.dst & 15u)) & 15u) : len;
            if (threadIdx.x < head) dst[threadIdx.x] = src[threadIdx.x];
            src += head;
            dst += head;
            len -= head;
            const u64 nv = len >> 4;
            const uint4* vs = (const uint4*)src;
            uint4* vd = (uint4*)dst;
            for (u64 i = threadIdx.x; i < nv; i += blockDim.x) vd[i] = vs[i];
            const u64 tail = len & 15u;
            if (threadIdx.x < tail) dst[(nv << 4) + threadIdx.x] = src[(nv << 4) + threadIdx.x];
        } else {
            for (u64 i = threadIdx.x; i < len; i += blockDim.x) dst[i] = src[i];
        }
    }
}
