/*
 * zxc_pstream_device.cuh -- the kernels of the push streams in HBM (zxc_b200_cstream_device / _dstream_device,
 * driven by zxc_pstream.c through the zxg_ps_* calls of zxc_gpu.cu).
 *
 *   zxc_ps_walk       one thread: the dstream's batch walk from in->pos -- each block's 8-byte header, its on-disk
 *                     length and its checksum trailer -- stopping where the host walk of ds_decode_batch stops
 *   zxc_ps_trailers   the cstream's per-block checksum trailers, read from the encode's staging slots next to their
 *                     sizes, so that one copy brings both back
 *   zxc_ps_gather     the copies a call makes into `out`, as one launch over a table of pieces; the dictionary
 *                     trainers pack device-resident samples with it too (zxc_gpu.cu, d2d_gather)
 *
 * Bytes of `in` are read byte by byte by the walk (dp_block_header, ld32): chunks may have any alignment and nothing
 * outside in->src[0 .. size) is read.  The gather reads nothing outside its pieces' sources.
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

/* bytes Q * 4 + sh / 8 .. + 15 of the 32 bytes (a, b): the 16 source bytes behind one aligned destination vector */
template <int Q>
__device__ __forceinline__ uint4 ps_funnel(const uint4 a, const uint4 b, const u32 sh) {
    const u32 w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    return make_uint4(__funnelshift_r(w[Q], w[Q + 1], sh), __funnelshift_r(w[Q + 1], w[Q + 2], sh),
                      __funnelshift_r(w[Q + 2], w[Q + 3], sh), __funnelshift_r(w[Q + 3], w[Q + 4], sh));
}

/* vd[i] = the 16 bytes at byte 4Q + sh / 8 of (vs[i], vs[i + 1]), for i in [lo, hi) */
template <int Q>
__device__ __forceinline__ void ps_copy_shifted(const uint4* __restrict__ vs, uint4* __restrict__ vd, const u32 lo,
                                                const u32 hi, const u32 sh) {
    for (u32 i = lo + threadIdx.x; i < hi; i += blockDim.x) vd[i] = ps_funnel<Q>(vs[i], vs[i + 1], sh);
}

/* One CTA per piece (grid-stride).  Pieces are at most ZXG_PS_PIECE bytes, cut on the host, so that a few large blocks
 * still spread over the SMs.  The destination is written as aligned 16-byte vectors between byte-wise edges:
 *   - source and destination share their alignment: one aligned 16-byte load per vector;
 *   - they do not: each vector is funnel-shifted out of the two aligned source vectors it straddles, and only the
 *     vectors whose two loads lie wholly inside src[0 .. len) go this way, so nothing outside the piece is read;
 *   - src == 0: zeros. */
__global__ void __launch_bounds__(256) zxc_ps_gather(const zxg_psseg_t* __restrict__ segs, const u32 n) {
    for (u32 k = blockIdx.x; k < n; k += gridDim.x) {
        const zxg_psseg_t g = segs[k];
        const u8* src = (const u8*)g.src;
        u8* dst = (u8*)g.dst;
        const u32 len = (u32)g.len;
        const u32 head = min((16u - (u32)(g.dst & 15u)) & 15u, len);
        uint4* vd = (uint4*)(dst + head);
        u32 lo = 0, hi = (len - head) >> 4; /* destination vectors [lo, hi) at dst + head */
        if (g.src == 0) {
            for (u32 i = threadIdx.x; i < hi; i += blockDim.x) vd[i] = make_uint4(0u, 0u, 0u, 0u);
        } else if (((g.src ^ g.dst) & 15u) == 0) {
            const uint4* vs = (const uint4*)(src + head);
            for (u32 i = threadIdx.x; i < hi; i += blockDim.x) vd[i] = vs[i];
        } else {
            /* vector i reads the aligned source vectors i and i + 1 from a: the first lies before src when a < src,
             * and there are (len - head + r) / 16 of them before src + len */
            const u32 r = (u32)((g.src + head) & 15u);
            const u8* a = src + head - r;
            const u32 n_src = (len - head + r) >> 4;
            lo = a < src ? min(1u, hi) : 0u;
            hi = max(min(hi, n_src > 0 ? n_src - 1u : 0u), lo);
            const uint4* vs = (const uint4*)a;
            const u32 sh = (r & 3u) * 8u;
            switch (r >> 2) {
                case 0: ps_copy_shifted<0>(vs, vd, lo, hi, sh); break;
                case 1: ps_copy_shifted<1>(vs, vd, lo, hi, sh); break;
                case 2: ps_copy_shifted<2>(vs, vd, lo, hi, sh); break;
                default: ps_copy_shifted<3>(vs, vd, lo, hi, sh); break;
            }
        }
        /* the edges byte by byte: [0, e0) and [e1, len) */
        const u32 e0 = head + 16u * lo, e1 = head + 16u * hi;
        for (u32 t = threadIdx.x; t < e0 + (len - e1); t += blockDim.x) {
            const u32 j = t < e0 ? t : e1 + (t - e0);
            dst[j] = src ? src[j] : (u8)0;
        }
    }
}
