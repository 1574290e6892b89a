/*
 * zxc_train.cuh -- dictionary training on sm_90a (device code only): the content trainer's k-gram count, candidate
 * segments, greedy pick and emission, and the literal histogram of the shared-table trainer.  The host side (argument
 * checks, the heap order of the segments, code lengths) is zxc_train.c; the launches are in zxc_gpu.cu.
 *
 * Behaviour restated (file:line in /root/reference/src/lib/zxc_dict.c):
 *   k-gram hash, frequency count          :231-235, :341-350
 *   candidate segments                    :352-390
 *   greedy pick against the live table    :402-435
 *   reverse emission                      :439-448
 *   literal histogram of level-6 parses   :490-549 (zxc_compress.c:1263-1268, reached through parse_done)
 *
 * Kernels:
 *   zxc_train_count_kernel    one thread per sampled position, u32 atomics (clamped to 65535 where the table is read:
 *                             the reference's saturating u16 counter gives the same value in any order)
 *   zxc_train_seg_kernel      one warp per segment start, the clamped table (128 KiB) in shared memory; each step
 *                             looks up 32 consecutive k-grams and a ballot finds the first infrequent one
 *   zxc_train_compact_kernel  one CTA: keeps the first seg_alloc valid starts in position order (scan)
 *   zxc_train_hash_kernel     one warp per segment, in the host's pick order: the k-gram hashes of every segment,
 *                             packed back to back, so the pick streams 2 bytes per k-gram
 *   zxc_train_pick_kernel     one CTA, the table in shared memory: the hash stream is staged in chunks and warp 0
 *                             walks the segments in order (re-score, skip or zero + record)
 *   zxc_train_emit_kernel     one warp per pick: copies it to its place in the reversed output
 *   zxc_train_lit_kernel      the level-6 parse of [dict | slice], one warp per slice, as zxc_encode_kernel<true>
 *                             runs it; the literals it leaves go into a per-warp histogram, flushed with atomics
 */
#pragma once
#include "zxc_encode.cuh"

#define TRN_K 5u                /* k-gram length (the format's minimum match) */
#define TRN_HASH_SIZE 65536u    /* 16-bit k-gram hash */
#define TRN_SEG_SPAN 4096u      /* a segment stops growing once it spans this many bytes */
#define TRN_CTA 1024u
#define TRN_CHUNK 16384u        /* k-gram hashes staged per step of the pick */
#define TRN_SEG_SMEM (TRN_HASH_SIZE * 2u)
#define TRN_PICK_SMEM (TRN_HASH_SIZE * 2u + TRN_CHUNK * 2u)

/* one candidate segment: corpus offset (32-bit, as the reference keeps it), length (0: no segment), coverage score */
struct TrainSeg {
    u32 offset, len, score;
};
/* one pick: corpus offset, bytes copied, bytes picked before it */
struct TrainPick {
    u32 offset, copy, before;
};

/* (le32(p) ^ p[4]) * 0x2D35182D >> 16 */
__device__ __forceinline__ u32 trn_hash(const u8* p) {
    const u32 v = (u32)p[0] | ((u32)p[1] << 8) | ((u32)p[2] << 16) | ((u32)p[3] << 24);
    return ((v ^ (u32)p[4]) * 0x2D35182Du) >> 16;
}

/* the u32 counts as the reference's saturating u16 table, into shared memory */
__device__ __forceinline__ void trn_load_table(unsigned short* t, const u32* freq) {
    for (u32 h = threadIdx.x; h < TRN_HASH_SIZE; h += blockDim.x) t[h] = (unsigned short)min(freq[h], 65535u);
    __syncthreads();
}

__global__ void zxc_train_count_kernel(const u8* corpus, unsigned long long kgram_limit, unsigned long long stride,
                                       u32* freq) {
    const unsigned long long n = (kgram_limit + stride - 1) / stride;
    for (unsigned long long k = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; k < n;
         k += (unsigned long long)gridDim.x * blockDim.x)
        atomicAdd(&freq[trn_hash(corpus + k * stride)], 1u);
}

/* start s is corpus position s * stride (all of them satisfy pos + 5 <= corpus_size) */
__global__ void __launch_bounds__(TRN_CTA, 1) zxc_train_seg_kernel(const u8* corpus, unsigned long long corpus_size,
                                                                  unsigned long long stride, u32 n_starts, const u32* freq,
                                                                  TrainSeg* seg) {
    extern __shared__ __align__(128) unsigned short s_freq[]; /* 128: the shared layout this kernel has always had */
    trn_load_table(s_freq, freq);
    const u32 lane = threadIdx.x & 31;
    const u32 nwarps = gridDim.x * (blockDim.x >> 5);
    for (u32 s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < n_starts; s += nwarps) {
        const unsigned long long i = (unsigned long long)s * stride;
        const u32 f = s_freq[trn_hash(corpus + i)];
        TrainSeg r = {(u32)i, 0u, 0u};
        if (f >= 2) {
            u32 cov = f, m = 1; /* k-grams taken: the segment is [i, i + 5m) */
            for (;;) {
                const u32 t = m + lane; /* the k-gram at i + 5t extends the segment when it is frequent */
                const unsigned long long e = i + (unsigned long long)TRN_K * t;
                u32 nf = 0;
                bool ok = false;
                if (TRN_K * t < TRN_SEG_SPAN && e + TRN_K <= corpus_size) {
                    nf = s_freq[trn_hash(corpus + e)];
                    ok = nf >= 2;
                }
                const u32 stop = __ballot_sync(FULL, !ok);
                const u32 take = stop ? (u32)(__ffs(stop) - 1) : 32u;
                u32 v = lane < take ? nf : 0u;
#pragma unroll
                for (int d = 16; d >= 1; d >>= 1) v += __shfl_xor_sync(FULL, v, d);
                cov += v;
                m += take;
                if (stop) break;
            }
            r.len = TRN_K * m;
            r.score = cov;
        }
        if (lane == 0) seg[s] = r;
    }
}

/* first seg_alloc starts with a segment, in position order */
__global__ void __launch_bounds__(TRN_CTA) zxc_train_compact_kernel(const TrainSeg* all, u32 n_starts, u32 seg_alloc,
                                                                    TrainSeg* out, u32* n_out) {
    __shared__ u32 s_cnt[TRN_CTA];
    const u32 t = threadIdx.x;
    const u32 per = (n_starts + blockDim.x - 1) / blockDim.x;
    const u32 lo = min(t * per, n_starts), hi = min(lo + per, n_starts);
    u32 c = 0;
    for (u32 s = lo; s < hi; s++) c += all[s].len != 0;
    s_cnt[t] = c;
    __syncthreads();
    for (u32 d = 1; d < blockDim.x; d <<= 1) {
        const u32 v = t >= d ? s_cnt[t - d] : 0u;
        __syncthreads();
        s_cnt[t] += v;
        __syncthreads();
    }
    u32 o = s_cnt[t] - c;
    for (u32 s = lo; s < hi && o < seg_alloc; s++)
        if (all[s].len) out[o++] = all[s];
    if (t == blockDim.x - 1) *n_out = min(s_cnt[t], seg_alloc);
}

/* hashes of segment j's k-grams at hoff[j] ..: len / 5 of them, read at its (32-bit) offset */
__global__ void zxc_train_hash_kernel(const u8* corpus, const TrainSeg* seg, const u32* hoff, u32 n_segs,
                                      unsigned short* hashes) {
    const u32 lane = threadIdx.x & 31;
    const u32 nwarps = (gridDim.x * blockDim.x) >> 5;
    for (u32 j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n_segs; j += nwarps) {
        const u32 nk = seg[j].len / TRN_K;
        const u8* p = corpus + seg[j].offset;
        unsigned short* h = hashes + hoff[j];
        for (u32 t = lane; t < nk; t += 32) h[t] = (unsigned short)trn_hash(p + (size_t)TRN_K * t);
    }
}

/* The greedy pick: segments in order, chunk c covering segments [chunk_first[c], chunk_first[c + 1]).  res[0] = picks,
 * res[1] = bytes picked. */
__global__ void __launch_bounds__(TRN_CTA, 1) zxc_train_pick_kernel(const TrainSeg* seg, const u32* hoff,
                                                                   const unsigned short* hashes, const u32* chunk_first,
                                                                   u32 n_chunks, const u32* freq, u32 capacity,
                                                                   TrainPick* picks, u32* res) {
    extern __shared__ __align__(128) unsigned short s_freq[]; /* 128: the shared layout this kernel has always had */
    unsigned short* s_h = s_freq + TRN_HASH_SIZE;
    __shared__ u32 s_state[2]; /* picks, total */
    trn_load_table(s_freq, freq);
    if (threadIdx.x == 0) s_state[0] = s_state[1] = 0;
    __syncthreads();
    const u32 lane = threadIdx.x & 31;
    for (u32 c = 0; c < n_chunks; c++) {
        if (s_state[1] >= capacity) break; /* uniform: written by warp 0 before the last barrier */
        const u32 s0 = chunk_first[c], s1 = chunk_first[c + 1];
        const u32 base = hoff[s0], len = hoff[s1] - base;
        for (u32 k = threadIdx.x; k < len; k += blockDim.x) s_h[k] = hashes[base + k];
        __syncthreads();
        if (threadIdx.x < 32) {
            u32 n_sel = s_state[0], total = s_state[1];
            for (u32 g = s0; g < s1 && total < capacity; g += 32) {
                /* 32 records at a time, handed out by shuffles */
                TrainSeg mine = {0u, 0u, 0u};
                u32 my_h = 0;
                if (g + lane < s1) {
                    mine = seg[g + lane];
                    my_h = hoff[g + lane] - base;
                }
                const u32 ng = min(32u, s1 - g);
                for (u32 q = 0; q < ng; q++) {
                    const u32 off = __shfl_sync(FULL, mine.offset, q), ln = __shfl_sync(FULL, mine.len, q);
                    const u32 score = __shfl_sync(FULL, mine.score, q), h0 = __shfl_sync(FULL, my_h, q);
                    const u32 nk = ln / TRN_K;
                    u32 cur = 0;
                    for (u32 t = lane; t < nk; t += 32) cur += s_freq[s_h[h0 + t]];
#pragma unroll
                    for (int d = 16; d >= 1; d >>= 1) cur += __shfl_xor_sync(FULL, cur, d);
                    if (cur * 2u < score) continue; /* earlier picks cover more than half of it */
                    const u32 copy = min(ln, capacity - total);
                    __syncwarp();
                    for (u32 t = lane; t < nk; t += 32) s_freq[s_h[h0 + t]] = 0;
                    __syncwarp();
                    if (lane == 0) picks[n_sel] = {off, copy, total};
                    n_sel++;
                    total += copy;
                    if (total >= capacity) break;
                }
            }
            if (lane == 0) {
                s_state[0] = n_sel;
                s_state[1] = total;
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        res[0] = s_state[0];
        res[1] = s_state[1];
    }
}

/* the picks in reverse: the first (highest-coverage) pick lands at the end of the output */
__global__ void zxc_train_emit_kernel(const u8* corpus, const TrainPick* picks, u32 n_picks, u32 total, u8* out) {
    const u32 lane = threadIdx.x & 31;
    const u32 nwarps = (gridDim.x * blockDim.x) >> 5;
    for (u32 j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n_picks; j += nwarps) {
        const TrainPick p = picks[j];
        u8* d = out + (total - p.before - p.copy);
        for (u32 k = lane; k < p.copy; k += 32) d[k] = corpus[(size_t)p.offset + k];
    }
}

/* one slice of the shared-table trainer: `len` bytes at `off` of the packed slice buffer */
struct TrainSlice {
    unsigned long long off;
    u32 len, pad;
};

/* The level-6 parse of [dict | slice] for every slice, exactly as zxc_encode_kernel<true> runs it at block size 4096
 * (P.block_size, P.level = 6 and the dictionary's seeded tables), stopped where the reference's parse_done hook reads
 * the literals.  lit_freq: 256 u32, accumulated with atomics. */
__global__ void __launch_bounds__(ENC_CTA_THREADS, ENC_OPT_MIN_CTAS) zxc_train_lit_kernel(const EncodeParams P,
                                                                                         const TrainSlice* slices,
                                                                                         u32* lit_freq) {
    const u32 lane = threadIdx.x & 31;
    const u32 wid = threadIdx.x >> 5;
    const u32 gwarp = blockIdx.x * ENC_WARPS_PER_CTA + wid;
    __shared__ u32 s_hist[ENC_WARPS_PER_CTA][256]; /* the parser's own scratch */
    __shared__ u32 s_acc[ENC_WARPS_PER_CTA][256];
    u32* acc = s_acc[wid];
    for (u32 k = lane; k < 256; k += 32) acc[k] = 0;
    u8* scratch = P.scratch + (size_t)gwarp * P.scratch_stride;
    const int level = (int)P.level;
    const EncLayout lay = enc_layout(P.block_size, level);
    u32* head = reinterpret_cast<u32*>(scratch);
    unsigned short* chain = reinterpret_cast<unsigned short*>(scratch + ENC_HASH_SIZE * 4);
    u8* literals = scratch + lay.literals;
    u8* tokens = scratch + lay.seqbuf;
    unsigned short* offsets = reinterpret_cast<unsigned short*>(scratch + lay.seqbuf + ((lay.seq_cap + 3) & ~3u));
    for (;;) {
        unsigned long long j = 0;
        if (lane == 0) j = atomicAdd(P.counter, 1ull);
        j = __shfl_sync(FULL, j, 0);
        if (j >= P.n_blocks) break;
        const u32 n = slices[j].len;
        const u8* src = enc_block_tables(P, lay, level, P.src + slices[j].off, n, scratch, head, chain, lane);
        const OptOut R = optimal_parse(src, P.dict_size, n, head, chain, level, lz_params(level),
                                       reinterpret_cast<u64*>(scratch + lay.dp), reinterpret_cast<u32*>(scratch + lay.ends),
                                       literals, tokens, offsets, scratch + lay.extras, s_hist[wid],
                                       reinterpret_cast<zxh_work_t*>(scratch + lay.work), scratch + lay.lens + 512, lane);
        for (u32 k = lane; k < R.lit_c; k += 32) atomicAdd(&acc[literals[k]], 1u);
        __syncwarp();
    }
    for (u32 k = lane; k < 256; k += 32)
        if (acc[k]) atomicAdd(&lit_freq[k], acc[k]);
}
