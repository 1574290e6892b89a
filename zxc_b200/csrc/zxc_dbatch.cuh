/*
 * zxc_dbatch.cuh -- many independent frames in HBM decoded in one stream-ordered call
 * (zxc_b200_decompress_device_batch).  Every step is zxc_dplan.cuh's per-frame algorithm run over all frames at once:
 *
 *   zxc_dbatch_tiles     per frame: the argument checks (NULL_INPUT, SRC_TOO_SMALL), its job-table share
 *                        J_i = ceil(cap_i / ZXC_BLOCK_SIZE_MIN) + 2, and the scan of the J_i within tiles of ASM_TILE
 *   zxc_dbatch_scan      one CTA: the tile sums' scan and the first frame whose share ends past the table (it and
 *                        every later frame that passed the checks get ZXC_ERROR_MEMORY)
 *   zxc_dbatch_probe     one thread per frame: its table offset, then dp_probe (the body of zxc_dplan_probe)
 *   zxc_dbatch_sek       one CTA per frame with a SEK table: the table's sum must close the chain at the EOF block,
 *                        then every block header at its predicted offset; any disagreement clears `fast`
 *   zxc_dbatch_walk      one warp per remaining frame: dp_walk (the body of zxc_dplan_walk)
 *   zxc_dbatch_count     per frame: the regular plan's n_fit and its launch slot; per tile and slot, the frames' job
 *                        counts scanned in frame order
 *   zxc_dbatch_slots     one CTA: per slot, the tile counts' scan, the slot's real jobs and its work counters
 *   zxc_dbatch_place     one thread per table entry: the frame's regular jobs into its slot's window, right-aligned
 *                        in frame order, with absolute device addresses; zeroed status words in front of them
 *   zxc_decode_kernel    (zxc_decode.cuh, unchanged) one launch_decode per slot over src = dst = 0
 *   zxc_dbatch_check     one thread per table entry: each frame's first job that did not produce its planned size
 *   zxc_dbatch_decide    one thread per frame: zxc_dplan_decide
 *   zxc_dbatch_split     general split, phase 0: the size of every block of a split frame that ran out of room
 *   zxc_dbatch_split_scan  one CTA per split frame: zxc_dsplit_scan
 *   zxc_dbatch_split     phase 1: every block of a split frame at its true offset
 *   zxc_dbatch_split_final one CTA per split frame: zxc_dsplit_final
 * The split kernels exit at once when no frame split, so the launch sequence is the same for every batch.
 *
 * A frame's table share [base_i, base_i + J_i) indexes its plan and split sizes.  Each (block size, checksum
 * verification) slot has its own window of Jt jobs and status words, because the decode kernels take block_cap as a
 * launch parameter and claim jobs up to a host count; the windows hold the frames' jobs compacted and right-aligned,
 * with counters preset to the first real job as in zxc_dplan_place.  Job offsets are device addresses over a zero
 * src / dst base, so one launch spans frames in unrelated allocations.
 */
#pragma once
#include <cuda_runtime.h>

#include "zxc_dplan.cuh"

#define DB_THREADS 256

/* the first bytes of the caller's scratch */
struct DBatchState {
    unsigned long long ctr[DP_SLOTS][4]; /* per launch slot: the decode's three work counters (launch_decode) */
    unsigned long long split_ctr[2];     /* the split decode's work counters, phase 0 and 1 */
    unsigned long long real[DP_SLOTS];   /* per slot: its real jobs */
    unsigned long long first_over;       /* first frame past the table (n: none) */
    unsigned int any_split, any_redecode;
};
#define DB_STATE_BYTES 1024
static_assert(sizeof(DBatchState) <= DB_STATE_BYTES, "DBatchState fits its region");

/* one frame's plan and verdict: the fields dp_probe, dp_walk, dp_planned and dp_tail use, as in DPlanState */
struct DBatchFrame {
    const u8* src;
    u8* dst;
    unsigned long long src_size, cap;
    unsigned long long n, n_fit, produced, footer_size, first_bad, sek_pos, eof_pos;
    unsigned long long pos; /* zxc_dbatch_count: its first job among the tile's jobs of its slot */
    unsigned int J, slot;   /* slot: DP_SLOTS when it has no regular job */
    unsigned int hint_n, block_size, has_checksum, verify, end, footer_hash, ghash;
    unsigned int fast, done, split, redecode;
};

struct DBatchArgs {
    const zxc_b200_frame_t* frames;
    long long* results;
    DBatchState* st;
    DBatchFrame* F;
    unsigned long long* base;   /* n: each frame's first table entry (ascending: the lookup's search key) */
    unsigned long long* tiles;  /* n_tiles: the J_i tile sums, then their exclusive scan */
    unsigned long long* stiles; /* n_tiles x n_slots: the slots' job counts per tile, then their exclusive scan */
    zxc_b200_job_t* plan;       /* Jt: the walk's src_off / src_len per block; the split's phase-1 jobs */
    i32* sizes;                 /* Jt: the split's true block sizes or errors, then its phase-1 status */
    zxc_b200_job_t* jobs;       /* n_slots windows of Jt */
    i32* status;                /* n_slots windows of Jt */
    unsigned long long Jt;
    unsigned int n, n_slots, max_block_size;
    unsigned int dict_id, have_dict;
    int huf_verdict;
    unsigned int checksum_enabled;
};

/* what dp_probe reads of one frame */
struct DBatchProbe {
    const u8* src;
    unsigned long long src_size, dst_capacity;
    DBatchFrame* st;
    long long* result;
    unsigned int J, max_block_size, dict_id, have_dict;
    int huf_verdict;
    unsigned int checksum_enabled;
};

/* the frame whose table share holds entry t: the last frame with base <= t */
__device__ __forceinline__ u32 db_frame_of(const DBatchArgs& A, u64 t) {
    u32 lo = 0, hi = A.n; /* base[lo] <= t < base[hi] */
    while (hi - lo > 1) {
        const u32 mid = lo + (hi - lo) / 2;
        if (A.base[mid] <= t) lo = mid;
        else hi = mid;
    }
    return lo;
}

/* the window index of frame f's first regular job */
__device__ __forceinline__ u64 db_first_job(const DBatchArgs& A, const DBatchFrame& F, u32 f) {
    const u32 s = F.slot;
    return A.Jt - A.st->real[s] + A.stiles[(u64)(f / ASM_TILE) * A.n_slots + s] + F.pos;
}

__global__ void __launch_bounds__(ASM_THREADS) zxc_dbatch_tiles(const DBatchArgs A) {
    const u64 first = (u64)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    u64 J[ASM_ITEMS], s = 0;
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        J[k] = 0;
        if (first + k < A.n) {
            const zxc_b200_frame_t d = A.frames[first + k];
            DBatchFrame& F = A.F[first + k];
            /* zxc_decompress's argument checks, in its order */
            long long v = 1;
            if (!d.src || (!d.dst && d.dst_capacity != 0)) v = ZXC_ERROR_NULL_INPUT;
            else if (d.src_size < ZXC_FILE_HEADER_SIZE + ZXC_FILE_FOOTER_SIZE) v = ZXC_ERROR_SRC_TOO_SMALL;
            if (v == 1) {
                const u64 j = d.dst_capacity / ZXC_BLOCK_SIZE_MIN + (d.dst_capacity % ZXC_BLOCK_SIZE_MIN != 0) + 2;
                J[k] = j <= A.Jt ? j : A.Jt + 1; /* past the table either way; keeps the sums far from overflow */
            } else {
                A.results[first + k] = v;
            }
            F.src = (const u8*)d.src;
            F.dst = (u8*)d.dst;
            F.src_size = d.src_size;
            F.cap = d.dst_capacity;
            F.J = (u32)J[k];
            F.done = v != 1;
            F.split = F.redecode = 0;
        }
        s += J[k];
    }
    unsigned long long total;
    u64 ex = asm_cta_excl(s, &total);
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        if (first + k < A.n) A.base[first + k] = ex;
        ex += J[k];
    }
    if (threadIdx.x == 0) A.tiles[blockIdx.x] = total;
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dbatch_scan(const DBatchArgs A) {
    __shared__ unsigned long long s_tile, s_first;
    DBatchState* S = A.st;
    const u32 n_tiles = (A.n + ASM_TILE - 1) / ASM_TILE;
    if (threadIdx.x == 0) s_tile = s_first = ~0ull;
    unsigned long long carry = 0;
    for (u32 b = 0; b < n_tiles; b += blockDim.x) {
        const u32 i = b + threadIdx.x;
        const unsigned long long v = i < n_tiles ? A.tiles[i] : 0;
        unsigned long long total;
        const unsigned long long ex = carry + asm_cta_excl(v, &total); /* its barriers also order s_tile */
        if (i < n_tiles) {
            A.tiles[i] = ex;
            if (ex + v > A.Jt) atomicMin(&s_tile, (unsigned long long)i);
        }
        carry += total;
    }
    __syncthreads();
    const u64 t = s_tile;
    if (t != ~0ull) { /* the first frame of that tile whose share ends past Jt */
        for (u64 i = t * ASM_TILE + threadIdx.x; i < A.n && i < (t + 1) * ASM_TILE; i += blockDim.x)
            if (A.F[i].J && A.tiles[t] + A.base[i] + A.F[i].J > A.Jt) atomicMin(&s_first, i);
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    S->first_over = t != ~0ull ? s_first : A.n;
    S->any_split = S->any_redecode = 0;
    S->split_ctr[0] = S->split_ctr[1] = 0;
}

__global__ void __launch_bounds__(DB_THREADS) zxc_dbatch_probe(const DBatchArgs A) {
    const u64 i = (u64)blockIdx.x * DB_THREADS + threadIdx.x;
    if (i >= A.n) return;
    A.base[i] += A.tiles[i / ASM_TILE];
    DBatchFrame* F = A.F + i;
    if (F->done) return;
    if (i >= A.st->first_over) {
        A.results[i] = ZXC_ERROR_MEMORY;
        F->done = 1;
        return;
    }
    DBatchProbe P;
    P.src = F->src;
    P.src_size = F->src_size;
    P.dst_capacity = F->cap;
    P.st = F;
    P.result = A.results + i;
    P.J = F->J;
    P.max_block_size = A.max_block_size;
    P.dict_id = A.dict_id;
    P.have_dict = A.have_dict;
    P.huf_verdict = A.huf_verdict;
    P.checksum_enabled = A.checksum_enabled;
    dp_probe(P);
}

/* zxc_dplan_sek_tiles / _scan / _blocks for one frame per CTA, its table in tiles of ASM_TILE entries: first the sum
 * (the chain must close at the EOF block in front of the table), then the headers at their predicted offsets, which
 * the sum keeps in front of the EOF block */
__global__ void __launch_bounds__(ASM_THREADS) zxc_dbatch_sek(const DBatchArgs A) {
    __shared__ unsigned int s_ok;
    for (u32 f = blockIdx.x; f < A.n; f += gridDim.x) {
        DBatchFrame* F = A.F + f;
        if (F->done || !F->fast) continue; /* uniform: only this CTA writes them, after the barriers below */
        const u32 nb = F->hint_n;
        const u8* e = F->src + F->sek_pos;
        u64 sum = 0;
        for (u64 b = threadIdx.x; b < nb; b += ASM_THREADS) sum += ld32(e + 4 * b);
        unsigned long long total;
        asm_cta_excl(sum, &total);
        if (threadIdx.x == 0) {
            u32 type = 0, comp = 1;
            s_ok = ZXC_FILE_HEADER_SIZE + total == F->eof_pos && dp_block_header(F->src + F->eof_pos, &type, &comp) &&
                   type == ZXF_BT_EOF && comp == 0;
        }
        __syncthreads();
        if (s_ok) {
            const u32 trailer = F->has_checksum ? ZXF_BLOCK_CKS : 0u;
            zxc_b200_job_t* plan = A.plan + A.base[f];
            u64 carry = 0;
            bool bad = false;
            u32 h = 0;
            for (u64 t0 = 0; t0 < nb; t0 += ASM_TILE) {
                const u64 first = t0 + threadIdx.x * ASM_ITEMS;
                u32 c[ASM_ITEMS];
                u64 s = 0;
#pragma unroll
                for (u32 k = 0; k < ASM_ITEMS; k++) {
                    c[k] = first + k < nb ? ld32(e + 4 * (first + k)) : 0u;
                    s += c[k];
                }
                u64 off = ZXC_FILE_HEADER_SIZE + carry + asm_cta_excl(s, &total);
#pragma unroll
                for (u32 k = 0; k < ASM_ITEMS; k++) {
                    const u64 j = first + k;
                    if (j >= nb) break;
                    u32 type, comp;
                    if (!dp_block_header(F->src + off, &type, &comp) || type > ZXF_BT_GHI ||
                        (u64)ZXF_BLOCK_HDR + comp + trailer != c[k]) {
                        bad = true;
                    } else {
                        zxc_b200_job_t Jb;
                        Jb.src_off = off;
                        Jb.dst_off = 0;
                        Jb.src_len = c[k];
                        Jb.dst_cap = 0;
                        plan[j] = Jb;
                        if (trailer) h ^= dp_rotl(ld32(F->src + off + ZXF_BLOCK_HDR + comp), (u32)((nb - 1 - j) & 31u));
                    }
                    off += c[k];
                }
                carry += total;
            }
            for (u32 d = 16; d; d >>= 1) h ^= __shfl_xor_sync(FULL, h, d);
            if ((threadIdx.x & 31) == 0 && h) atomicXor(&F->ghash, h);
            if (bad) s_ok = 0;
            __syncthreads();
            if (threadIdx.x == 0 && s_ok) {
                F->n = nb;
                F->end = ZXW_END_EOF;
            }
        }
        if (threadIdx.x == 0 && !s_ok) F->fast = 0;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(DB_THREADS) zxc_dbatch_walk(const DBatchArgs A) {
    const u64 f = ((u64)blockIdx.x * DB_THREADS + threadIdx.x) >> 5;
    if (f >= A.n) return;
    DBatchFrame* F = A.F + f;
    if (F->done || F->fast) return;
    dp_walk(F->src, F->src_size, A.plan + A.base[f], F->J, F, threadIdx.x & 31);
}

/* zxc_dplan_place's n_fit and slot per frame; each frame's place among its tile's jobs of the same slot */
__global__ void __launch_bounds__(ASM_THREADS) zxc_dbatch_count(const DBatchArgs A) {
    __shared__ unsigned int s_used;
    if (threadIdx.x == 0) s_used = 0;
    __syncthreads();
    const u64 first = (u64)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    u64 nf[ASM_ITEMS];
    u32 sl[ASM_ITEMS];
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        nf[k] = 0;
        sl[k] = DP_SLOTS;
        if (first + k >= A.n) continue;
        DBatchFrame* F = A.F + first + k;
        if (!F->done) {
            const u64 n = F->n;
            const u32 bs = F->block_size;
            if (n > 0) {
                const u64 kk = F->cap / bs;
                nf[k] = kk < n - 1 ? kk : (n - 1 + ((n - 1) * bs + dp_planned(F, n - 1, n) <= F->cap ? 1 : 0));
            }
            F->first_bad = ~0ull;
            F->n_fit = nf[k];
            F->produced = nf[k] ? (nf[k] - 1) * bs + dp_planned(F, nf[k] - 1, n) : 0;
            if (nf[k]) sl[k] = (__ffs(bs) - 1 - ZXC_BLOCK_SIZE_MIN_LOG2) * 2 + F->verify;
        }
        F->slot = sl[k];
        if (sl[k] < DP_SLOTS) atomicOr(&s_used, 1u << sl[k]);
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
        for (u32 k = 0; k < ASM_ITEMS; k++) v += sl[k] == s ? nf[k] : 0;
        unsigned long long total;
        u64 ex = asm_cta_excl(v, &total);
#pragma unroll
        for (u32 k = 0; k < ASM_ITEMS; k++) {
            if (sl[k] == s) {
                A.F[first + k].pos = ex;
                ex += nf[k];
            }
        }
        if (threadIdx.x == 0) A.stiles[(u64)blockIdx.x * A.n_slots + s] = total;
    }
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dbatch_slots(const DBatchArgs A) {
    DBatchState* S = A.st;
    const u32 n_tiles = (A.n + ASM_TILE - 1) / ASM_TILE;
    for (u32 s = 0; s < DP_SLOTS; s++) {
        unsigned long long carry = 0;
        if (s < A.n_slots) {
            for (u32 b = 0; b < n_tiles; b += blockDim.x) {
                const u32 i = b + threadIdx.x;
                unsigned long long* p = A.stiles + (u64)i * A.n_slots + s;
                const unsigned long long v = i < n_tiles ? *p : 0;
                unsigned long long total;
                const unsigned long long ex = carry + asm_cta_excl(v, &total);
                if (i < n_tiles) *p = ex;
                carry += total;
            }
        }
        if (threadIdx.x == 0) { /* counters as in zxc_dplan_place */
            S->real[s] = carry;
            S->ctr[s][0] = A.Jt - carry;
            S->ctr[s][1] = 0;
            S->ctr[s][2] = 0;
        }
    }
}

__global__ void __launch_bounds__(DB_THREADS) zxc_dbatch_place(const DBatchArgs A) {
    const DBatchState* S = A.st;
    const u64 nthreads = (u64)gridDim.x * DB_THREADS;
    for (u64 t = (u64)blockIdx.x * DB_THREADS + threadIdx.x; t < A.Jt; t += nthreads) {
        /* no stale deferral marks in front of the real jobs (the deferred launch may scan the status words from 0) */
        for (u32 s = 0; s < A.n_slots; s++)
            if (S->real[s] && t < A.Jt - S->real[s]) A.status[s * A.Jt + t] = 0;
        const u32 f = db_frame_of(A, t);
        const DBatchFrame& F = A.F[f];
        const u64 k = t - A.base[f];
        if (F.done || k >= F.n_fit) continue;
        zxc_b200_job_t Jb = A.plan[t];
        Jb.src_off += (u64)F.src;
        Jb.dst_off = (u64)F.dst + k * F.block_size;
        Jb.dst_cap = dp_planned(&F, k, F.n);
        A.jobs[F.slot * A.Jt + db_first_job(A, F, f) + k] = Jb;
    }
}

__global__ void __launch_bounds__(DB_THREADS) zxc_dbatch_check(const DBatchArgs A) {
    const u64 nthreads = (u64)gridDim.x * DB_THREADS;
    for (u64 t = (u64)blockIdx.x * DB_THREADS + threadIdx.x; t < A.Jt; t += nthreads) {
        const u32 f = db_frame_of(A, t);
        DBatchFrame& F = A.F[f];
        const u64 k = t - A.base[f];
        if (F.done || k >= F.n_fit) continue;
        const i32 st = A.status[F.slot * A.Jt + db_first_job(A, F, f) + k];
        if (st < 0 || (u32)st != dp_planned(&F, k, F.n)) atomicMin(&F.first_bad, k);
    }
}

/* the general split needs every block in the frame's table share (dp_split) */
__device__ __forceinline__ void db_split(const DBatchArgs& A, DBatchFrame* F, u32 f) {
    if (F->n > F->J) {
        A.results[f] = ZXC_ERROR_MEMORY;
        F->done = 1;
    } else {
        F->split = 1;
        A.st->any_split = 1;
    }
}

/* zxc_dplan_decide per frame */
__global__ void __launch_bounds__(DB_THREADS) zxc_dbatch_decide(const DBatchArgs A) {
    const u64 f = (u64)blockIdx.x * DB_THREADS + threadIdx.x;
    if (f >= A.n) return;
    DBatchFrame* F = A.F + f;
    if (F->done) return;
    const u64 n = F->n, n_fit = F->n_fit;
    if (F->first_bad != ~0ull) {
        const i32 st = A.status[F->slot * A.Jt + db_first_job(A, *F, (u32)f) + F->first_bad];
        if (st >= 0 || st == ZXC_ERROR_OVERFLOW || st == ZXC_ERROR_DST_TOO_SMALL) {
            db_split(A, F, (u32)f);
            return;
        }
        A.results[f] = st;
        F->done = 1;
        return;
    }
    if (n_fit < n && F->end == ZXW_END_EOF && F->footer_size <= F->cap) {
        db_split(A, F, (u32)f);
        return;
    }
    A.results[f] = dp_tail(F, F->produced, n_fit == n);
    F->done = 1;
}

/* ---- general split (zxc_dsplit_* per frame) ---- */
struct DBatchSplitArgs {
    DBatchArgs a;
    u8* zero;  /* NULL: the base of the jobs' device addresses */
    u8* slots; /* probe_warps slots of `room` bytes */
    u8* scratch;
    const u8* dict;
    const u8* dict_huf;
    u32 dict_size, scratch_stride, room, probe_warps;
};

/* zxc_dsplit_decode over every split frame: a warp claims 32 table entries at a time, and decodes those that are
 * blocks of a split frame (phase 0: the ones whose regular decode ran out of room or did not run, into its slot; phase
 * 1: all of them at their true offsets) */
template <bool HAS_DICT>
__global__ void __launch_bounds__(CTA_THREADS) zxc_dbatch_split(const DBatchSplitArgs D, const u32 phase) {
    extern __shared__ __align__(16) u8 smem[];
    const DBatchArgs& A = D.a;
    DBatchState* S = A.st;
    if (!(phase == 0 ? S->any_split : S->any_redecode)) return;
    const u32 lane = threadIdx.x & 31;
    const u32 wic = threadIdx.x >> 5;
    const u32 gwarp = blockIdx.x * WARPS_PER_CTA + wic;
    if (phase == 0 && gwarp >= D.probe_warps) return;
    u8* scratch = D.scratch + (size_t)gwarp * D.scratch_stride + 256;
    u8* ring = smem + (size_t)wic * WARP_SMEM_BYTES;
#if ZXC_STAGE
    st_init(smem_addr(ring) + RING_BYTES, lane);
#endif
    /* a warp's jobs may belong to different frames: their offsets are device addresses over a zero base, as in the
     * regular decode.  The base is a kernel parameter, which the compiler takes for a global pointer, so the shared
     * decode body keeps its global loads and stores. */
    DecodeParams P;
    P.src = D.zero;
    P.dst = phase == 0 ? D.slots + (size_t)gwarp * D.room : D.zero;
    P.jobs = NULL;
    P.status = NULL;
    P.dict = D.dict;
    P.dict_huf = D.dict_huf;
    P.scratch = D.scratch;
    P.counter = NULL;
    P.n_jobs = 0;
    P.dict_size = D.dict_size;
    P.scratch_stride = D.scratch_stride;
    P.defer_list = NULL;
    P.defer_count = NULL;
    P.defer_cap = 0;
    for (;;) {
        unsigned long long t0 = 0;
        if (lane == 0) t0 = atomicAdd(&S->split_ctr[phase], 32ull);
        t0 = __shfl_sync(FULL, t0, 0);
        if (t0 >= A.Jt) break;
        const u64 t = t0 + lane;
        u32 f = 0;
        bool work = false;
        if (t < A.Jt) {
            f = db_frame_of(A, t);
            const DBatchFrame& F = A.F[f];
            const u64 k = t - A.base[f];
            work = !F.done && (phase == 0 ? F.split : F.redecode) && k < F.n;
            if (work && phase == 0 && k < F.n_fit) {
                const i32 r = A.status[F.slot * A.Jt + db_first_job(A, F, f) + k];
                if (r != ZXC_ERROR_OVERFLOW && r != ZXC_ERROR_DST_TOO_SMALL) {
                    A.sizes[t] = r;
                    work = false;
                }
            }
        }
        for (u32 m = __ballot_sync(FULL, work); m; m &= m - 1) {
            const u32 src_lane = __ffs(m) - 1;
            const u32 g = __shfl_sync(FULL, f, src_lane);
            const u64 tt = t0 + src_lane;
            const DBatchFrame& F = A.F[g];
            zxc_b200_job_t job = A.plan[tt];
            if (phase == 0) {
                job.src_off += (u64)F.src;
                job.dst_off = 0;
                job.dst_cap = D.room;
            }
            P.flags = F.verify ? FLAG_VERIFY : 0u;
            P.block_cap = F.block_size;
            const int r = decode_job<false, HAS_DICT, false>(P, job, scratch, ring, lane);
            flush_wait(lane); /* nothing of this block is still on its way out of the ring */
            __syncwarp();
            if (lane == 0) A.sizes[tt] = r;
        }
    }
}

/* zxc_dsplit_scan per split frame, one CTA each; phase 1's jobs replace the frame's plan entries */
__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dbatch_split_scan(const DBatchArgs A) {
    __shared__ unsigned long long s_fail;
    DBatchState* S = A.st;
    if (!S->any_split) return;
    for (u32 f = blockIdx.x; f < A.n; f += gridDim.x) {
        DBatchFrame* F = A.F + f;
        if (!F->split || F->done) continue;
        const u64 n = F->n, cap = F->cap, b0 = A.base[f];
        if (threadIdx.x == 0) s_fail = ~0ull;
        unsigned long long carry = 0;
        bool failed = false;
        for (u64 b = 0; b < n; b += blockDim.x) {
            const u64 i = b + threadIdx.x;
            const i32 v = i < n ? A.sizes[b0 + i] : 0;
            unsigned long long total;
            const u64 op = carry + asm_cta_excl(v > 0 ? (u64)v : 0ull, &total); /* its barriers also order s_fail */
            const bool err = i < n && v < 0;
            const bool over = i < n && v >= 0 && op <= cap && (u64)v > cap - op;
            if (err || over) atomicMin(&s_fail, i);
            __syncthreads();
            const u64 fl = s_fail;
            if (fl != ~0ull) {
                if (i == fl) {
                    A.results[f] = err ? (long long)v : (long long)ZXC_ERROR_DST_TOO_SMALL;
                    F->done = 1;
                }
                failed = true;
                break;
            }
            if (i < n) {
                zxc_b200_job_t Jb = A.plan[b0 + i];
                Jb.src_off += (u64)F->src;
                Jb.dst_off = (u64)F->dst + op;
                Jb.dst_cap = (u32)v;
                A.plan[b0 + i] = Jb;
            }
            carry += total;
        }
        if (threadIdx.x == 0 && !failed) {
            F->produced = carry;
            F->redecode = carry > 0;
            if (carry > 0) S->any_redecode = 1;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dbatch_split_final(const DBatchArgs A) {
    __shared__ unsigned long long s_bad;
    if (!A.st->any_split) return;
    for (u32 f = blockIdx.x; f < A.n; f += gridDim.x) {
        DBatchFrame* F = A.F + f;
        if (!F->split || F->done) continue;
        const u64 n = F->n, b0 = A.base[f];
        if (threadIdx.x == 0) s_bad = ~0ull;
        __syncthreads();
        if (F->redecode) {
            for (u64 i = threadIdx.x; i < n; i += blockDim.x) {
                const i32 st = A.sizes[b0 + i];
                if (st < 0 || (u32)st != A.plan[b0 + i].dst_cap) atomicMin(&s_bad, i);
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            if (s_bad != ~0ull) {
                const i32 st = A.sizes[b0 + s_bad];
                A.results[f] = st < 0 ? st : ZXC_ERROR_CORRUPT_DATA;
            } else {
                A.results[f] = dp_tail(F, F->produced, true);
            }
            F->done = 1;
        }
        __syncthreads();
    }
}
