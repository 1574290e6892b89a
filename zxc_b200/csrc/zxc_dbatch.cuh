/*
 * zxc_dbatch.cuh -- many independent frames in HBM decoded in one stream-ordered call
 * (zxc_b200_decompress_device_batch).  Every step is zxc_dplan.cuh's per-frame algorithm run over all frames at once:
 *
 *   zxc_dbatch_tiles     per frame: the argument checks (NULL_INPUT, SRC_TOO_SMALL), its job-table share
 *                        J_i = ceil(cap_i / ZXC_BLOCK_SIZE_MIN) + 2, and the scan of the J_i within tiles of ASM_TILE
 *   zxc_dbatch_scan      one CTA: the tile sums' scan and the first frame whose share ends past the table (it and
 *                        every later frame that passed the checks get ZXC_ERROR_MEMORY)
 *   zxc_dbatch_probe     one thread per frame: its table offset, then dp_probe
 *   zxc_dbatch_sek       one CTA per frame with a SEK table: dp_sek_closes on the table's sum, then dp_sek_tile over
 *                        its tiles; any disagreement clears `fast`
 *   zxc_dbatch_walk      one warp per remaining frame: dp_walk
 *   zxc_dbatch_count     per frame: dp_n_fit / dp_fit and its launch slot (dp_slot); per tile and slot, the frames'
 *                        job counts scanned in frame order
 *   zxc_dbatch_slots     one CTA: per slot, the tile counts' scan, the slot's real jobs and its work counters
 *   zxc_dbatch_place     one thread per table entry: the frame's regular jobs into its slot's window, right-aligned
 *                        in frame order, with absolute device addresses; zeroed status words in front of them
 *   zxc_decode_kernel    (zxc_decode.cuh, unchanged) one launch_decode per slot over src = dst = 0
 *   zxc_dbatch_check     one thread per table entry: each frame's first job that did not produce its planned size
 *   zxc_dbatch_decide    one thread per frame: dp_decide
 *   zxc_dbatch_split     general split, phase 0: the size of every block of a split frame that ran out of room
 *   zxc_dbatch_split_scan  one CTA per split frame: dp_split_scan
 *   zxc_dbatch_split     phase 1: every block of a split frame at its true offset
 *   zxc_dbatch_split_final one CTA per split frame: dp_split_final
 * The split kernels exit at once when no frame split, so the launch sequence is the same for every batch.
 *
 * A frame's table share [base_i, base_i + J_i) indexes its plan and split sizes.  Each (block size, checksum
 * verification) slot has its own window of Jt jobs and status words, because the decode kernels take block_cap as a
 * launch parameter and claim jobs up to a host count; the windows hold the frames' jobs compacted and right-aligned,
 * with counters preset to the first real job (dp_preset).  Job offsets are device addresses over a zero
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

/* one frame's plan and verdict (J: its table share), and where its regular jobs go */
struct DBatchFrame : DFrame {
    const u8* src;
    u8* dst;
    unsigned long long pos; /* zxc_dbatch_count: its first job among the tile's jobs of its slot */
    unsigned int slot;      /* DP_SLOTS when it has no regular job */
};
static_assert(sizeof(DBatchFrame) == 152, "the scratch layout's per-frame records (DESIGN.md section 7h)");

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
    unsigned int n, n_slots;
    DDecodeOpts o;
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
    dp_probe(A.o, F->src, F, A.results + i);
}

/* the SEK-guided plan (dp_sek_closes, dp_sek_tile) for one frame per CTA, its table in tiles of ASM_TILE entries:
 * first the sum, then the headers at their predicted offsets */
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
        if (threadIdx.x == 0) s_ok = dp_sek_closes(F, F->src, total);
        __syncthreads();
        if (s_ok) {
            zxc_b200_job_t* plan = A.plan + A.base[f];
            u64 carry = 0;
            bool ok = true;
            u32 h = 0;
            for (u64 t0 = 0; t0 < nb; t0 += ASM_TILE) {
                ok &= dp_sek_tile(F, F->src, t0 + threadIdx.x * ASM_ITEMS, ZXC_FILE_HEADER_SIZE + carry, plan, &h,
                                  &total);
                carry += total;
            }
            dp_ghash_xor(F, h);
            if (!ok) s_ok = 0;
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
    dp_walk(F, F->src, F->src_size, F->J, A.plan + A.base[f], threadIdx.x & 31);
}

/* the regular plan's n_fit and slot per frame; each frame's place among its tile's jobs of the same slot */
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
            nf[k] = dp_n_fit(F);
            dp_fit(F, nf[k]);
            if (nf[k]) sl[k] = dp_slot(F);
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
        if (threadIdx.x == 0) {
            S->real[s] = carry;
            dp_preset(S->ctr[s], A.Jt - carry);
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

__global__ void __launch_bounds__(DB_THREADS) zxc_dbatch_decide(const DBatchArgs A) {
    const u64 f = (u64)blockIdx.x * DB_THREADS + threadIdx.x;
    if (f >= A.n) return;
    DBatchFrame* F = A.F + f;
    if (F->done) return;
    const u64 fb = F->first_bad;
    const i32 bad_status = fb != ~0ull ? A.status[F->slot * A.Jt + db_first_job(A, *F, (u32)f) + fb] : 0;
    if (dp_decide(F, bad_status, A.results + f)) A.st->any_split = 1;
}

/* ---- general split (dp_split_* per frame) ---- */
/* phase 0 and phase 1 over every split frame: a warp claims 32 table entries at a time, and decodes those that are
 * blocks of a split frame.  A warp's jobs may belong to different frames: their offsets are device addresses over a
 * zero base (D.src = D.dst = NULL), as in the regular decode. */
template <bool HAS_DICT>
__global__ void __launch_bounds__(CTA_THREADS) zxc_dbatch_split(const DBatchArgs A, const DSplitArgs D,
                                                                 const u32 phase) {
    extern __shared__ __align__(16) u8 smem[];
    DBatchState* S = A.st;
    if (!(phase == 0 ? S->any_split : S->any_redecode)) return;
    DecodeParams P;
    u8 *scratch, *ring;
    if (!dp_split_warp(D, phase, smem, &P, &scratch, &ring)) return;
    const u32 lane = threadIdx.x & 31;
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
            const int r = dp_split_block<HAS_DICT>(P, D, F, A.plan[tt], (u64)F.src, phase, scratch, ring, lane);
            if (lane == 0) A.sizes[tt] = r;
        }
    }
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dbatch_split_scan(const DBatchArgs A) {
    DBatchState* S = A.st;
    if (!S->any_split) return;
    for (u32 f = blockIdx.x; f < A.n; f += gridDim.x) {
        DBatchFrame* F = A.F + f;
        if (!F->split || F->done) continue;
        const u64 b0 = A.base[f];
        if (dp_split_scan(F, A.plan + b0, A.sizes + b0, (u64)F->src, (u64)F->dst, A.results + f) && threadIdx.x == 0)
            S->any_redecode = 1;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dbatch_split_final(const DBatchArgs A) {
    if (!A.st->any_split) return;
    for (u32 f = blockIdx.x; f < A.n; f += gridDim.x) {
        DBatchFrame* F = A.F + f;
        if (!F->split || F->done) continue;
        const u64 b0 = A.base[f];
        dp_split_final(F, A.plan + b0, A.sizes + b0, A.results + f);
        __syncthreads();
    }
}
