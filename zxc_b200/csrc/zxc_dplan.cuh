/*
 * zxc_dplan.cuh -- frame decode with the frame in HBM (zxc_b200_decompress_device): the frame walk, the job table and
 * zxc_decompress's verdict on the device, on the caller's stream, with no host round trip.  Stream order:
 *
 *   zxc_dplan_probe       one thread: the dst_capacity == 0 shortcut, the file-header checks of zxf_read_file_header,
 *                         the scratch's block-size limit, the dictionary verdicts, the footer, and the SEK table probe
 *                         of zxw_walk's prefetch hint
 *   zxc_dplan_sek_tiles   \  SEK-guided plan: tile sums of the table's sizes, one CTA's scan of them into predicted
 *   zxc_dplan_sek_scan     | header offsets (and the chain's end at the EOF block), then per block the header at its
 *   zxc_dplan_sek_blocks  /  predicted offset, its plan entry and its global-hash term; any disagreement with what the
 *                            sequential walk would see clears `fast`
 *   zxc_dplan_walk        one warp: zxw_walk, for frames without a table or when `fast` was cleared (blocks beyond
 *                         the job table are counted, not stored)
 *   zxc_dplan_place       the plan's first n_fit blocks into the decode job table, right-aligned in [J - n_fit, J),
 *                         and the work counters of every decode launch slot
 *   zxc_decode_kernel     (zxc_decode.cuh, unchanged) one launch_decode per slot; only the frame's slot has work
 *   zxc_dplan_check       first job that did not produce its planned size
 *   zxc_dplan_decide      decompress_frame's order: block error, plan mismatch, capacity, EOF, footer, global hash
 *   zxc_dsplit_decode     general split, phase 0: the size of every block that ran out of room, in a per-warp slot
 *   zxc_dsplit_scan       true offsets in the reference's order (a block's error, then whether it fits)
 *   zxc_dsplit_decode     phase 1: every block at its true offset
 *   zxc_dsplit_final      the split's verdict
 * Every kernel after the probe exits at once when an earlier one has written the result, and the split kernels exit
 * at once unless the regular plan saw a mismatch, so the launch sequence is the same for every frame.
 *
 * The decode kernels loop `j < P.n_jobs` on a host value and claim jobs through work counters.  The job table has J
 * entries (known on the host from the scratch size); the n real jobs sit in [J - n, J) and the first launch's counter
 * starts at J - n, so its claim loop and the status array see only the real jobs.  The deferred launch claims
 * positions in the list of jobs the first one deferred, so its counter starts at 0 as before.  One launch slot per (block size, checksum
 * verification): DecodeParams is a kernel parameter, so each block size the scratch allows gets its own launch with
 * its own block_cap, and the slots that do not match the frame get counters preset to J and exit at once.
 *
 * Frame bytes are read byte by byte: d_src may have any alignment and nothing outside it is read.
 */
#pragma once
#include <cuda_runtime.h>

#include "zxc_b200.h"
#include "zxc_error.h"
#include "zxc_format.h"
#include "zxc_frame.h"

#define DP_SLOTS ((ZXC_BLOCK_SIZE_MAX_LOG2 - ZXC_BLOCK_SIZE_MIN_LOG2 + 1) * 2) /* block sizes x verify off / on */
#define DP_THREADS 256

/* the first bytes of the caller's scratch (DP_STATE_BYTES) */
struct DPlanState {
    unsigned long long ctr[DP_SLOTS][4]; /* per launch slot: the decode's three work counters (launch_decode) */
    unsigned long long split_ctr[2];     /* zxc_dsplit_decode's work counters, phase 0 and 1 */
    unsigned long long n;                /* blocks ahead of the end of the block stream */
    unsigned long long n_fit;            /* the regular plan's blocks that fit dst_capacity */
    unsigned long long produced;
    unsigned long long footer_size;
    unsigned long long first_bad; /* zxc_dplan_check: first job in stream order that failed */
    unsigned long long sek_pos;   /* offset of the SEK table's first entry */
    unsigned long long eof_pos;   /* where the table says the EOF block is */
    unsigned int hint_n;          /* SEK entries (0: no table) */
    unsigned int block_size, has_checksum, verify, end, footer_hash, ghash;
    unsigned int fast;     /* the SEK-guided plan holds */
    unsigned int done;     /* *result is written */
    unsigned int split;    /* the general split runs */
    unsigned int redecode; /* the split's second decode has work */
};
#define DP_STATE_BYTES 1024
static_assert(sizeof(DPlanState) <= DP_STATE_BYTES, "DPlanState fits its region");

struct DPlanArgs {
    const u8* src;
    unsigned long long src_size, dst_capacity;
    zxc_b200_job_t* plan; /* J entries: the walk's src_off / src_len per block */
    zxc_b200_job_t* jobs; /* J entries: the decode job table, real jobs right-aligned */
    i32* status;          /* J entries, indexed like jobs */
    i32* sizes;           /* J entries: the split's true block sizes, or a block's error */
    unsigned long long* tiles;
    DPlanState* st;
    long long* result;
    unsigned int J, max_block_size;
    unsigned int dict_id;   /* zxc_dict_id of the caller's dictionary */
    unsigned int have_dict; /* a dictionary was given */
    int huf_verdict;        /* dict_huf_attach of its table: 1 usable, 0 none, < 0 malformed */
    unsigned int checksum_enabled;
};

/* zxc_hash16 (zxc_format.c) over the 16 file-header bytes with bytes 14-15 zero */
__device__ __forceinline__ u32 dp_hash16(u64 a, u64 b) {
    u64 h = a ^ b ^ 0xD2D84A61D2D84A61ull;
    h ^= h << 13;
    h ^= h >> 7;
    h ^= h << 17;
    const u32 r = (u32)((h >> 32) ^ h);
    return ((r >> 16) ^ r) & 0xFFFFu;
}

/* zxf_read_block_header on 8 readable bytes: false on a bad CRC */
__device__ __forceinline__ bool dp_block_header(const u8* p, u32* type, u32* comp) {
    const u64 v = ld64(p);
    *type = (u32)(v & 0xFFu);
    *comp = (u32)(v >> 24);
    return (u32)(v >> 56) == (u32)dev_hash8(v & 0x00FFFFFFFFFFFFFFull);
}

__device__ __forceinline__ u32 dp_rotl(u32 v, u32 r) { return r ? (v << r) | (v >> (32 - r)) : v; }

/* expected_block_bytes / decompress_frame's planned size of block i: block_size for every block but the last; the
 * last gets the footer's remainder (block_size when that is 0) */
template <class St>
__device__ __forceinline__ u32 dp_planned(const St* S, u64 i, u64 n) {
    const u32 bs = S->block_size;
    if (i + 1 < n) return bs;
    const u64 start = i * bs;
    const u64 f = S->footer_size;
    const u32 e = f <= start ? 0u : (f - start >= bs ? bs : (u32)(f - start));
    return e ? e : bs;
}

/* decompress_frame's checks behind the decode (the `decoded:` label) */
template <class St>
__device__ __forceinline__ long long dp_tail(const St* S, u64 produced, bool all_fit) {
    if (!all_fit) return ZXC_ERROR_DST_TOO_SMALL;
    if (S->end == ZXW_END_BAD_HEADER) return ZXC_ERROR_BAD_HEADER;
    if (S->end == ZXW_END_EOF) {
        if (S->footer_size != produced) return ZXC_ERROR_CORRUPT_DATA;
        if (S->verify && S->footer_hash != S->ghash) return ZXC_ERROR_BAD_CHECKSUM;
    }
    return (long long)produced;
}

__device__ __forceinline__ void dp_prefetch(const u8* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

/* zxc_dplan_probe's body for one frame of size >= header + footer; zxc_dbatch_probe runs it per frame too.  Ar has
 * DPlanArgs's fields the probe reads, and its `st` points to a DPlanState or a DBatchFrame (one frame's plan). */
template <class Ar>
__device__ __forceinline__ void dp_probe(const Ar A) {
    auto* S = A.st;
    const u8* s = A.src;
    const u64 size = A.src_size; /* >= header + footer: checked before (on the host, or by zxc_dbatch_tiles) */
    S->done = S->fast = S->split = S->redecode = 0;
    S->hint_n = 0;
    S->ghash = 0;
    S->n = 0;
    S->end = ZXW_END_RAN_OFF;
    const u64 footer = ld64(s + size - ZXC_FILE_FOOTER_SIZE);
    S->footer_size = footer;
    S->footer_hash = ld32(s + size - 4);
    long long v = 1; /* 1: undecided */
    u32 bs = 0;
    if (A.dst_capacity == 0) { /* the empty-frame shortcut of decompress_entry */
        v = ld32(s) != ZXF_MAGIC ? ZXC_ERROR_BAD_MAGIC : (footer == 0 ? 0 : ZXC_ERROR_DST_TOO_SMALL);
    } else if (ld32(s) != ZXF_MAGIC) {
        v = ZXC_ERROR_BAD_MAGIC;
    } else if (s[4] != ZXF_VERSION) {
        v = ZXC_ERROR_BAD_VERSION;
    } else if (ld16(s + 14) != dp_hash16(ld64(s), ld64(s + 8) & 0x0000FFFFFFFFFFFFull) || (s[6] & 0x0Fu) != 0) {
        v = ZXC_ERROR_BAD_HEADER;
    } else if (s[5] < ZXC_BLOCK_SIZE_MIN_LOG2 || s[5] > ZXC_BLOCK_SIZE_MAX_LOG2) {
        v = ZXC_ERROR_BAD_BLOCK_SIZE;
    } else if ((1u << s[5]) > A.max_block_size) {
        v = ZXC_ERROR_MEMORY; /* the scratch was sized for smaller blocks */
    } else {
        bs = 1u << s[5];
        const u32 did = (s[6] & ZXF_FLAG_DICT) ? ld32(s + 7) : 0u;
        if (did != 0 && !A.have_dict) v = ZXC_ERROR_DICT_REQUIRED;
        else if (did != 0 && A.dict_id != did) v = ZXC_ERROR_DICT_MISMATCH;
        else if (A.have_dict && A.huf_verdict < 0) v = A.huf_verdict;
    }
    if (v != 1) {
        *A.result = v;
        S->done = 1;
        return;
    }
    S->block_size = bs;
    S->has_checksum = (s[6] & ZXF_FLAG_CHECKSUM) ? 1u : 0u;
    S->verify = S->has_checksum && A.checksum_enabled;
    /* zxw_walk's prefetch hint: a SEK block header where a table for the footer's size would start */
    if (footer > 0) {
        const u64 nb = (footer + bs - 1) / bs;
        const u64 sek_total = ZXF_BLOCK_HDR + nb * ZXF_SEEK_ENTRY;
        if (nb <= 0xFFFFFFFFull && sek_total + ZXC_FILE_FOOTER_SIZE + ZXC_FILE_HEADER_SIZE <= size) {
            const u64 sp = size - ZXC_FILE_FOOTER_SIZE - sek_total;
            if (s[sp] == ZXF_BT_SEK && ld32(s + sp + 3) == (u32)(nb * ZXF_SEEK_ENTRY)) {
                S->hint_n = (u32)nb;
                S->sek_pos = sp + ZXF_BLOCK_HDR;
                S->eof_pos = sp - ZXF_BLOCK_HDR;
                S->fast = nb <= A.J;
            }
        }
    }
}

__global__ void zxc_dplan_probe(const DPlanArgs A) {
    dp_probe(A);
}

__global__ void __launch_bounds__(ASM_THREADS) zxc_dplan_sek_tiles(const DPlanArgs A) {
    const DPlanState* S = A.st;
    if (S->done || !S->fast) return;
    const u32 nb = S->hint_n;
    if ((u64)blockIdx.x * ASM_TILE >= nb) return;
    const u8* e = A.src + S->sek_pos;
    const u64 base = (u64)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    u64 s = 0;
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++)
        if (base + k < nb) s += ld32(e + 4 * (base + k));
    unsigned long long total;
    asm_cta_excl(s, &total);
    if (threadIdx.x == 0) A.tiles[blockIdx.x] = total;
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dplan_sek_scan(const DPlanArgs A) {
    DPlanState* S = A.st;
    if (S->done || !S->fast) return;
    const u32 n_tiles = (u32)(((u64)S->hint_n + ASM_TILE - 1) / ASM_TILE);
    unsigned long long carry = 0;
    for (u32 b = 0; b < n_tiles; b += blockDim.x) {
        const u32 i = b + threadIdx.x;
        const unsigned long long v = i < n_tiles ? A.tiles[i] : 0;
        unsigned long long total;
        const unsigned long long ex = asm_cta_excl(v, &total);
        if (i < n_tiles) A.tiles[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) {
        /* the chain closes at the EOF block in front of the table, and that block is a valid empty EOF */
        u32 type = 0, comp = 1;
        const bool closes = ZXC_FILE_HEADER_SIZE + carry == S->eof_pos &&
                            dp_block_header(A.src + S->eof_pos, &type, &comp) && type == ZXF_BT_EOF && comp == 0;
        if (closes) {
            S->n = S->hint_n;
            S->end = ZXW_END_EOF;
        } else {
            S->fast = 0;
        }
    }
}

__global__ void __launch_bounds__(ASM_THREADS) zxc_dplan_sek_blocks(const DPlanArgs A) {
    DPlanState* S = A.st;
    if (S->done || !S->fast) return;
    const u32 nb = S->hint_n;
    if ((u64)blockIdx.x * ASM_TILE >= nb) return;
    const u8* e = A.src + S->sek_pos;
    const u64 base = (u64)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    u32 c[ASM_ITEMS];
    u64 s = 0;
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        c[k] = base + k < nb ? ld32(e + 4 * (base + k)) : 0u;
        s += c[k];
    }
    unsigned long long total;
    u64 off = ZXC_FILE_HEADER_SIZE + A.tiles[blockIdx.x] + asm_cta_excl(s, &total);
    const u32 trailer = S->has_checksum ? ZXF_BLOCK_CKS : 0u;
    bool bad = false;
    u32 h = 0;
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        const u64 j = base + k;
        if (j >= nb) break;
        u32 type, comp;
        /* every offset lies in front of the EOF block (the scan checked the sum), so the 8 header bytes are there */
        if (!dp_block_header(A.src + off, &type, &comp) || type > ZXF_BT_GHI ||
            (u64)ZXF_BLOCK_HDR + comp + trailer != c[k]) {
            bad = true;
        } else {
            zxc_b200_job_t Jb;
            Jb.src_off = off;
            Jb.dst_off = 0;
            Jb.src_len = c[k];
            Jb.dst_cap = 0;
            A.plan[j] = Jb;
            if (trailer) h ^= dp_rotl(ld32(A.src + off + ZXF_BLOCK_HDR + comp), (u32)((nb - 1 - j) & 31u));
        }
        off += c[k];
    }
    for (u32 d = 16; d; d >>= 1) h ^= __shfl_xor_sync(FULL, h, d);
    if ((threadIdx.x & 31) == 0 && h) atomicXor(&S->ghash, h);
    if (bad) S->fast = 0;
}

/* zxw_walk, warp-uniform: every lane follows the chain (the header loads are broadcasts), lane 0 stores.  With a SEK
 * table the lanes prefetch the next 32 predicted headers into L2, a window ahead of the walk, like the host walk; a
 * wrong or forged table only prefetches the wrong lines. */
template <class St>
__device__ __forceinline__ void dp_walk(const u8* s, const u64 size, zxc_b200_job_t* plan, const u32 J, St* S,
                                        const u32 lane) {
    const u32 trailer = S->has_checksum ? ZXF_BLOCK_CKS : 0u;
    const u32 hint_n = S->hint_n;
    const u8* he = s + S->sek_pos;
    u64 ip = ZXC_FILE_HEADER_SIZE, hint_off = ZXC_FILE_HEADER_SIZE, n = 0;
    u32 g = 0, end = ZXW_END_RAN_OFF, hint_idx = 0;
    while (ip < size) {
        if (hint_idx < hint_n && hint_idx < n + 32) {
            const u32 i = hint_idx + lane;
            const u64 c = i < hint_n ? ld32(he + 4ull * i) : 0ull;
            const u64 inc = asm_warp_incl(c, lane);
            const u64 o = hint_off + inc - c;
            if (i < hint_n && o + ZXF_BLOCK_HDR <= size) {
                dp_prefetch(s + o - 4); /* the previous block's checksum trailer */
                dp_prefetch(s + o + ZXF_BLOCK_HDR - 1);
            }
            hint_off += __shfl_sync(FULL, inc, 31);
            hint_idx = hint_n - hint_idx < 32u ? hint_n : hint_idx + 32u;
        }
        const u64 rem = size - ip;
        u32 type, comp;
        if (rem < ZXF_BLOCK_HDR || !dp_block_header(s + ip, &type, &comp)) {
            end = ZXW_END_BAD_HEADER;
            break;
        }
        if (type == ZXF_BT_EOF) {
            end = comp == 0 ? ZXW_END_EOF : ZXW_END_BAD_HEADER;
            break;
        }
        const u64 on_disk = (u64)ZXF_BLOCK_HDR + comp + trailer;
        if (lane == 0 && n < J) { /* beyond the table only the count matters (zxc_dplan_decide) */
            zxc_b200_job_t Jb;
            Jb.src_off = ip;
            Jb.dst_off = 0;
            Jb.src_len = (u32)(on_disk < rem ? on_disk : (rem > 0xFFFFFFFFull ? 0xFFFFFFFFull : rem));
            Jb.dst_cap = 0;
            plan[n] = Jb;
        }
        n++;
        if (trailer && on_disk <= rem) g = dp_rotl(g, 1) ^ ld32(s + ip + ZXF_BLOCK_HDR + comp);
        if (on_disk >= rem) break;
        ip += on_disk;
    }
    if (lane != 0) return;
    S->n = n;
    S->end = end;
    S->ghash = g;
}

__global__ void zxc_dplan_walk(const DPlanArgs A) {
    DPlanState* S = A.st;
    if (S->done || S->fast) return;
    dp_walk(A.src, A.src_size, A.plan, A.J, S, threadIdx.x & 31);
}

/* regular plan: block i at i * block_size with its planned size, as far as dst_capacity goes */
__global__ void __launch_bounds__(DP_THREADS) zxc_dplan_place(const DPlanArgs A) {
    DPlanState* S = A.st;
    const bool done = S->done != 0;
    const u64 J = A.J;
    u64 n = 0, n_fit = 0;
    if (!done) {
        n = S->n;
        const u32 bs = S->block_size;
        if (n > 0) {
            const u64 k = A.dst_capacity / bs;
            n_fit = k < n - 1 ? k : (n - 1 + ((n - 1) * bs + dp_planned(S, n - 1, n) <= A.dst_capacity ? 1 : 0));
        }
    }
    const u64 i = (u64)blockIdx.x * DP_THREADS + threadIdx.x;
    if (i < J - n_fit) A.status[i] = 0; /* no stale deferral marks in front of the real jobs (see below) */
    if (i < n_fit) {
        zxc_b200_job_t Jb = A.plan[i];
        Jb.dst_off = i * S->block_size;
        Jb.dst_cap = dp_planned(S, i, n);
        A.jobs[J - n_fit + i] = Jb;
    }
    if (i == 0) {
        const u32 slot = done ? DP_SLOTS : (__ffs(S->block_size) - 1 - ZXC_BLOCK_SIZE_MIN_LOG2) * 2 + S->verify;
        /* counter 0 claims job indices (the first launch); counter 1 claims positions in the deferred-job list, or,
         * when the list overflowed, status words from 0 (those in front of the real jobs are 0, never deferred);
         * counter 2 is the list's length */
        for (u32 t = 0; t < DP_SLOTS; t++) {
            S->ctr[t][0] = t == slot ? J - n_fit : J;
            S->ctr[t][1] = 0;
            S->ctr[t][2] = 0;
        }
        S->split_ctr[0] = S->split_ctr[1] = 0;
        S->first_bad = ~0ull;
        S->n_fit = n_fit;
        S->produced = n_fit ? (n_fit - 1) * S->block_size + dp_planned(S, n_fit - 1, n) : 0;
    }
}

__global__ void __launch_bounds__(DP_THREADS) zxc_dplan_check(const DPlanArgs A) {
    DPlanState* S = A.st;
    if (S->done) return;
    const u64 n_fit = S->n_fit;
    const u64 i = (u64)blockIdx.x * DP_THREADS + threadIdx.x;
    if (i < n_fit) {
        const u64 k = A.J - n_fit + i;
        const i32 st = A.status[k];
        if (st < 0 || (u32)st != A.jobs[k].dst_cap) atomicMin(&S->first_bad, i);
    }
}

/* the general split needs every block in the job table: more blocks than it holds is this call's limit */
__device__ __forceinline__ void dp_split(const DPlanArgs& A, DPlanState* S) {
    if (S->n > A.J) {
        *A.result = ZXC_ERROR_MEMORY;
        S->done = 1;
    } else {
        S->split = 1;
    }
}

/* decompress_frame after the regular decode: first_failure, then the general split or the tail checks.  The regular
 * plan never holds more than J - 1 blocks (n_fit <= dst_capacity / block_size + 1), whatever the frame's length. */
__global__ void zxc_dplan_decide(const DPlanArgs A) {
    DPlanState* S = A.st;
    if (S->done) return;
    const u64 n = S->n, n_fit = S->n_fit;
    if (S->first_bad != ~0ull) {
        const i32 st = A.status[A.J - n_fit + S->first_bad];
        if (st >= 0 || st == ZXC_ERROR_OVERFLOW || st == ZXC_ERROR_DST_TOO_SMALL) {
            dp_split(A, S); /* the plan, not the block, may be at fault */
            return;
        }
        *A.result = st;
        S->done = 1;
        return;
    }
    if (n_fit < n && S->end == ZXW_END_EOF && S->footer_size <= A.dst_capacity) { /* short blocks may fit */
        dp_split(A, S);
        return;
    }
    *A.result = dp_tail(S, S->produced, n_fit == n);
    S->done = 1;
}

/* ---- general split (decompress_frame_any_split) ---- */
struct DSplitArgs {
    DPlanArgs a;
    u8* dst;
    u8* slots; /* probe_warps slots of `room` bytes */
    u8* scratch;
    const u8* dict;
    const u8* dict_huf;
    u32 dict_size, scratch_stride, room, probe_warps;
};

/* phase 0: every block that ran out of room (or was not decoded because it did not fit) is decoded alone into this
 * warp's slot of block_size + ZXF_TAIL_PAD bytes -- the room the reference gives a block -- and its size kept; the
 * bytes are thrown away.  Every other block's regular result is already its true size or its error.
 * phase 1: every block at its true offset in d_dst, from the job table zxc_dsplit_scan wrote. */
template <bool HAS_DICT>
__global__ void __launch_bounds__(CTA_THREADS) zxc_dsplit_decode(const DSplitArgs D, const u32 phase) {
    extern __shared__ __align__(16) u8 smem[];
    const DPlanArgs& A = D.a;
    DPlanState* S = A.st;
    if (!(phase == 0 ? S->split : S->redecode)) return;
    const u32 lane = threadIdx.x & 31;
    const u32 wic = threadIdx.x >> 5;
    const u32 gwarp = blockIdx.x * WARPS_PER_CTA + wic;
    if (phase == 0 && gwarp >= D.probe_warps) return;
    u8* scratch = D.scratch + (size_t)gwarp * D.scratch_stride + 256;
    u8* ring = smem + (size_t)wic * WARP_SMEM_BYTES;
#if ZXC_STAGE
    st_init(smem_addr(ring) + RING_BYTES, lane);
#endif
    DecodeParams P;
    P.src = A.src;
    P.dst = phase == 0 ? D.slots + (size_t)gwarp * D.room : D.dst;
    P.jobs = NULL;
    P.status = NULL;
    P.dict = D.dict;
    P.dict_huf = D.dict_huf;
    P.scratch = D.scratch;
    P.counter = NULL;
    P.n_jobs = 0;
    P.dict_size = D.dict_size;
    P.scratch_stride = D.scratch_stride;
    P.flags = S->verify ? FLAG_VERIFY : 0u;
    P.block_cap = S->block_size;
    P.defer_list = NULL;
    P.defer_count = NULL;
    P.defer_cap = 0;
    const u64 n = S->n, n_fit = S->n_fit, J = A.J;
    for (;;) {
        unsigned long long j = 0;
        if (lane == 0) j = atomicAdd(&S->split_ctr[phase], 1ull);
        j = __shfl_sync(FULL, j, 0);
        if (j >= n) break;
        zxc_b200_job_t job;
        if (phase == 0) {
            if (j < n_fit) {
                const i32 r = A.status[J - n_fit + j];
                if (r != ZXC_ERROR_OVERFLOW && r != ZXC_ERROR_DST_TOO_SMALL) {
                    if (lane == 0) A.sizes[j] = r;
                    continue;
                }
            }
            job = A.plan[j];
            job.dst_off = 0;
            job.dst_cap = D.room;
        } else {
            job = A.jobs[J - n + j];
        }
        const int r = decode_job<false, HAS_DICT, false>(P, job, scratch, ring, lane);
        flush_wait(lane); /* nothing of this block is still on its way out of the ring */
        __syncwarp();
        if (lane == 0) {
            if (phase == 0) A.sizes[j] = r;
            else A.status[J - n + j] = r;
        }
    }
}

/* the reference's order over the sizes: the first block with an error gives it, the first that does not fit the rest
 * of dst_capacity gives DST_TOO_SMALL; otherwise the job table for phase 1, right-aligned like the regular one */
__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dsplit_scan(const DPlanArgs A) {
    __shared__ unsigned long long s_fail;
    DPlanState* S = A.st;
    if (!S->split) return;
    const u64 n = S->n, J = A.J, cap = A.dst_capacity;
    if (threadIdx.x == 0) s_fail = ~0ull;
    unsigned long long carry = 0;
    for (u64 b = 0; b < n; b += blockDim.x) {
        const u64 i = b + threadIdx.x;
        const i32 v = i < n ? A.sizes[i] : 0;
        unsigned long long total;
        const u64 op = carry + asm_cta_excl(v > 0 ? (u64)v : 0ull, &total); /* its barriers also order s_fail */
        const bool err = i < n && v < 0;
        const bool over = i < n && v >= 0 && op <= cap && (u64)v > cap - op;
        if (err || over) atomicMin(&s_fail, i);
        __syncthreads();
        const u64 f = s_fail;
        if (f != ~0ull) {
            if (i == f) {
                *A.result = err ? (long long)v : (long long)ZXC_ERROR_DST_TOO_SMALL;
                S->done = 1;
            }
            return;
        }
        if (i < n) {
            zxc_b200_job_t Jb = A.plan[i];
            Jb.dst_off = op;
            Jb.dst_cap = (u32)v;
            A.jobs[J - n + i] = Jb;
        }
        carry += total;
    }
    if (threadIdx.x == 0) {
        S->produced = carry;
        S->redecode = carry > 0;
    }
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dsplit_final(const DPlanArgs A) {
    __shared__ unsigned long long s_bad;
    DPlanState* S = A.st;
    if (!S->split || S->done) return;
    const u64 n = S->n, J = A.J;
    if (threadIdx.x == 0) s_bad = ~0ull;
    __syncthreads();
    if (S->redecode) {
        for (u64 i = threadIdx.x; i < n; i += blockDim.x) {
            const i32 st = A.status[J - n + i];
            if (st < 0 || (u32)st != A.jobs[J - n + i].dst_cap) atomicMin(&s_bad, i);
        }
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    if (s_bad != ~0ull) {
        const i32 st = A.status[J - n + s_bad];
        *A.result = st < 0 ? st : ZXC_ERROR_CORRUPT_DATA;
    } else {
        *A.result = dp_tail(S, S->produced, true);
    }
    S->done = 1;
}
