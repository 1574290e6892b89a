/*
 * zxc_dplan.cuh -- frame decode with the frame in HBM (zxc_b200_decompress_device): the frame walk, the job table and
 * zxc_decompress's verdict on the device, on the caller's stream, with no host round trip.  Stream order:
 *
 *   zxc_dplan_probe       one thread: dp_probe -- the dst_capacity == 0 shortcut, the file-header checks of
 *                         zxf_read_file_header, the scratch's block-size limit, the dictionary verdicts, the footer,
 *                         and the SEK table probe of zxw_walk's prefetch hint
 *   zxc_dplan_sek_tiles   \  SEK-guided plan: tile sums of the table's sizes, one CTA's scan of them into predicted
 *   zxc_dplan_sek_scan     | header offsets (dp_sek_closes: the chain's end at the EOF block), then per tile
 *   zxc_dplan_sek_blocks  /  dp_sek_tile: the header at each predicted offset, its plan entry and its global-hash
 *                            term; any disagreement with what the sequential walk would see clears `fast`
 *   zxc_dplan_walk        one warp: dp_walk (zxw_walk), for frames without a table or when `fast` was cleared
 *   zxc_dplan_place       the regular plan (dp_n_fit, dp_fit): its first n_fit blocks into the decode job table,
 *                         right-aligned in [J - n_fit, J), and the work counters of every launch slot (dp_preset)
 *   zxc_decode_kernel     (zxc_decode.cuh, unchanged) one launch_decode per slot; only the frame's slot has work
 *   zxc_dplan_check       first job that did not produce its planned size
 *   zxc_dplan_decide      dp_decide: decompress_frame's order -- block error, plan mismatch, capacity, EOF, footer,
 *                         global hash
 *   zxc_dsplit_decode     general split, phase 0: the size of every block that ran out of room, in a per-warp slot
 *   zxc_dsplit_scan       dp_split_scan: true offsets in the reference's order (a block's error, then whether it fits)
 *   zxc_dsplit_decode     phase 1: every block at its true offset
 *   zxc_dsplit_final      dp_split_final: the split's verdict
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

/* one frame's plan and verdict, shared by the single-frame, in-place and batched calls.  The bodies below that read
 * the frame take its bytes as an argument: a kernel parameter where there is one, which the compiler takes for a
 * global pointer, so their loads stay global loads. */
struct DFrame {
    unsigned long long src_size, cap; /* cap: dst_capacity */
    unsigned long long n;             /* blocks ahead of the end of the block stream */
    unsigned long long n_fit;         /* the regular plan's blocks that fit cap */
    unsigned long long produced;
    unsigned long long footer_size;
    unsigned long long first_bad; /* the first regular job in stream order that failed */
    unsigned long long sek_pos;   /* offset of the SEK table's first entry */
    unsigned long long eof_pos;   /* where the table says the EOF block is */
    unsigned int J;               /* its job table's entries */
    unsigned int hint_n;          /* SEK entries (0: no table) */
    unsigned int block_size, has_checksum, verify, end, footer_hash, ghash;
    unsigned int fast;     /* the SEK-guided plan holds */
    unsigned int done;     /* its result is written */
    unsigned int split;    /* the general split runs */
    unsigned int redecode; /* the split's second decode has work */
};

/* the first bytes of the caller's scratch (DP_STATE_BYTES) */
struct DPlanState : DFrame {
    unsigned long long ctr[DP_SLOTS][4]; /* per launch slot: the decode's three work counters (launch_decode) */
    unsigned long long split_ctr[2];     /* zxc_dsplit_decode's work counters, phase 0 and 1 */
};
#define DP_STATE_BYTES 1024
static_assert(sizeof(DPlanState) <= DP_STATE_BYTES, "DPlanState fits its region");

/* the call's decode options, from the host */
struct DDecodeOpts {
    unsigned int max_block_size; /* the scratch's block size */
    unsigned int dict_id;        /* zxc_dict_id of the caller's dictionary */
    unsigned int have_dict;      /* a dictionary was given */
    int huf_verdict;             /* dict_huf_attach of its table: 1 usable, 0 none, < 0 malformed */
    unsigned int checksum_enabled;
};

struct DPlanArgs {
    const u8* src;
    unsigned long long src_size, dst_capacity;
    zxc_b200_job_t* plan; /* J entries: the walk's src_off / src_len per block; the split's phase-1 jobs */
    zxc_b200_job_t* jobs; /* J entries: the decode job table, real jobs right-aligned */
    i32* status;          /* J entries, indexed like jobs */
    i32* sizes;           /* J entries: the split's true block sizes or errors, then its phase-1 status */
    unsigned long long* tiles;
    DPlanState* st;
    long long* result;
    unsigned int J;
    DDecodeOpts o;
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
__device__ __forceinline__ u32 dp_planned(const DFrame* F, u64 i, u64 n) {
    const u32 bs = F->block_size;
    if (i + 1 < n) return bs;
    const u64 start = i * bs;
    const u64 f = F->footer_size;
    const u32 e = f <= start ? 0u : (f - start >= bs ? bs : (u32)(f - start));
    return e ? e : bs;
}

/* decompress_frame's checks behind the decode (the `decoded:` label) */
__device__ __forceinline__ long long dp_tail(const DFrame* F, u64 produced, bool all_fit) {
    if (!all_fit) return ZXC_ERROR_DST_TOO_SMALL;
    if (F->end == ZXW_END_BAD_HEADER) return ZXC_ERROR_BAD_HEADER;
    if (F->end == ZXW_END_EOF) {
        if (F->footer_size != produced) return ZXC_ERROR_CORRUPT_DATA;
        if (F->verify && F->footer_hash != F->ghash) return ZXC_ERROR_BAD_CHECKSUM;
    }
    return (long long)produced;
}

__device__ __forceinline__ void dp_prefetch(const u8* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

/* zxf_read_file_header's rejects of the 16 header bytes at s, in its order; 1 when the header holds.  dp_probe makes
 * the same checks inline, interleaved with its own: calling this from there changed its code generation. */
__device__ __forceinline__ long long dp_file_header(const u8* s) {
    if (ld32(s) != ZXF_MAGIC) return ZXC_ERROR_BAD_MAGIC;
    if (s[4] != ZXF_VERSION) return ZXC_ERROR_BAD_VERSION;
    if (ld16(s + 14) != dp_hash16(ld64(s), ld64(s + 8) & 0x0000FFFFFFFFFFFFull) || (s[6] & 0x0Fu) != 0)
        return ZXC_ERROR_BAD_HEADER;
    if (s[5] < ZXC_BLOCK_SIZE_MIN_LOG2 || s[5] > ZXC_BLOCK_SIZE_MAX_LOG2) return ZXC_ERROR_BAD_BLOCK_SIZE;
    return 1;
}

/* the probe of frame s, of size >= header + footer, whose src_size, cap and J are set */
__device__ __forceinline__ void dp_probe(const DDecodeOpts& o, const u8* s, DFrame* F, long long* result) {
    const u64 size = F->src_size; /* >= header + footer: checked before (on the host, or by zxc_dbatch_tiles) */
    F->done = F->fast = F->split = F->redecode = 0;
    F->hint_n = 0;
    F->ghash = 0;
    F->n = 0;
    F->end = ZXW_END_RAN_OFF;
    const u64 footer = ld64(s + size - ZXC_FILE_FOOTER_SIZE);
    F->footer_size = footer;
    F->footer_hash = ld32(s + size - 4);
    long long v = 1; /* 1: undecided */
    u32 bs = 0;
    if (F->cap == 0) { /* the empty-frame shortcut of decompress_entry */
        v = ld32(s) != ZXF_MAGIC ? ZXC_ERROR_BAD_MAGIC : (footer == 0 ? 0 : ZXC_ERROR_DST_TOO_SMALL);
    } else if (ld32(s) != ZXF_MAGIC) {
        v = ZXC_ERROR_BAD_MAGIC;
    } else if (s[4] != ZXF_VERSION) {
        v = ZXC_ERROR_BAD_VERSION;
    } else if (ld16(s + 14) != dp_hash16(ld64(s), ld64(s + 8) & 0x0000FFFFFFFFFFFFull) || (s[6] & 0x0Fu) != 0) {
        v = ZXC_ERROR_BAD_HEADER;
    } else if (s[5] < ZXC_BLOCK_SIZE_MIN_LOG2 || s[5] > ZXC_BLOCK_SIZE_MAX_LOG2) {
        v = ZXC_ERROR_BAD_BLOCK_SIZE;
    } else if ((1u << s[5]) > o.max_block_size) {
        v = ZXC_ERROR_MEMORY; /* the scratch was sized for smaller blocks */
    } else {
        bs = 1u << s[5];
        const u32 did = (s[6] & ZXF_FLAG_DICT) ? ld32(s + 7) : 0u;
        if (did != 0 && !o.have_dict) v = ZXC_ERROR_DICT_REQUIRED;
        else if (did != 0 && o.dict_id != did) v = ZXC_ERROR_DICT_MISMATCH;
        else if (o.have_dict && o.huf_verdict < 0) v = o.huf_verdict;
    }
    if (v != 1) {
        *result = v;
        F->done = 1;
        return;
    }
    F->block_size = bs;
    F->has_checksum = (s[6] & ZXF_FLAG_CHECKSUM) ? 1u : 0u;
    F->verify = F->has_checksum && o.checksum_enabled;
    /* zxw_walk's prefetch hint: a SEK block header where a table for the footer's size would start */
    if (footer > 0) {
        const u64 nb = (footer + bs - 1) / bs;
        const u64 sek_total = ZXF_BLOCK_HDR + nb * ZXF_SEEK_ENTRY;
        if (nb <= 0xFFFFFFFFull && sek_total + ZXC_FILE_FOOTER_SIZE + ZXC_FILE_HEADER_SIZE <= size) {
            const u64 sp = size - ZXC_FILE_FOOTER_SIZE - sek_total;
            if (s[sp] == ZXF_BT_SEK && ld32(s + sp + 3) == (u32)(nb * ZXF_SEEK_ENTRY)) {
                F->hint_n = (u32)nb;
                F->sek_pos = sp + ZXF_BLOCK_HDR;
                F->eof_pos = sp - ZXF_BLOCK_HDR;
                F->fast = nb <= F->J;
            }
        }
    }
}

/* SEK-guided plan: the chain closes at the EOF block in front of the table (the table's entries sum to `sum`), and
 * that block is a valid empty EOF */
__device__ __forceinline__ bool dp_sek_closes(const DFrame* F, const u8* src, u64 sum) {
    u32 type = 0, comp = 1;
    return ZXC_FILE_HEADER_SIZE + sum == F->eof_pos && dp_block_header(src + F->eof_pos, &type, &comp) &&
           type == ZXF_BT_EOF && comp == 0;
}

/* SEK-guided plan, one tile of ASM_TILE entries per CTA: this thread's ASM_ITEMS entries from `first`, the tile's
 * first block at frame offset off0.  Each block's header at its predicted offset, its plan entry and its global-hash
 * term (XORed into *h); false on any disagreement with what the sequential walk would see.  *total: the tile's sum.
 * Every offset lies in front of the EOF block (dp_sek_closes checked the sum), so the 8 header bytes are there. */
__device__ __forceinline__ bool dp_sek_tile(const DFrame* F, const u8* src, u64 first, u64 off0, zxc_b200_job_t* plan,
                                            u32* h, unsigned long long* total) {
    const u32 nb = F->hint_n;
    const u8* e = src + F->sek_pos;
    u32 c[ASM_ITEMS];
    u64 s = 0;
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        c[k] = first + k < nb ? ld32(e + 4 * (first + k)) : 0u;
        s += c[k];
    }
    u64 off = off0 + asm_cta_excl(s, total);
    const u32 trailer = F->has_checksum ? ZXF_BLOCK_CKS : 0u;
    bool ok = true;
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        const u64 j = first + k;
        if (j >= nb) break;
        u32 type, comp;
        if (!dp_block_header(src + off, &type, &comp) || type > ZXF_BT_GHI ||
            (u64)ZXF_BLOCK_HDR + comp + trailer != c[k]) {
            ok = false;
        } else {
            zxc_b200_job_t Jb;
            Jb.src_off = off;
            Jb.dst_off = 0;
            Jb.src_len = c[k];
            Jb.dst_cap = 0;
            plan[j] = Jb;
            if (trailer) *h ^= dp_rotl(ld32(src + off + ZXF_BLOCK_HDR + comp), (u32)((nb - 1 - j) & 31u));
        }
        off += c[k];
    }
    return ok;
}

/* a warp's global-hash terms into the frame's */
__device__ __forceinline__ void dp_ghash_xor(DFrame* F, u32 h) {
    for (u32 d = 16; d; d >>= 1) h ^= __shfl_xor_sync(FULL, h, d);
    if ((threadIdx.x & 31) == 0 && h) atomicXor(&F->ghash, h);
}

__global__ void zxc_dplan_probe(const DPlanArgs A) {
    DPlanState* S = A.st;
    S->src_size = A.src_size;
    S->cap = A.dst_capacity;
    S->J = A.J;
    dp_probe(A.o, A.src, S, A.result);
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
        if (dp_sek_closes(S, A.src, carry)) {
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
    if ((u64)blockIdx.x * ASM_TILE >= S->hint_n) return;
    u32 h = 0;
    unsigned long long total;
    const bool ok = dp_sek_tile(S, A.src, (u64)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS,
                                ZXC_FILE_HEADER_SIZE + A.tiles[blockIdx.x], A.plan, &h, &total);
    dp_ghash_xor(S, h);
    if (!ok) S->fast = 0;
}

/* zxw_walk, warp-uniform: every lane follows the chain (the header loads are broadcasts), lane 0 stores.  With a SEK
 * table the lanes prefetch the next 32 predicted headers into L2, a window ahead of the walk, like the host walk; a
 * wrong or forged table only prefetches the wrong lines.  Blocks beyond the J plan entries are counted, not stored.
 * The frame's size and J come as arguments like its bytes: kernel parameters in zxc_dplan_walk, where this loop of
 * dependent loads ran 2 % slower with them read from the record. */
__device__ __forceinline__ void dp_walk(DFrame* F, const u8* s, const u64 size, const u32 J, zxc_b200_job_t* plan,
                                        const u32 lane) {
    const u32 trailer = F->has_checksum ? ZXF_BLOCK_CKS : 0u;
    const u32 hint_n = F->hint_n;
    const u8* he = s + F->sek_pos;
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
        if (lane == 0 && n < J) { /* beyond the table only the count matters (dp_decide) */
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
    F->n = n;
    F->end = end;
    F->ghash = g;
}

__global__ void zxc_dplan_walk(const DPlanArgs A) {
    DPlanState* S = A.st;
    if (S->done || S->fast) return;
    dp_walk(S, A.src, A.src_size, A.J, A.plan, threadIdx.x & 31);
}

/* the regular plan: block i at i * block_size with its planned size, as far as cap goes */
__device__ __forceinline__ u64 dp_n_fit(const DFrame* F) {
    const u64 n = F->n;
    if (n == 0) return 0;
    const u32 bs = F->block_size;
    const u64 k = F->cap / bs;
    return k < n - 1 ? k : (n - 1 + ((n - 1) * bs + dp_planned(F, n - 1, n) <= F->cap ? 1 : 0));
}

/* the regular plan's n_fit, what it produces, and no failed job yet */
__device__ __forceinline__ void dp_fit(DFrame* F, u64 n_fit) {
    F->first_bad = ~0ull;
    F->n_fit = n_fit;
    F->produced = n_fit ? (n_fit - 1) * F->block_size + dp_planned(F, n_fit - 1, F->n) : 0;
}

/* the frame's decode launch slot: one per (block size, checksum verification) */
__device__ __forceinline__ u32 dp_slot(const DFrame* F) {
    return (__ffs(F->block_size) - 1 - ZXC_BLOCK_SIZE_MIN_LOG2) * 2 + F->verify;
}

/* a launch slot's work counters, its first real job at `first`: counter 0 claims job indices (the first launch);
 * counter 1 claims positions in the deferred-job list, or, when the list overflowed, status words from 0 (those in
 * front of the real jobs are 0, never deferred); counter 2 is the list's length */
__device__ __forceinline__ void dp_preset(unsigned long long* ctr, u64 first) {
    ctr[0] = first;
    ctr[1] = 0;
    ctr[2] = 0;
}

__global__ void __launch_bounds__(DP_THREADS) zxc_dplan_place(const DPlanArgs A) {
    DPlanState* S = A.st;
    const bool done = S->done != 0;
    const u64 J = A.J;
    const u64 n = done ? 0 : S->n;
    const u64 n_fit = done ? 0 : dp_n_fit(S);
    const u64 i = (u64)blockIdx.x * DP_THREADS + threadIdx.x;
    if (i < J - n_fit) A.status[i] = 0; /* no stale deferral marks in front of the real jobs (dp_preset) */
    if (i < n_fit) {
        zxc_b200_job_t Jb = A.plan[i];
        Jb.dst_off = i * S->block_size;
        Jb.dst_cap = dp_planned(S, i, n);
        A.jobs[J - n_fit + i] = Jb;
    }
    if (i == 0) {
        const u32 slot = done ? DP_SLOTS : dp_slot(S);
        for (u32 t = 0; t < DP_SLOTS; t++) dp_preset(S->ctr[t], t == slot ? J - n_fit : J);
        S->split_ctr[0] = S->split_ctr[1] = 0;
        dp_fit(S, n_fit);
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

/* decompress_frame after the regular decode: first_failure (bad_status: the status of regular job first_bad, when
 * there is one), then the general split or the tail checks.  True when the frame goes to the general split, which
 * needs every block in the frame's job table: more blocks than it holds is the call's limit.  The regular plan never
 * holds more than J - 1 blocks (n_fit <= cap / block_size + 1), whatever the frame's length. */
__device__ __forceinline__ bool dp_decide(DFrame* F, i32 bad_status, long long* result) {
    const u64 n = F->n, n_fit = F->n_fit;
    bool split;
    long long v;
    if (F->first_bad != ~0ull) {
        v = bad_status;
        split = v >= 0 || v == ZXC_ERROR_OVERFLOW || v == ZXC_ERROR_DST_TOO_SMALL; /* the plan may be at fault */
    } else {
        split = n_fit < n && F->end == ZXW_END_EOF && F->footer_size <= F->cap; /* short blocks may fit */
        if (!split) v = dp_tail(F, F->produced, n_fit == n);
    }
    if (split && n <= F->J) {
        F->split = 1;
        return true;
    }
    *result = split ? ZXC_ERROR_MEMORY : v;
    F->done = 1;
    return false;
}

__global__ void zxc_dplan_decide(const DPlanArgs A) {
    DPlanState* S = A.st;
    if (S->done) return;
    const u64 fb = S->first_bad;
    dp_decide(S, fb != ~0ull ? A.status[A.J - S->n_fit + fb] : 0, A.result);
}

/* ---- general split (decompress_frame_any_split) ----
 * Phase 0: every block that ran out of room (or was not decoded because it did not fit) is decoded alone into a
 * warp's slot of block_size + ZXF_TAIL_PAD bytes -- the room the reference gives a block -- and its size kept in the
 * frame's `sizes`; the bytes are thrown away.  Every other block's regular result is already its true size or its
 * error.  The scan then rewrites the frame's plan entries into phase 1's jobs, and phase 1 decodes every block at its
 * true offset with its status in `sizes`. */
struct DSplitArgs {
    const u8* src; /* the base of the plan's source offsets */
    u8* dst;       /* the base of phase 1's destination offsets */
    u8* slots;     /* probe_warps slots of `room` bytes */
    u8* scratch;
    const u8* dict;
    const u8* dict_huf;
    u32 dict_size, scratch_stride, room, probe_warps;
};

/* the split decode's per-warp set-up; false for a warp without a phase-0 slot.  The bases are kernel parameters,
 * which the compiler takes for global pointers, so the decode body keeps its global loads and stores (DESIGN.md
 * section 7h). */
__device__ __forceinline__ bool dp_split_warp(const DSplitArgs& D, u32 phase, u8* smem, DecodeParams* P, u8** scratch,
                                              u8** ring) {
    const u32 wic = threadIdx.x >> 5;
    const u32 gwarp = blockIdx.x * WARPS_PER_CTA + wic;
    if (phase == 0 && gwarp >= D.probe_warps) return false;
    *scratch = D.scratch + (size_t)gwarp * D.scratch_stride + 256;
    *ring = smem + (size_t)wic * WARP_SMEM_BYTES;
#if ZXC_STAGE
    st_init(smem_addr(*ring) + RING_BYTES, threadIdx.x & 31);
#endif
    P->src = D.src;
    P->dst = phase == 0 ? D.slots + (size_t)gwarp * D.room : D.dst;
    P->jobs = NULL;
    P->status = NULL;
    P->dict = D.dict;
    P->dict_huf = D.dict_huf;
    P->scratch = D.scratch;
    P->counter = NULL;
    P->n_jobs = 0;
    P->dict_size = D.dict_size;
    P->scratch_stride = D.scratch_stride;
    P->defer_list = NULL;
    P->defer_count = NULL;
    P->defer_cap = 0;
    return true;
}

/* one block of frame F alone, its plan entry `job` (phase 0: into the warp's slot, its source offset taken from
 * src_base); nothing of it is still on its way out of the ring when this returns */
template <bool HAS_DICT>
__device__ __forceinline__ int dp_split_block(DecodeParams& P, const DSplitArgs& D, const DFrame& F,
                                              zxc_b200_job_t job, u64 src_base, u32 phase, u8* scratch, u8* ring,
                                              u32 lane) {
    if (phase == 0) {
        job.src_off += src_base;
        job.dst_off = 0;
        job.dst_cap = D.room;
    }
    P.flags = F.verify ? FLAG_VERIFY : 0u;
    P.block_cap = F.block_size;
    const int r = decode_job<false, HAS_DICT, false>(P, job, scratch, ring, lane);
    flush_wait(lane);
    __syncwarp();
    return r;
}

/* one CTA over a split frame's phase-0 sizes, in the reference's order: the first block with an error gives it, the
 * first that does not fit the rest of cap gives DST_TOO_SMALL; otherwise the plan entries become phase 1's jobs, at
 * src_base + src_off and dst_base + their true offset.  True (in every thread) when phase 1 has work. */
__device__ __forceinline__ bool dp_split_scan(DFrame* F, zxc_b200_job_t* plan, const i32* sizes, u64 src_base,
                                              u64 dst_base, long long* result) {
    __shared__ unsigned long long s_fail;
    const u64 n = F->n, cap = F->cap;
    if (threadIdx.x == 0) s_fail = ~0ull;
    unsigned long long carry = 0;
    for (u64 b = 0; b < n; b += blockDim.x) {
        const u64 i = b + threadIdx.x;
        const i32 v = i < n ? sizes[i] : 0;
        unsigned long long total;
        const u64 op = carry + asm_cta_excl(v > 0 ? (u64)v : 0ull, &total); /* its barriers also order s_fail */
        const bool err = i < n && v < 0;
        const bool over = i < n && v >= 0 && op <= cap && (u64)v > cap - op;
        if (err || over) atomicMin(&s_fail, i);
        __syncthreads();
        const u64 f = s_fail;
        if (f != ~0ull) {
            if (i == f) {
                *result = err ? (long long)v : (long long)ZXC_ERROR_DST_TOO_SMALL;
                F->done = 1;
            }
            return false;
        }
        if (i < n) {
            zxc_b200_job_t Jb = plan[i];
            Jb.src_off += src_base;
            Jb.dst_off = dst_base + op;
            Jb.dst_cap = (u32)v;
            plan[i] = Jb;
        }
        carry += total;
    }
    if (threadIdx.x == 0) {
        F->produced = carry;
        F->redecode = carry > 0;
    }
    return carry > 0;
}

/* one CTA: a split frame's verdict after phase 1 */
__device__ __forceinline__ void dp_split_final(DFrame* F, const zxc_b200_job_t* plan, const i32* sizes,
                                               long long* result) {
    __shared__ unsigned long long s_bad;
    const u64 n = F->n;
    if (threadIdx.x == 0) s_bad = ~0ull;
    __syncthreads();
    if (F->redecode) {
        for (u64 i = threadIdx.x; i < n; i += blockDim.x) {
            const i32 st = sizes[i];
            if (st < 0 || (u32)st != plan[i].dst_cap) atomicMin(&s_bad, i);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (s_bad != ~0ull) {
            const i32 st = sizes[s_bad];
            *result = st < 0 ? st : ZXC_ERROR_CORRUPT_DATA;
        } else {
            *result = dp_tail(F, F->produced, true);
        }
        F->done = 1;
    }
}

/* phase 0 and phase 1 over the frame, one job per claim */
template <bool HAS_DICT>
__global__ void __launch_bounds__(CTA_THREADS) zxc_dsplit_decode(const DPlanArgs A, const DSplitArgs D,
                                                                  const u32 phase) {
    extern __shared__ __align__(16) u8 smem[];
    DPlanState* S = A.st;
    if (!(phase == 0 ? S->split : S->redecode)) return;
    DecodeParams P;
    u8 *scratch, *ring;
    if (!dp_split_warp(D, phase, smem, &P, &scratch, &ring)) return;
    const u32 lane = threadIdx.x & 31;
    const u64 n = S->n, n_fit = S->n_fit, J = A.J;
    for (;;) {
        unsigned long long j = 0;
        if (lane == 0) j = atomicAdd(&S->split_ctr[phase], 1ull);
        j = __shfl_sync(FULL, j, 0);
        if (j >= n) break;
        if (phase == 0 && j < n_fit) {
            const i32 r = A.status[J - n_fit + j];
            if (r != ZXC_ERROR_OVERFLOW && r != ZXC_ERROR_DST_TOO_SMALL) {
                if (lane == 0) A.sizes[j] = r;
                continue;
            }
        }
        const int r = dp_split_block<HAS_DICT>(P, D, *S, A.plan[j], 0, phase, scratch, ring, lane);
        if (lane == 0) A.sizes[j] = r;
    }
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dsplit_scan(const DPlanArgs A) {
    DPlanState* S = A.st;
    if (!S->split) return;
    dp_split_scan(S, A.plan, A.sizes, 0, 0, A.result);
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dsplit_final(const DPlanArgs A) {
    DPlanState* S = A.st;
    if (!S->split || S->done) return;
    dp_split_final(S, A.plan, A.sizes, A.result);
}
