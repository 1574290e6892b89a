/*
 * zxc_dindex.cuh -- a SEK table for a frame in HBM (zxc_b200_add_seek_table_device): the frame's block chain found on
 * the device in parallel, proven against the sequential walk, and the table written in place, on the caller's stream.
 * Stream order:
 *
 *   zxc_dindex_probe    one thread: the file-header checks of zxf_read_file_header (dp_file_header), the footer
 *   zxc_dindex_count    per tile of DI_TILE frame offsets: the candidate headers (di_candidate) it holds
 *   zxc_dindex_tscan    one CTA: the tiles' counts into exclusive prefixes; more than C candidates abandons the guess
 *   zxc_dindex_emit     per tile again: its candidates' offsets and on-disk sizes, in offset order, into the list
 *   zxc_dindex_links    per candidate: its successor, the candidate at offset + on-disk size (binary search), and the
 *                       start mark on the candidate at offset 16
 *   zxc_dindex_round    DI_ROUNDS launches of pointer doubling: a marked node marks its 2^r-th successor, and the jump
 *                       table squares; after round r the first 2^(r+1) nodes of the chain from offset 16 are marked
 *   zxc_dindex_mtiles   \  the marked data blocks compacted in offset order into the plan (ASM_TILE candidates per
 *   zxc_dindex_mscan     | CTA, one CTA's scan of the tile sums), and the marked EOF block
 *   zxc_dindex_memit    /
 *   zxc_dindex_prove    per plan entry: the proof that the sequential walk visits exactly these offsets (entry 0 at
 *                       16, a valid header of a data type, entry j + its on-disk size = entry j + 1, the last one
 *                       followed by a valid empty EOF block); any failure clears `fast`
 *   zxc_dindex_walk     one warp: dp_walk (zxw_walk) when the guess was abandoned or failed its proof
 *   zxc_dindex_check    per plan entry: a block type other than RAW, GLO or GHI; the tail's table against the plan
 *   zxc_dindex_decide   one thread: the verdict, in the order of zxc_b200.h
 *   zxc_dindex_write    per plan entry: the SEK table at the old footer's offset, then the footer behind it
 * Every kernel after the probe exits at once when the result is written or its stage is not needed, so the launch
 * sequence is the same for every frame.  Nothing is written into the frame before zxc_dindex_decide has accepted it.
 *
 * The speculation keeps every offset p whose 8 bytes pass the block-header CRC, whose type is RAW, GLO, GHI or an empty
 * EOF, and whose data block is at most block_size + 12 bytes on disk (the largest block the reference's encoder
 * writes) and leaves room for an EOF header in front of the footer.  A real chain of such blocks is among them; a
 * chain with a longer block, or a list past its capacity, only sends the frame to the walk.
 */
#pragma once
#include <cuda_runtime.h>

#include "zxc_assemble.cuh"
#include "zxc_dplan.cuh"

#define DI_THREADS 256
#define DI_TILE 8192                             /* frame offsets per CTA of the candidate scan */
#define DI_WARP_SPAN (DI_TILE / (DI_THREADS / 32)) /* offsets per warp: DI_STEPS steps of 32 four-byte words */
#define DI_STEPS (DI_WARP_SPAN / 128)
#define DI_ROUNDS 30 /* 2^30 > any candidate count: C < 2^30 */
#define DI_NONE 0xFFFFFFFFu
#define DI_SCAN_ITEMS 8
#define DI_GRID_MAX 2048 /* CTAs of the grid-stride kernels over the candidates and the plan */

enum { DI_PATH_NONE = 0, DI_PATH_SPEC = 1, DI_PATH_WALK = 2 };

/* the first bytes of the caller's scratch; `path` at offset 0 tells which path decided the chain */
struct DIdxState {
    unsigned int path;       /* DI_PATH_*: 0 when the frame was rejected before its chain was known */
    unsigned int write;      /* zxc_dindex_write has work */
    unsigned int bad_type;   /* a block of the chain is not RAW, GLO or GHI */
    unsigned int table_diff; /* the tail's table entries differ from the chain's sizes */
    unsigned long long m;    /* candidates found (may exceed C) */
    unsigned long long eof_pos;
    DFrame F; /* src_size, block_size, has_checksum, footer_size / footer_hash (the old footer), and the chain:
               * n, end, fast (the guess holds), done (the result is written) */
};
#define DI_STATE_BYTES 256
static_assert(sizeof(DIdxState) <= DI_STATE_BYTES, "DIdxState fits its region");

struct DIdxArgs {
    u8* buf;                   /* the frame; read until zxc_dindex_write */
    unsigned long long size;   /* frame_size */
    unsigned long long cap;    /* buffer_capacity */
    DIdxState* st;
    unsigned long long* tiles; /* per scan tile: its candidates, then their exclusive prefix */
    unsigned long long* off;   /* C candidates: frame offsets, ascending */
    unsigned int* len;         /* their on-disk sizes; 0 for an EOF block */
    unsigned int* jump[2];     /* the jump tables, read and written in turn */
    unsigned char* mark;       /* on the chain from offset 16 */
    unsigned long long* mtiles; /* per ASM_TILE candidates: marked data blocks, then their exclusive prefix */
    zxc_b200_job_t* plan;       /* J entries: src_off / src_len per block of the chain */
    long long* result;
    unsigned int C, J, n_tiles;
};

/* a candidate header at frame offset p, its 8 bytes at q: *len its on-disk size, 0 for an empty EOF block */
__device__ __forceinline__ bool di_candidate(const u8* q, u64 p, u64 size, u32 bs, u32 trailer, u32* len) {
    u32 type, comp;
    if (!dp_block_header(q, &type, &comp)) return false;
    if (type == ZXF_BT_EOF) {
        *len = 0;
        return comp == 0;
    }
    const u64 od = (u64)ZXF_BLOCK_HDR + comp + trailer;
    if (type > ZXF_BT_GHI || od > (u64)bs + ZXF_BLOCK_HDR + ZXF_BLOCK_CKS ||
        p + od + ZXF_BLOCK_HDR > size - ZXC_FILE_FOOTER_SIZE)
        return false;
    *len = (u32)od;
    return true;
}

/* the tile's bytes [t0, t0 + DI_TILE + 7) (as far as they lie in front of the footer) into sm, shifted by the
 * frame's misalignment: frame offset p is at sm[p - t0 + *mis].  16-byte loads where a chunk lies wholly inside, the
 * edges byte by byte: nothing outside the frame is read. */
__device__ __forceinline__ void di_load(const DIdxArgs& A, u64 t0, u8* sm, u32* mis) {
    const u64 end = A.size - ZXC_FILE_FOOTER_SIZE;
    const u64 hi = t0 + DI_TILE + 7 < end ? t0 + DI_TILE + 7 : end;
    const uintptr_t a = (uintptr_t)(A.buf + t0), a0 = a & ~(uintptr_t)15, ahi = (uintptr_t)(A.buf + hi);
    *mis = (u32)(a - a0);
    const u32 chunks = (u32)((ahi - a0 + 15) / 16);
    for (u32 c = threadIdx.x; c < chunks; c += DI_THREADS) {
        const uintptr_t ca = a0 + 16u * c;
        if (ca >= a && ca + 16 <= ahi) {
            *(uint4*)(sm + 16u * c) = __ldcs((const uint4*)ca);
        } else {
#pragma unroll
            for (u32 i = 0; i < 16; i++) sm[16u * c + i] = (ca + i >= a && ca + i < ahi) ? *(const u8*)(ca + i) : 0;
        }
    }
    __syncthreads();
}

/* step k of this lane: the candidate bits of its 4 offsets (bit j: offset t0 + rel + j), *rel set.  A byte can only
 * start a candidate when it reads 0, 1, 2 or 255: (b + 1) mod 256 <= 3 for all four bytes at once. */
__device__ __forceinline__ u32 di_word(const DIdxArgs& A, const u8* sm, u32 mis, u64 t0, u32 k, u32 bs, u32 trailer,
                                       u32* rel, u32* lens) {
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    *rel = warp * DI_WARP_SPAN + k * 128 + lane * 4;
    const u32 i = mis + *rel;
    const u32* sw = (const u32*)sm;
    const u32 w = __funnelshift_r(sw[i >> 2], sw[(i >> 2) + 1], (i & 3) * 8);
    const u32 hit = __vcmpleu4(__vadd4(w, 0x01010101u), 0x03030303u);
    u32 bits = 0;
    if (hit) {
        const u64 lim = A.size - ZXC_FILE_FOOTER_SIZE - ZXF_BLOCK_HDR; /* p <= lim: the header lies in front */
#pragma unroll
        for (u32 j = 0; j < 4; j++) {
            const u64 p = t0 + *rel + j;
            if (((hit >> (8 * j)) & 0xFFu) && p >= ZXC_FILE_HEADER_SIZE && p <= lim &&
                di_candidate(sm + i + j, p, A.size, bs, trailer, &lens[j]))
                bits |= 1u << j;
        }
    }
    return bits;
}

__device__ __forceinline__ u32 di_trailer(const DFrame* F) { return F->has_checksum ? ZXF_BLOCK_CKS : 0u; }

/* one tile's candidates, counted by warp: the lane's count over its DI_STEPS words */
__device__ __forceinline__ u32 di_count_lane(const DIdxArgs& A, const u8* sm, u32 mis, u64 t0, u32 bs, u32 trailer) {
    u32 c = 0;
    for (u32 k = 0; k < DI_STEPS; k++) {
        u32 rel, lens[4];
        c += __popc(di_word(A, sm, mis, t0, k, bs, trailer, &rel, lens));
    }
    return c;
}

__global__ void zxc_dindex_probe(const DIdxArgs A) {
    DIdxState* S = A.st;
    DFrame* F = &S->F;
    const u8* s = A.buf;
    S->path = DI_PATH_NONE;
    S->write = S->bad_type = S->table_diff = 0;
    S->m = 0;
    S->eof_pos = ~0ull;
    F->src_size = A.size;
    F->done = F->split = F->redecode = 0;
    F->fast = 1;
    F->hint_n = 0;
    F->sek_pos = 0;
    F->n = 0;
    F->end = ZXW_END_RAN_OFF;
    F->ghash = 0;
    F->footer_size = ld64(s + A.size - ZXC_FILE_FOOTER_SIZE);
    F->footer_hash = ld32(s + A.size - 4);
    const long long v = dp_file_header(s);
    if (v != 1) {
        *A.result = v;
        F->done = 1;
        return;
    }
    F->block_size = 1u << s[5];
    F->has_checksum = (s[6] & ZXF_FLAG_CHECKSUM) ? 1u : 0u;
}

__global__ void __launch_bounds__(DI_THREADS) zxc_dindex_count(const DIdxArgs A) {
    __shared__ __align__(16) u8 sm[DI_TILE + 48];
    const DFrame* F = &A.st->F;
    if (F->done) return;
    const u64 t0 = (u64)blockIdx.x * DI_TILE;
    u32 mis;
    di_load(A, t0, sm, &mis);
    const u32 c = di_count_lane(A, sm, mis, t0, F->block_size, di_trailer(F));
    unsigned long long total;
    asm_cta_excl(c, &total);
    if (threadIdx.x == 0) A.tiles[blockIdx.x] = total;
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dindex_tscan(const DIdxArgs A) {
    DIdxState* S = A.st;
    if (S->F.done) return;
    const u32 n = A.n_tiles;
    unsigned long long carry = 0;
    for (u64 b = 0; b < n; b += (u64)ASM_SCAN_THREADS * DI_SCAN_ITEMS) {
        const u64 i0 = b + (u64)threadIdx.x * DI_SCAN_ITEMS;
        unsigned long long c[DI_SCAN_ITEMS], s = 0;
#pragma unroll
        for (u32 k = 0; k < DI_SCAN_ITEMS; k++) {
            c[k] = i0 + k < n ? A.tiles[i0 + k] : 0;
            s += c[k];
        }
        unsigned long long total;
        unsigned long long ex = carry + asm_cta_excl(s, &total);
#pragma unroll
        for (u32 k = 0; k < DI_SCAN_ITEMS; k++) {
            if (i0 + k < n) A.tiles[i0 + k] = ex;
            ex += c[k];
        }
        carry += total;
    }
    if (threadIdx.x == 0) {
        S->m = carry;
        if (carry > A.C) S->F.fast = 0; /* the list would overflow: the walk decides */
    }
}

__global__ void __launch_bounds__(DI_THREADS) zxc_dindex_emit(const DIdxArgs A) {
    __shared__ __align__(16) u8 sm[DI_TILE + 48];
    const DFrame* F = &A.st->F;
    if (F->done || !F->fast) return;
    const u64 t0 = (u64)blockIdx.x * DI_TILE;
    const u32 bs = F->block_size, trailer = di_trailer(F), lane = threadIdx.x & 31;
    u32 mis;
    di_load(A, t0, sm, &mis);
    /* the warp's place in the tile: the earlier warps' counts */
    const u32 wc = __reduce_add_sync(FULL, di_count_lane(A, sm, mis, t0, bs, trailer));
    unsigned long long total;
    const unsigned long long wx = asm_cta_excl(lane == 0 ? wc : 0u, &total);
    u64 pos = A.tiles[blockIdx.x] + __shfl_sync(FULL, wx, 0);
    for (u32 k = 0; k < DI_STEPS; k++) {
        u32 rel, lens[4];
        const u32 bits = di_word(A, sm, mis, t0, k, bs, trailer, &rel, lens);
        const u32 c = __popc(bits);
        if (!__any_sync(FULL, c != 0)) continue;
        const u32 inc = warp_incl_scan(c, lane);
        u64 q = pos + inc - c;
#pragma unroll
        for (u32 j = 0; j < 4; j++) {
            if (bits & (1u << j)) {
                A.off[q] = t0 + rel + j;
                A.len[q] = lens[j];
                q++;
            }
        }
        pos += __shfl_sync(FULL, inc, 31);
    }
}

/* the candidate in [lo, m) at offset `target` (the list is ascending), or DI_NONE */
__device__ __forceinline__ u32 di_find(const unsigned long long* off, u64 lo, const u64 m, u64 target) {
    u64 hi = m;
    while (lo < hi) {
        const u64 mid = (lo + hi) >> 1;
        if (off[mid] < target) lo = mid + 1;
        else hi = mid;
    }
    return lo < m && off[lo] == target ? (u32)lo : DI_NONE;
}

/* the guess is still open: the frame passed the probe and its candidates fit the list */
__device__ __forceinline__ bool di_open(const DIdxState* S) { return !S->F.done && S->F.fast; }

__global__ void __launch_bounds__(DI_THREADS) zxc_dindex_links(const DIdxArgs A) {
    DIdxState* S = A.st;
    if (!di_open(S)) return;
    const u64 m = S->m;
    if (blockIdx.x == 0 && threadIdx.x == 0 && (m == 0 || A.off[0] != ZXC_FILE_HEADER_SIZE)) S->F.fast = 0;
    for (u64 v = (u64)blockIdx.x * DI_THREADS + threadIdx.x; v < m; v += (u64)gridDim.x * DI_THREADS) {
        const u32 l = A.len[v];
        u32 t = (u32)v; /* an EOF block ends its chain */
        if (l != 0) {
            const u64 target = A.off[v] + l;
            t = v + 1 < m && A.off[v + 1] == target ? (u32)(v + 1) : di_find(A.off, v + 2, m, target);
        }
        A.jump[0][v] = t;
        A.mark[v] = v == 0;
    }
}

/* round r: every marked node marks its 2^r-th successor, and jump[(r + 1) & 1] = jump[r & 1] squared.  The first 2^r
 * nodes of the chain were marked by the rounds before, so this marks the next 2^r; a mark another thread sets in the
 * same round and this one reads can only add a node that really is on the chain. */
__global__ void __launch_bounds__(DI_THREADS) zxc_dindex_round(const DIdxArgs A, const u32 r) {
    const DIdxState* S = A.st;
    if (!di_open(S)) return;
    const u64 m = S->m;
    if ((1ull << r) >= m) return; /* the chain has at most m nodes: all marked */
    const u32* ji = (r & 1) ? A.jump[1] : A.jump[0]; /* not A.jump[r & 1]: that copies the parameters to the stack */
    u32* jo = (r & 1) ? A.jump[0] : A.jump[1];
    for (u64 v = (u64)blockIdx.x * DI_THREADS + threadIdx.x; v < m; v += (u64)gridDim.x * DI_THREADS) {
        const u32 t = ji[v];
        if (t != DI_NONE && A.mark[v]) A.mark[t] = 1;
        jo[v] = t == DI_NONE ? DI_NONE : ji[t];
    }
}

/* this thread's ASM_ITEMS candidates from `first`: the marked data blocks among them (bit k), and the marked EOF */
__device__ __forceinline__ u32 di_marked(const DIdxArgs& A, DIdxState* S, u64 first, u64 m) {
    u32 bits = 0;
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        const u64 i = first + k;
        if (i < m && A.mark[i]) {
            if (A.len[i]) bits |= 1u << k;
            else atomicMin(&S->eof_pos, A.off[i]);
        }
    }
    return bits;
}

__global__ void __launch_bounds__(ASM_THREADS) zxc_dindex_mtiles(const DIdxArgs A) {
    DIdxState* S = A.st;
    if (!di_open(S)) return;
    const u64 m = S->m;
    if ((u64)blockIdx.x * ASM_TILE >= m) return;
    const u32 bits = di_marked(A, S, (u64)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS, m);
    unsigned long long total;
    asm_cta_excl(__popc(bits), &total);
    if (threadIdx.x == 0) A.mtiles[blockIdx.x] = total;
}

__global__ void __launch_bounds__(ASM_SCAN_THREADS) zxc_dindex_mscan(const DIdxArgs A) {
    DIdxState* S = A.st;
    if (!di_open(S)) return;
    const u32 n = (u32)((S->m + ASM_TILE - 1) / ASM_TILE);
    unsigned long long carry = 0;
    for (u32 b = 0; b < n; b += blockDim.x) {
        const u32 i = b + threadIdx.x;
        const unsigned long long v = i < n ? A.mtiles[i] : 0;
        unsigned long long total;
        const unsigned long long ex = asm_cta_excl(v, &total);
        if (i < n) A.mtiles[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) {
        if (S->eof_pos == ~0ull || carry > A.J) { /* no EOF on the chain, or a plan the scratch cannot hold */
            S->F.fast = 0;
        } else {
            S->F.n = carry;
            S->F.end = ZXW_END_EOF;
        }
    }
}

__global__ void __launch_bounds__(ASM_THREADS) zxc_dindex_memit(const DIdxArgs A) {
    DIdxState* S = A.st;
    if (!di_open(S)) return;
    const u64 m = S->m;
    if ((u64)blockIdx.x * ASM_TILE >= m) return;
    const u64 first = (u64)blockIdx.x * ASM_TILE + threadIdx.x * ASM_ITEMS;
    const u32 bits = di_marked(A, S, first, m);
    unsigned long long total;
    u64 j = A.mtiles[blockIdx.x] + asm_cta_excl(__popc(bits), &total);
#pragma unroll
    for (u32 k = 0; k < ASM_ITEMS; k++) {
        if (bits & (1u << k)) {
            zxc_b200_job_t Jb;
            Jb.src_off = A.off[first + k];
            Jb.dst_off = 0;
            Jb.src_len = A.len[first + k];
            Jb.dst_cap = 0;
            A.plan[j++] = Jb;
        }
    }
}

/* the proof, whatever built the plan: the sequential walk from offset 16 reads a valid header of a data type at every
 * entry, steps by exactly its on-disk size to the next one, and after the last one reads a valid empty EOF block */
__global__ void __launch_bounds__(DI_THREADS) zxc_dindex_prove(const DIdxArgs A) {
    DIdxState* S = A.st;
    if (!di_open(S)) return;
    const u64 n = S->F.n, eof = S->eof_pos;
    const u32 trailer = di_trailer(&S->F);
    bool ok = true;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        u32 type, comp;
        ok = dp_block_header(A.buf + eof, &type, &comp) && type == ZXF_BT_EOF && comp == 0 &&
             (n > 0 || eof == ZXC_FILE_HEADER_SIZE);
    }
    for (u64 j = (u64)blockIdx.x * DI_THREADS + threadIdx.x; j < n; j += (u64)gridDim.x * DI_THREADS) {
        const zxc_b200_job_t Jb = A.plan[j];
        const u64 next = j + 1 < n ? A.plan[j + 1].src_off : eof;
        u32 type, comp;
        if (!dp_block_header(A.buf + Jb.src_off, &type, &comp) || type > ZXF_BT_GHI ||
            (u64)ZXF_BLOCK_HDR + comp + trailer != Jb.src_len || Jb.src_off + Jb.src_len != next ||
            (j == 0 && Jb.src_off != ZXC_FILE_HEADER_SIZE))
            ok = false;
    }
    if (!ok) S->F.fast = 0;
}

__global__ void zxc_dindex_walk(const DIdxArgs A) {
    DIdxState* S = A.st;
    if (S->F.done) return;
    const u32 lane = threadIdx.x & 31;
    if (S->F.fast) {
        if (lane == 0) S->path = DI_PATH_SPEC;
        return;
    }
    dp_walk(&S->F, A.buf, A.size, A.J, A.plan, lane);
    if (lane != 0) return;
    S->path = DI_PATH_WALK;
    const u64 n = S->F.n;
    if (S->F.end == ZXW_END_EOF && n <= A.J)
        S->eof_pos = n ? A.plan[n - 1].src_off + A.plan[n - 1].src_len : ZXC_FILE_HEADER_SIZE;
}

/* the chain can be judged: it ends at an EOF block and the plan holds all of it */
__device__ __forceinline__ bool di_judged(const DIdxState* S, u32 J) {
    return !S->F.done && S->F.end == ZXW_END_EOF && S->F.n <= J;
}

/* the tail behind the EOF block: the footer alone (12 bytes), or a table of n entries and the footer */
__device__ __forceinline__ u64 di_tail(const DIdxArgs& A, const DIdxState* S) {
    return A.size - S->eof_pos - ZXF_BLOCK_HDR;
}

__global__ void __launch_bounds__(DI_THREADS) zxc_dindex_check(const DIdxArgs A) {
    DIdxState* S = A.st;
    if (!di_judged(S, A.J)) return;
    const u64 n = S->F.n;
    const bool table = di_tail(A, S) == ZXC_FILE_FOOTER_SIZE + ZXF_BLOCK_HDR + 4 * n;
    const u8* ent = A.buf + S->eof_pos + 2 * ZXF_BLOCK_HDR;
    bool bad = false, diff = false;
    for (u64 j = (u64)blockIdx.x * DI_THREADS + threadIdx.x; j < n; j += (u64)gridDim.x * DI_THREADS) {
        const zxc_b200_job_t Jb = A.plan[j];
        bad |= A.buf[Jb.src_off] > ZXF_BT_GHI;
        diff |= table && ld32(ent + 4 * j) != Jb.src_len;
    }
    if (bad) S->bad_type = 1;
    if (diff) S->table_diff = 1;
}

/* the SEK block header of a table of n entries (zxf_write_block_header) */
__device__ __forceinline__ u64 di_sek_header(u64 n) {
    const u64 v = (u64)ZXF_BT_SEK | ((u64)(u32)(n * ZXF_SEEK_ENTRY) << 24);
    return v | ((u64)dev_hash8(v) << 56);
}

__global__ void zxc_dindex_decide(const DIdxArgs A) {
    DIdxState* S = A.st;
    const DFrame* F = &S->F;
    if (F->done) return;
    const u64 n = F->n, bs = F->block_size, f = F->footer_size;
    const u64 need = f / bs + (f % bs != 0); /* the blocks a reader of the table expects */
    const u64 table = (u64)ZXF_BLOCK_HDR + n * ZXF_SEEK_ENTRY;
    long long v;
    if (F->end != ZXW_END_EOF) {
        v = ZXC_ERROR_BAD_HEADER;
    } else if (n > A.J) { /* the plan does not hold the chain: its types and sizes are unknown */
        v = n != need ? ZXC_ERROR_CORRUPT_DATA
                      : (n > 0xFFFFFFFFull / ZXF_SEEK_ENTRY ? ZXC_ERROR_OVERFLOW : ZXC_ERROR_MEMORY);
    } else if (S->bad_type) {
        v = ZXC_ERROR_BAD_BLOCK_TYPE;
    } else {
        const u64 tail = di_tail(A, S);
        if (tail == ZXC_FILE_FOOTER_SIZE + table && !S->table_diff &&
            ld64(A.buf + S->eof_pos + ZXF_BLOCK_HDR) == di_sek_header(n))
            v = (long long)A.size; /* the frame already carries this table */
        else if (tail != ZXC_FILE_FOOTER_SIZE || n != need)
            v = ZXC_ERROR_CORRUPT_DATA;
        else if (n == 0)
            v = (long long)A.size;
        else if (n > 0xFFFFFFFFull / ZXF_SEEK_ENTRY)
            v = ZXC_ERROR_OVERFLOW;
        else if (A.cap < A.size + table)
            v = ZXC_ERROR_DST_TOO_SMALL;
        else {
            v = (long long)(A.size + table);
            S->write = 1;
        }
    }
    *A.result = v;
}

/* byte stores: the buffer may have any alignment */
__device__ __forceinline__ void di_st(u8* p, u64 v, u32 bytes) {
    for (u32 i = 0; i < bytes; i++) p[i] = (u8)(v >> (8 * i));
}

__global__ void __launch_bounds__(DI_THREADS) zxc_dindex_write(const DIdxArgs A) {
    const DIdxState* S = A.st;
    if (!S->write) return;
    const u64 n = S->F.n;
    u8* t = A.buf + A.size - ZXC_FILE_FOOTER_SIZE;
    for (u64 j = (u64)blockIdx.x * DI_THREADS + threadIdx.x; j < n; j += (u64)gridDim.x * DI_THREADS)
        di_st(t + ZXF_BLOCK_HDR + 4 * j, A.plan[j].src_len, 4);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        di_st(t, di_sek_header(n), 8);
        u8* ft = t + ZXF_BLOCK_HDR + 4 * n;
        di_st(ft, S->F.footer_size, 8);
        di_st(ft + 8, S->F.footer_hash, 4);
    }
}
