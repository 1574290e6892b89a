/*
 * zxc_encode.cuh -- sm_90a block encoder (device code only): the reference's hash-chain match
 * finder and greedy/lazy parsers for levels 1-5, one warp per independent block, emitting blocks
 * that are bit-identical to the reference encoder's.  Levels 6-7 (optimal parser, Huffman sections)
 * share the block driver below and live in zxc_encode_opt.cuh.
 *
 * What is replicated (SURVEY.md section 8 rows E1-E3, E5-E7, Appendix B):
 *   E1 hash            zxc_hash_func                  src/lib/zxc_compress.c:45-53
 *   E2 match tables    head table + u16 chain         src/lib/zxc_internal.h:1633-1690 (in HBM, per warp)
 *   E3 match finder    zxc_lz77_find_best_match       src/lib/zxc_compress.c:185-547
 *   E5 parse loops     GLO lazy :1174-1255, GHI greedy :1858-1921
 *   E6 dict seeding    zxc_lz_seed_dict               :1060-1100
 *   E7 select+emit     RLE sizing :1270-1534, GLO writer :1628-1798, GHI writer :1929-1986,
 *                      RAW fallback + checksum :2041-2074
 *
 * The parse is a sequential state machine per block (every step depends on the previous match),
 * so parallelism is across blocks (warps) and inside one find_best_match call: the 32 lanes
 * compare 128 bytes of candidate vs. current position per step, extend backwards 32 bytes per
 * step, and copy literal runs cooperatively.
 *
 * Differences in mechanism that do not change the output:
 *   - no epoch: the head table is cleared per block (the reference bumps an epoch so stale
 *     entries read as empty, :1132-1140 -- same observable state);
 *   - no tag table: a valid head's stored tag is by construction the tag of the 4 bytes at that
 *     position (table and tag are always written together, :219-220, :1241-1242, :1073-1075), so
 *     it is recomputed from the source instead of stored.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "zxc_decode.cuh" /* u8/u32, FULL, warp_checksum, ld helpers */
#include "zxc_hufenc.h"

#ifndef ZXC_LANE_STAT
#define ZXC_LANE_STAT(i, v) /* tests/simt counts one lane's own event here (every lane); nothing in the product build */
#endif

#define ENC_HUFWORK_BYTES ((sizeof(zxh_work_t) + 255u) & ~(size_t)255u)
#define ENC_PLAN_BYTES 8192u

#define ENC_WARPS_PER_CTA 4
#define ENC_CTA_THREADS (ENC_WARPS_PER_CTA * 32)
#define ENC_CTAS_PER_SM 8u
#define ENC_HASH_BITS 15
#define ENC_HASH_SIZE (1u << ENC_HASH_BITS)
#define ENC_WINDOW 65536u
#define ENC_MAX_DIST 65535u

struct EncodeParams {
    const u8* src;          /* input bytes (16-byte aligned base, >= 16 bytes readable past the end) */
    u8* staging;            /* one slot of staging_stride bytes per block */
    u32* out_size;          /* per block: bytes written to its slot (header + payload + checksum) */
    u8* scratch;            /* per warp: tables + stream buffers */
    unsigned long long* counter;
    const u8* dict;         /* dictionary content or NULL */
    const u32* seed_head;   /* dictionary-seeded head table (ENC_HASH_SIZE entries) or NULL */
    const unsigned short* seed_chain; /* chain links of the seeded dictionary positions */
    unsigned long long src_size;
    unsigned long long scratch_stride;
    u32 block_size;
    u32 n_blocks;
    u32 staging_stride;
    u32 level;
    u32 checksum;
    u32 dict_size;
    const u8* dict_huf_lens; /* 256 unpacked code lengths of the dictionary's literal table, or NULL */
};

/* per-warp scratch layout (bytes from the warp's base) */
struct EncLayout {
    size_t literals, seqbuf, extras, comb, dp, ends, work, plan, freq, lens, total;
    u32 seq_cap;
};
__host__ __device__ inline EncLayout enc_layout(u32 bs, int level) {
    EncLayout L;
    L.seq_cap = bs / 5 + 32;
    size_t o = (size_t)ENC_HASH_SIZE * 4 + (size_t)ENC_WINDOW * 2;
    L.literals = o;
    o += (((size_t)bs + 63) & ~(size_t)63) + 64;
    L.seqbuf = o;
    o += (size_t)L.seq_cap * 4;
    L.extras = o;
    o += bs / 4 + 64;
    L.comb = o; /* [dict | block | 16] when a dictionary is attached */
    o += 65536 + (size_t)bs + 64;
    o = (o + 255) & ~(size_t)255;
    L.dp = L.ends = L.work = L.plan = L.freq = L.lens = 0;
    if (level >= 6) {
        L.dp = o; /* u64 per position */
        o += ((size_t)bs + 1) * 8;
        o = (o + 255) & ~(size_t)255;
        L.ends = o;
        o += (size_t)L.seq_cap * 4;
        o = (o + 255) & ~(size_t)255;
        L.work = o; /* zxh_work_t */
        o += ENC_HUFWORK_BYTES;
        L.plan = o; /* PivcoPlan */
        o += ENC_PLAN_BYTES;
        L.freq = o; /* literal and token histograms */
        o += 2 * 256 * 4;
        L.lens = o; /* literal, token and temporary code lengths */
        o += 3 * 256;
    }
    L.total = (o + 255) & ~(size_t)255;
    return L;
}

struct LzParams {
    int search_depth, sufficient_len, use_lazy, lazy_attempts, lazy_len_threshold;
    u32 step_base, step_shift;
};

/* zxc_get_lz77_params (src/lib/zxc_internal.h:965-979) */
__device__ __forceinline__ LzParams lz_params(int level) {
    switch (level) {
        case 2: return {3, 18, 0, 0, 0, 3, 6};
        case 3: return {3, 16, 1, 4, 128, 1, 4};
        case 4: return {3, 18, 1, 4, 128, 1, 5};
        case 5: return {64, 256, 1, 16, 128, 1, 8};
        case 6: return {64, 256, 0, 0, 0, 1, 8};
        default: return level >= 7 ? LzParams{128, 256, 0, 0, 0, 1, 8} : LzParams{3, 16, 0, 0, 0, 4, 4};
    }
}

/* unaligned little-endian loads built from aligned words (base must be 4-byte aligned) */
__device__ __forceinline__ u32 ldu32(const u8* base, u32 pos) {
    const u32* w = reinterpret_cast<const u32*>(base + (pos & ~3u));
    return __funnelshift_r(w[0], w[1], (pos & 3u) * 8u);
}
__device__ __forceinline__ u64 ldu64(const u8* base, u32 pos) {
    const u32* w = reinterpret_cast<const u32*>(base + (pos & ~3u));
    const u32 sh = (pos & 3u) * 8u;
    const u32 a = w[0], b = w[1], c = w[2];
    return (u64)__funnelshift_r(a, b, sh) | ((u64)__funnelshift_r(b, c, sh) << 32);
}

/* zxc_hash_func (zxc_compress.c:45-53) */
__device__ __forceinline__ u32 enc_hash(u64 v, bool hash5) {
    if (hash5) return (u32)(((v & 0xFFFFFFFFFFull) * 0x2545F4914F6CDD1Dull) >> (64 - ENC_HASH_BITS));
    return ((u32)(v ^ (v >> 15)) * 0x2D35182Du) >> (32 - ENC_HASH_BITS);
}
__device__ __forceinline__ u32 enc_tag(u32 v) { return (v ^ (v >> 16)) & 0xFFu; }

/* common prefix length of src[a..] and src[b..] (b < a), bounded so that a + len <= end;
 * the first `known` bytes are already known equal.  128 bytes per warp step. */
__device__ __forceinline__ u32 warp_lcp(const u8* src, u32 a, u32 b, u32 end, u32 known, u32 cap, u32 lane) {
    u32 len = known;
    for (;;) {
        const u32 pa = a + len + 4u * lane;
        u32 x = 0xFFFFFFFFu; /* "all four bytes differ" for lanes past the end */
        if (pa + 4u <= end) x = ldu32(src, pa) ^ ldu32(src, b + len + 4u * lane);
        else if (pa < end) {
            const u32 n = end - pa; /* 1..3 valid bytes */
            x = (ldu32(src, pa) ^ ldu32(src, b + len + 4u * lane)) | (0xFFFFFFFFu << (8u * n));
        }
        const u32 diff = __ballot_sync(FULL, x != 0);
        if (diff) {
            const int l = __ffs(diff) - 1;
            const u32 xl = __shfl_sync(FULL, x, l);
            return len + 4u * (u32)l + ((u32)(__ffs(xl) - 1) >> 3);
        }
        len += 128u;
        if (len >= cap) return len;
    }
}

struct Match {
    u32 ref; /* position of the match source, valid when found */
    u32 len;
    u32 backtrack;
    bool found;
};

/* zxc_lz77_find_best_match (zxc_compress.c:185-547); every lane computes the same scalars */
__device__ Match find_best_match(const u8* src, u32 ip, u32 iend, u32 search_limit, u32 anchor, u32* head,
                                 unsigned short* chain, int level, const LzParams& p, u32 lane) {
    const bool hash5 = level >= 3;
    Match best;
    best.ref = 0;
    best.len = 4; /* ZXC_LZ_MIN_MATCH_LEN - 1 */
    best.backtrack = 0;
    best.found = false;

    const u64 cur8 = ldu64(src, ip);
    const u32 cur_val = (u32)cur8;
    const u32 h = enc_hash(cur8, hash5);
    const u32 cur_tag = enc_tag(cur_val);

    u32 match_idx = head[h];
    /* the tag the reference would have stored for a valid head */
    const u32 stored_tag = match_idx ? enc_tag(ldu32(src, match_idx)) : 0xFFFFFFFFu;
    if (level <= 2 && match_idx && stored_tag != cur_tag) match_idx = 0; /* tag-first filter :206-208 */
    const bool skip_head = match_idx != 0 && stored_tag != cur_tag;

    __syncwarp();
    if (lane == 0) {
        head[h] = ip;
        const u32 dist = ip - match_idx;
        chain[ip & (ENC_WINDOW - 1)] = (match_idx != 0 && dist < ENC_WINDOW) ? (unsigned short)dist : 0;
    }
    __syncwarp();

    int attempts = p.search_depth;
    if (match_idx != 0) {
        if (skip_head) {
            ZXC_STAT(92, 1); /* a head whose tag differs is skipped */
            const u32 delta = chain[match_idx & (ENC_WINDOW - 1)];
            match_idx = delta ? match_idx - delta : 0;
            attempts--;
        }
        while (match_idx > 0) {
            ZXC_STAT(78, attempts >= 0 && ip - match_idx > ENC_MAX_DIST); /* candidates beyond the window */
            if (attempts-- < 0 || ip - match_idx > ENC_MAX_DIST) break;
            const u32 delta = chain[match_idx & (ENC_WINDOW - 1)];
            const u32 next_idx = match_idx - delta;
            if (ldu32(src, match_idx) == cur_val) {
                /* the reference also gates on ref[best.len] == ip[best.len]; a candidate failing
                 * that gate cannot be strictly longer, so evaluating it changes nothing */
                const u32 mlen = warp_lcp(src, ip, match_idx, iend, 4, 0xFFFFFFFFu, lane);
                if (mlen > best.len) {
                    best.len = mlen;
                    best.ref = match_idx;
                    best.found = true;
                }
                if (best.len >= (u32)p.sufficient_len || ip + best.len >= iend) break;
            }
            match_idx = delta ? next_idx : 0;
        }
    }

    if (best.found) {
        /* backward extension (:440-451): while b_ip > anchor && b_ref > 0 && equal */
        u32 back = 0;
        for (;;) {
            const u32 k = back + lane + 1;
            const bool ok = (ip - anchor >= k) && (best.ref >= k) && src[ip - k] == src[best.ref - k];
            const u32 nb = ~__ballot_sync(FULL, ok);
            if (nb) {
                back += (u32)(__ffs(nb) - 1);
                break;
            }
            back += 32;
        }
        best.len += back;
        best.backtrack = back;
        best.ref -= back;
    }

    if (p.use_lazy && best.found && best.len < (u32)p.lazy_len_threshold && ip + 1 < search_limit) {
        u32 max_lazy[2] = {0, 0};
        const int n_lazy = (level >= 4 && ip + 2 < search_limit) ? 2 : 1;
        for (int t = 0; t < n_lazy; t++) {
            const u32 lp = ip + 1 + (u32)t;
            const u64 v8 = ldu64(src, lp);
            const u32 v = (u32)v8;
            u32 idx = head[enc_hash(v8, hash5)];
            const bool skip_first = idx > 0 && enc_tag(ldu32(src, idx)) != enc_tag(v);
            int att = p.lazy_attempts;
            bool first = true;
            while (idx > 0) {
                ZXC_STAT(78, att > 0 && lp - idx > ENC_MAX_DIST);
                if (att-- <= 0 || lp - idx > ENC_MAX_DIST) break;
                if ((!first || !skip_first) && ldu32(src, idx) == v) {
                    /* only compared against best.len + 1/2 < 130: one 128-byte step is enough */
                    const u32 l2 = warp_lcp(src, lp, idx, iend, 4, 132, lane);
                    max_lazy[t] = l2 > max_lazy[t] ? l2 : max_lazy[t];
                }
                const u32 delta = chain[idx & (ENC_WINDOW - 1)];
                if (delta == 0) break;
                idx -= delta;
                first = false;
            }
        }
        if (max_lazy[0] > best.len + 1 || max_lazy[1] > best.len + 2) {
            ZXC_STAT(79, 1); /* lazy replacements */
            best.found = false;
        }
    }
    return best;
}

/* prefix varint writer (zxc_compress.c:115-142); returns bytes written */
__device__ __forceinline__ u32 put_varint(u8* dst, u32 val) {
    if (val < (1u << 7)) {
        dst[0] = (u8)val;
        return 1;
    }
    if (val < (1u << 14)) {
        dst[0] = (u8)(0x80 | (val & 0x3F));
        dst[1] = (u8)(val >> 6);
        return 2;
    }
    dst[0] = (u8)(0xC0 | (val & 0x1F));
    dst[1] = (u8)(val >> 5);
    dst[2] = (u8)(val >> 13);
    return 3;
}

/* RLE size of a literal stream (zxc_compress.c:1270-1525), scalar semantics:
 * maximal runs >= 4 cost 2 bytes per 131 (+ remainder), the gaps cost len + ceil(len/128). */
__device__ u32 rle_size_of(const u8* lit, u32 n) {
    u32 size = 0, p = 0;
    while (p < n) {
        const u8 b = lit[p];
        const u32 run_start = p++;
        while (p < n && lit[p] == b) p++;
        const u32 run = p - run_start;
        if (run >= 4) {
            const u32 full = run / 131, rem = run - full * 131;
            size += full * 2;
            if (rem >= 4) size += 2;
            else if (rem > 0) size += 1 + rem;
        } else {
            while (p < n) {
                if (p + 3 < n && lit[p] == lit[p + 1] && lit[p + 1] == lit[p + 2] && lit[p + 2] == lit[p + 3]) break;
                p++;
            }
            const u32 lr = p - run_start;
            size += lr + ((lr + 127) >> 7);
        }
    }
    return size;
}

/* RLE writer (zxc_compress.c:1671-1722); returns bytes written */
__device__ u32 rle_write(const u8* lit, u32 n, u8* dst) {
    u32 p = 0, o = 0;
    while (p < n) {
        const u8 b = lit[p];
        const u32 run_start = p++;
        while (p < n && lit[p] == b) p++;
        u32 run = p - run_start;
        if (run >= 4) {
            while (run >= 4) {
                const u32 chunk = run > 131 ? 131 : run;
                dst[o++] = (u8)(0x80 | (chunk - 4));
                dst[o++] = b;
                run -= chunk;
            }
            if (run > 0) {
                dst[o++] = (u8)(run - 1);
                for (u32 k = 0; k < run; k++) dst[o++] = b;
            }
        } else {
            while (p < n) {
                if (p + 3 < n && lit[p] == lit[p + 1] && lit[p + 1] == lit[p + 2] && lit[p + 2] == lit[p + 3]) break;
                p++;
            }
            u32 lr = p - run_start, s = run_start;
            while (lr > 0) {
                const u32 chunk = lr > 128 ? 128 : lr;
                dst[o++] = (u8)(chunk - 1);
                for (u32 k = 0; k < chunk; k++) dst[o++] = lit[s + k];
                s += chunk;
                lr -= chunk;
            }
        }
    }
    return o;
}

__device__ __forceinline__ void warp_bytes(u8* d, const u8* s, u32 n, u32 lane) {
    for (u32 k = lane; k < n; k += 32) d[k] = s[k];
}

/* zxc_hash8 (zxc_internal.h:1188-1195) over the 8 header bytes with byte 7 zero */
__device__ __forceinline__ u8 dev_hash8(u64 v) {
    u64 h = v ^ 0x9E3779B97F4A7C15ull;
    h ^= h << 13;
    h ^= h >> 7;
    h ^= h << 17;
    return (u8)((h >> 32) ^ h);
}
__device__ __forceinline__ void put_block_header(u8* dst, u32 type, u32 comp_size) {
    const u64 v = (u64)type | ((u64)comp_size << 24);
    for (int i = 0; i < 7; i++) dst[i] = (u8)(v >> (8 * i));
    dst[7] = dev_hash8(v);
}
__device__ __forceinline__ void st32(u8* p, u32 v) {
    p[0] = (u8)v;
    p[1] = (u8)(v >> 8);
    p[2] = (u8)(v >> 16);
    p[3] = (u8)(v >> 24);
}

__device__ __forceinline__ void seed_step(const u8* src, u32 i, u32 half, bool hash5, u32* head, unsigned short* chain);
__device__ __forceinline__ u32 seed_shared_stop(u32 dict_size, bool hash5);

/* one block: zxc_compress_chunk_wrapper (zxc_compress.c:2041-2074) */
#include "zxc_huffman.cuh" /* HUF_MAXLEN, HUF_KIND_*: the section geometry shared with the decoder */
#include "zxc_encode_opt.cuh"
static_assert(sizeof(PivcoPlan) <= ENC_PLAN_BYTES, "PivcoPlan must fit its scratch slot");

/* The warp's match tables for one block, and the bytes the parse reads: with a dictionary, the seeded tables cloned
 * and [dict | block] materialised in scratch (the block at position dict_size); without, cleared tables and the
 * block itself. */
__device__ __forceinline__ const u8* enc_block_tables(const EncodeParams& P, const EncLayout& lay, int level, const u8* blk,
                                                      u32 n, u8* scratch, u32* head, unsigned short* chain, u32 lane) {
    const u32 base = P.dict ? P.dict_size : 0u; /* the dictionary is logically prepended to the block */
    const u8* src = blk; /* block start is 4-byte aligned (block_size multiple of 4096, aligned base) */
    if (base) {
        /* tables as zxc_lz_seed_dict leaves them (:1060-1100), cloned instead of re-seeded per block
         * (SURVEY 8(f)-4: output-identical); [dict | block] materialised so positions are contiguous */
        for (u32 k = lane; k < ENC_HASH_SIZE / 4; k += 32)
            reinterpret_cast<uint4*>(head)[k] = reinterpret_cast<const uint4*>(P.seed_head)[k];
        const u32 nchain = min(base, ENC_WINDOW);
        for (u32 k = lane; k < nchain; k += 32) chain[k] = P.seed_chain[k];
        u8* comb = scratch + lay.comb;
        for (u32 k = lane; k < base; k += 32) comb[k] = P.dict[k];
        for (u32 k = lane; k < n; k += 32) comb[base + k] = blk[k];
        for (u32 k = lane; k < 16; k += 32) comb[base + n + k] = 0;
        src = comb;
        __syncwarp();
        if (base >= 5 && lane == 0) { /* positions whose hash window reaches into the block */
            ZXC_STAT(91, 1);
            const bool h5 = level >= 3;
            for (u32 i = seed_shared_stop(base, h5); i < base - 4; i++) seed_step(src, i, (base - 4) / 2, h5, head, chain);
        }
    } else {
        /* fresh tables per block (the reference's epoch bump) */
        for (u32 k = lane; k < ENC_HASH_SIZE / 4; k += 32) reinterpret_cast<uint4*>(head)[k] = make_uint4(0, 0, 0, 0);
    }
    __syncwarp();
    return src;
}

/* OPT = levels 6-7 (optimal parser + entropy stage); a separate instantiation keeps the level 1-5
 * kernel at its own register budget */
template <bool OPT>
__device__ u32 encode_block(const EncodeParams& P, const u8* blk, u32 n, u8* dst, u8* scratch, u32* hist, u32 lane) {
    const int level = (int)P.level;
    const LzParams lzp = lz_params(level);
    const bool ghi = level <= 2;
    const u32 bs = P.block_size;

    const EncLayout lay = enc_layout(bs, level);
    u32* head = reinterpret_cast<u32*>(scratch);
    unsigned short* chain = reinterpret_cast<unsigned short*>(scratch + ENC_HASH_SIZE * 4);
    u8* literals = scratch + lay.literals;
    const u32 seq_cap = lay.seq_cap;
    u8* seqbuf = scratch + lay.seqbuf;                      /* GLO: tokens then u16 offsets; GHI: u32 words */
    u8* extras = scratch + lay.extras;
    u8* tokens = seqbuf;
    unsigned short* offsets = reinterpret_cast<unsigned short*>(seqbuf + ((seq_cap + 3) & ~3u));
    u32* seqwords = reinterpret_cast<u32*>(seqbuf);

    const u32 base = P.dict ? P.dict_size : 0u; /* the dictionary is logically prepended to the block */
    const u8* src = enc_block_tables(P, lay, level, blk, n, scratch, head, chain, lane);

    const u32 iend = base + n;
    u32 ip = base, anchor = base;
    u32 seq_c = 0, lit_c = 0, ext_c = 0, max_off = 0;

#ifdef ZXC_OPT_PROFILE
    const long long tb0 = clock64();
    long long tb1 = tb0, tb2 = tb0;
#endif
    if constexpr (OPT) {
        const OptOut R = optimal_parse(src, base, n, head, chain, level, lzp, reinterpret_cast<u64*>(scratch + lay.dp),
                                       reinterpret_cast<u32*>(scratch + lay.ends), literals, tokens, offsets, extras, hist,
                                       reinterpret_cast<zxh_work_t*>(scratch + lay.work), scratch + lay.lens + 512, lane);
        seq_c = R.seq_c;
        lit_c = R.lit_c;
        ext_c = R.ext_c;
        max_off = R.max_off;
        anchor = iend; /* the parser has already gathered the trailing literals */
    } else if (n + base > 8 && iend - 8 > base) {
        const u32 search_limit = iend - 8;
        while (ip < search_limit) {
            const u32 dist = ip - anchor;
            u32 step = lzp.step_base + (dist >> lzp.step_shift);
            if (ip + step >= search_limit) step = 1;
            const Match m = find_best_match(src, ip, iend, search_limit, anchor, head, chain, level, lzp, lane);
            if (m.found) {
                ZXC_STAT(81, m.backtrack != 0); /* backtracked starts */
                ip -= m.backtrack;
                const u32 ll = ip - anchor;
                const u32 ml = m.len - 5;
                const u32 off = ip - m.ref;
                warp_bytes(literals + lit_c, src + anchor, ll, lane);
                if (lane == 0) {
                    if (!ghi) {
                        tokens[seq_c] = (u8)(((ll >= 15 ? 15u : ll) << 4) | (ml >= 15 ? 15u : ml));
                        offsets[seq_c] = (unsigned short)(off - 1);
                    } else {
                        seqwords[seq_c] = ((ll >= 255 ? 255u : ll) << 24) | ((ml >= 255 ? 255u : ml) << 16) | ((off - 1) & 0xFFFFu);
                    }
                }
                lit_c += ll;
                if (off - 1 > max_off) max_off = off - 1;
                const u32 esc = ghi ? 255u : 15u;
                if (ll >= esc) {
                    u32 nb = 0;
                    if (lane == 0) nb = put_varint(extras + ext_c, ll - esc);
                    ext_c += __shfl_sync(FULL, nb, 0);
                }
                if (ml >= esc) {
                    u32 nb = 0;
                    if (lane == 0) nb = put_varint(extras + ext_c, ml - esc);
                    ext_c += __shfl_sync(FULL, nb, 0);
                }
                seq_c++;
                if (!ghi && m.len > 2 && level > 4) { /* level 5: also index match_end - 2 (:1231-1248) */
                    const u32 match_end = ip + m.len;
                    if (match_end + 7 < iend) {
                        ZXC_STAT(82, 1);
                        const u32 pos_u = match_end - 2;
                        const u32 h_u = enc_hash(ldu64(src, pos_u), true);
                        const u32 prev = head[h_u];
                        __syncwarp();
                        if (lane == 0) {
                            head[h_u] = pos_u;
                            chain[pos_u & (ENC_WINDOW - 1)] = (prev > 0 && pos_u - prev < ENC_WINDOW) ? (unsigned short)(pos_u - prev) : 0;
                        }
                        __syncwarp();
                    }
                }
                ip += m.len;
                anchor = ip;
            } else {
                ZXC_STAT(80, step > 1); /* step skips */
                ip += step;
            }
        }
    }
    const u32 last = iend - anchor;
    warp_bytes(literals + lit_c, src + anchor, last, lane);
    lit_c += last;
    __syncwarp();

#ifdef ZXC_OPT_PROFILE
    tb1 = clock64();
#endif
    /* ---- section selection + serialisation.  Sizes are known before a byte is written, so a
     * block that would expand goes straight to RAW and the slot never overflows. ---- */
    u8* p = dst + 8;
    u32 w;
    u32 enc_lit = ENC_RAW, enc_tok = ENC_RAW, rle_sz = 0, huf_lit_sz = 0, huf_tok_sz = 0;
    u32 best_j = lit_c; /* J = size + decode tax (zxc_compress.c:1270-1626) */
    if (!ghi && lit_c > 0) {
        rle_sz = rle_size_of(literals, lit_c);
        const u32 prem = level >= 6 ? 1u : 8u; /* zxc_ss_prem_rle_q8 */
        const u32 j = rle_sz + ((lit_c * prem) >> 8);
        if (j < best_j) {
            enc_lit = ENC_RLE;
            best_j = j;
        }
    }
    u32* freq_lit = reinterpret_cast<u32*>(scratch + lay.freq);
    u32* freq_tok = freq_lit + 256;
    u8* cl_lit = scratch + lay.lens;
    u8* cl_tok = cl_lit + 256;
    PivcoPlan* plan = reinterpret_cast<PivcoPlan*>(scratch + lay.plan);
    zxh_work_t* hw = reinterpret_cast<zxh_work_t*>(scratch + lay.work);
    if constexpr (OPT) {
        const int cap = level >= 7 ? 11 : 8; /* zxc_huf_enc_max_code_len */
        bool have_hist = false;
        if (lit_c >= HUF_MIN_LITERALS) {
            warp_histogram(literals, lit_c, 1, hist, lane);
            for (u32 k = lane; k < 256; k += 32) freq_lit[k] = hist[k];
            __syncwarp();
            have_hist = true;
            if (build_section_lengths(freq_lit, cl_lit, cap, hw, lane)) {
                ZXC_STAT(93, 1); /* literal Huffman codes built */
                const u32 pay = pivco_plan(freq_lit, cl_lit, plan, lane);
                if (pay != 0xFFFFFFFFu) {
                    const u32 j = pay + 128u + ((lit_c * 4u) >> 8); /* zxc_ss_prem_huf_q8 */
                    if (j < best_j) {
                        enc_lit = ENC_HUF;
                        best_j = j;
                        huf_lit_sz = pay + 128u;
                    }
                }
            }
        }
        if (P.dict_huf_lens && lit_c > 0) { /* the dictionary's shared table: same bitstream, no header */
            if (!have_hist) {
                warp_histogram(literals, lit_c, 1, hist, lane);
                for (u32 k = lane; k < 256; k += 32) freq_lit[k] = hist[k];
                __syncwarp();
            }
            const u32 pay = pivco_plan(freq_lit, P.dict_huf_lens, plan, lane);
            if (pay != 0xFFFFFFFFu && pay + ((lit_c * 4u) >> 8) < best_j) {
                enc_lit = ENC_HUF_DICT;
                huf_lit_sz = pay;
            }
        }
        if (level >= 7 && seq_c >= HUF_MIN_LITERALS) {
            warp_histogram(tokens, seq_c, 1, hist, lane);
            for (u32 k = lane; k < 256; k += 32) freq_tok[k] = hist[k];
            __syncwarp();
            if (build_section_lengths(freq_tok, cl_tok, cap, hw, lane)) {
                const u32 pay = pivco_plan(freq_tok, cl_tok, plan, lane);
                if (pay != 0xFFFFFFFFu && pay + 128u + ((seq_c * 4u) >> 8) < seq_c) {
                    enc_tok = ENC_HUF;
                    huf_tok_sz = pay + 128u;
                }
            }
        }
    }
#ifdef ZXC_OPT_PROFILE
    tb2 = clock64();
#endif
    const u32 off8 = max_off <= 255 ? 1u : 0u;
    const u32 sz_lit = enc_lit == ENC_RLE ? rle_sz : (enc_lit >= ENC_HUF ? huf_lit_sz : lit_c);
    const u32 sz_tok = enc_tok == ENC_HUF ? huf_tok_sz : seq_c;
    const u32 sz_off = off8 ? seq_c : seq_c * 2;
    const u32 desc = (enc_lit != ENC_RAW ? 4u : 0u) + (enc_tok == ENC_HUF ? 4u : 0u);
    {
        const u32 behind = ghi ? seq_c * 4 + ext_c : sz_tok + sz_off + ext_c;
        const u32 pad = behind < 32 ? 32 - behind : 0;
        w = 8 + 12 + (ghi ? lit_c : desc + sz_lit) + behind + pad;
    }
    ZXC_STAT(83, w >= n); /* RAW blocks */
    if (w >= n) {
        /* expansion: store RAW (:2055-2058) */
    } else if (!ghi) {
        ZXC_STAT(84, enc_lit == ENC_RLE);
        ZXC_STAT(85, enc_lit == ENC_HUF);
        ZXC_STAT(86, enc_lit == ENC_HUF_DICT);
        ZXC_STAT(87, enc_tok == ENC_HUF);
        ZXC_STAT(88, off8);
        if (lane == 0) {
            st32(p, seq_c);
            st32(p + 4, lit_c);
            p[8] = (u8)enc_lit;
            p[9] = (u8)enc_tok;
            p[10] = 0;
            p[11] = (u8)off8;
            u8* dsc = p + 12;
            if (enc_lit != ENC_RAW) {
                st32(dsc, sz_lit);
                dsc += 4;
            }
            if (enc_tok == ENC_HUF) st32(dsc, sz_tok);
        }
        __syncwarp();
        u8* q = p + 12 + desc;
        if (enc_lit == ENC_RLE) {
            if (lane == 0) rle_write(literals, lit_c, q);
        } else if (OPT && enc_lit == ENC_HUF) {
            (void)pivco_plan(freq_lit, cl_lit, plan, lane);
            (void)pivco_write(literals, lit_c, cl_lit, plan, q, true, lane);
        } else if (OPT && enc_lit == ENC_HUF_DICT) {
            (void)pivco_plan(freq_lit, P.dict_huf_lens, plan, lane);
            (void)pivco_write(literals, lit_c, P.dict_huf_lens, plan, q, false, lane);
        } else {
            warp_bytes(q, literals, lit_c, lane);
        }
        q += sz_lit;
        if (OPT && enc_tok == ENC_HUF) {
            (void)pivco_plan(freq_tok, cl_tok, plan, lane);
            (void)pivco_write(tokens, seq_c, cl_tok, plan, q, true, lane);
        } else {
            warp_bytes(q, tokens, seq_c, lane);
        }
        q += sz_tok;
        if (off8) {
            for (u32 k = lane; k < seq_c; k += 32) q[k] = (u8)offsets[k];
        } else {
            warp_bytes(q, reinterpret_cast<const u8*>(offsets), seq_c * 2, lane);
        }
        q += sz_off;
        warp_bytes(q, extras, ext_c, lane);
        q += ext_c;
        const u32 behind = sz_tok + sz_off + ext_c;
        const u32 pad = behind < 32 ? 32 - behind : 0;
        if (lane < pad) q[lane] = 0;
    } else {
        if (lane == 0) {
            st32(p, seq_c);
            st32(p + 4, lit_c);
            p[8] = p[9] = p[10] = p[11] = 0;
        }
        u8* q = p + 12;
        warp_bytes(q, literals, lit_c, lane);
        q += lit_c;
        warp_bytes(q, reinterpret_cast<const u8*>(seqwords), seq_c * 4, lane);
        q += seq_c * 4;
        warp_bytes(q, extras, ext_c, lane);
        q += ext_c;
        const u32 behind = seq_c * 4 + ext_c;
        const u32 pad = behind < 32 ? 32 - behind : 0;
        if (lane < pad) q[lane] = 0;
    }
    __syncwarp();
#ifdef ZXC_OPT_PROFILE
    if (OPT && lane == 0)
        printf("block profile n=%u lit %u seq %u enc_lit %u enc_tok %u | cycles: parse %lld select %lld write %lld\n", n, lit_c, seq_c,
               enc_lit, enc_tok, tb1 - tb0, tb2 - tb1, clock64() - tb2);
#endif
    u32 type = ghi ? BT_GHI : BT_GLO;
    if (w >= n) {
        warp_bytes(dst + 8, blk, n, lane);
        w = 8 + n;
        type = BT_RAW;
    }
    if (lane == 0) put_block_header(dst, type, w - 8);
    __syncwarp();
    if (P.checksum) {
        const u32 crc = warp_checksum(dst + 8, w - 8, lane);
        if (lane == 0) st32(dst + w, crc);
        w += 4;
    }
    return w;
}

#ifndef ENC_OPT_MIN_CTAS
#define ENC_OPT_MIN_CTAS 0 /* resident CTAs per SM the level 6-7 instantiation is compiled for */
#endif
template <bool OPT>
__global__ void __launch_bounds__(ENC_CTA_THREADS, OPT ? ENC_OPT_MIN_CTAS : 0) zxc_encode_kernel(const EncodeParams P) {
    const u32 lane = threadIdx.x & 31;
    const u32 gwarp = blockIdx.x * ENC_WARPS_PER_CTA + (threadIdx.x >> 5);
    __shared__ u32 s_hist[OPT ? ENC_WARPS_PER_CTA : 1][256];
    u32* hist = s_hist[OPT ? (threadIdx.x >> 5) : 0];
    u8* scratch = P.scratch + (size_t)gwarp * P.scratch_stride;
    for (;;) {
        unsigned long long j = 0;
        if (lane == 0) j = atomicAdd(P.counter, 1ull);
        j = __shfl_sync(FULL, j, 0);
        if (j >= P.n_blocks) break;
        const unsigned long long off = j * (unsigned long long)P.block_size;
        const unsigned long long rem = P.src_size - off;
        const u32 n = rem < P.block_size ? (u32)rem : P.block_size;
        const u32 w = encode_block<OPT>(P, P.src + off, n, P.staging + (size_t)j * P.staging_stride, scratch, hist, lane);
        __syncwarp();
        if (lane == 0) P.out_size[j] = w;
    }
}

/* zxc_lz_seed_dict (zxc_compress.c:1060-1100): sparse first half (every 4th position, chain link
 * 0), dense second half with chain links.  Sequential by nature; runs once per call on one thread. */
__device__ __forceinline__ void seed_step(const u8* src, u32 i, u32 half, bool hash5, u32* head, unsigned short* chain) {
    if (i < half) {
        if ((i & 3u) == 0) {
            head[enc_hash(ldu64(src, i), hash5)] = i;
            chain[i & (ENC_WINDOW - 1)] = 0;
        }
    } else {
        const u32 h = enc_hash(ldu64(src, i), hash5);
        const u32 prev = head[h];
        head[h] = i;
        chain[i & (ENC_WINDOW - 1)] = (prev != 0 && i - prev < ENC_WINDOW) ? (unsigned short)(i - prev) : 0;
    }
}
/* The 4-byte hash of levels 1-2 mixes 6 input bytes, so the last seeded position reads the first
 * byte of the BLOCK; that one position is seeded per block (encode_block), the rest here. */
__device__ __forceinline__ u32 seed_shared_stop(u32 dict_size, bool hash5) {
    const u32 limit = dict_size - 4;
    return hash5 ? limit : limit - 1;
}
__global__ void zxc_seed_kernel(const u8* dict, u32 dict_size, u32 level, u32* head, unsigned short* chain) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (dict_size < 5) return;
    const bool hash5 = level >= 3;
    const u32 half = (dict_size - 4) / 2;
    const u32 stop = seed_shared_stop(dict_size, hash5);
    for (u32 i = 0; i < stop; i++) seed_step(dict, i, half, hash5, head, chain);
}

/* gather the per-block slots into the contiguous frame body */
__global__ void zxc_compact_kernel(const u8* staging, u32 staging_stride, const unsigned long long* dst_off,
                                   const u32* sizes, u8* out, u32 n_blocks) {
    const u32 lane = threadIdx.x & 31;
    const u32 warps = (gridDim.x * blockDim.x) >> 5;
    for (u32 j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n_blocks; j += warps) {
        const u8* s = staging + (size_t)j * staging_stride;
        u8* d = out + dst_off[j];
        const u32 n = sizes[j];
        for (u32 k = lane; k < n; k += 32) d[k] = s[k];
    }
}
