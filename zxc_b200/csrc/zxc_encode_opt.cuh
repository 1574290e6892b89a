/*
 * zxc_encode_opt.cuh -- levels 6-7 of the sm_90a block encoder (device code only): the price-based
 * optimal parser and the PivCo (Huffman) section writer, bit-identical to the reference's output.
 *
 * Replicated behaviour (SURVEY.md section 8 rows E4, E7):
 *   literal price         zxc_opt_estimate_lit_bits         src/lib/zxc_compress.c:720-749
 *   forward DP + emission zxc_lz77_optimal_parse_glo        src/lib/zxc_compress.c:795-1042
 *   section choice        zxc_encode_block_glo              src/lib/zxc_compress.c:1536-1626
 *   PivCo section bytes   zxc_pivco_encode_core             src/lib/zxc_huffman.c:1257-1342
 *   code lengths          zxc_hufenc.h (package-merge + nudge; also compiled and pinned on the host)
 *
 * Mechanism (one warp per block, as for levels 1-5):
 *   - match finding runs on batches of 32 * OPT_K consecutive positions.  The batch's inserts are
 *     applied in position order first (same-hash positions link to each other through
 *     __match_any_sync), then every lane walks OPT_K chains in lockstep so that the chain-link and
 *     gate-byte loads of all walks are in flight together.  The result per position is what the
 *     reference's sequential search returns because a walk only ever sees inserts of lower positions
 *     (a chain slot recycled by a higher position of the batch is read from a saved copy);
 *   - what is inherently sequential runs afterwards in position order: the repeat-offset probe (its
 *     length is known arithmetically while inside the last stretch measured at that offset) and the
 *     DP transitions.  A match of >= 256 bytes ends the batch there: the reference neither searches
 *     nor inserts the positions it covers, so the later inserts are undone;
 *   - DP state is one u64 per position: cost in the high word, (match length << 16 | biased offset)
 *     in the low word.  The entries of the next 64 positions live in registers (two per lane); a
 *     transition is a compare and a register move, strict '<' as in the reference, and only matches
 *     longer than that reach the global array;
 *   - the backtrack skips literal runs 32 positions per step, records match ends newest-first, and
 *     the emission walks that list forwards 32 sequences per step (scans for the literal / extras
 *     cursors);
 *   - the PivCo writer needs no trie: a symbol's path is (depth d, prefix v >> (len - d)) in the
 *     (level, value) geometry already used by the decoder (zxc_huffman.cuh); lanes that sit on the
 *     same node in the same step take consecutive bit slots (__match_any_sync), bits land with
 *     atomicOr on the zeroed run area.
 */
#pragma once
#include "zxc_hufenc.h"

#ifndef OPT_K
#define OPT_K 4 /* positions per lane in one match-finder batch */
#endif
#define OPT_MATCH_COST_BASE 24u
#define OPT_LONG_MATCH_SKIP 256u
#define OPT_LIT_SAMPLE_MIN 1024u
#define HUF_MIN_LITERALS 139u
#define ENC_RAW 0u
#define ENC_RLE 1u
#define ENC_HUF 2u
#define ENC_HUF_DICT 3u

/* per-warp tables of one PivCo section under construction (global scratch) */
struct PivcoPlan {
    u32 count[HUF_MAXNODES];
    u32 runoff[HUF_MAXNODES];
    u32 wpos[HUF_MAXNODES];
    u8 kind[HUF_MAXNODES];
    u8 sorted[256];
    unsigned short code[256]; /* canonical code value of each symbol */
    u32 first[HUF_MAXLEN + 2], cnt[HUF_MAXLEN + 2], lbase[HUF_MAXLEN + 2], leafb[HUF_MAXLEN + 2];
    u32 n_nodes, single, payload;
};

/* Builds the section geometry for (freq, code_len): node kinds, per-node symbol counts and run
 * offsets.  Returns the payload size in bytes (without the 128-byte lengths header), or 0xFFFFFFFF
 * when the lengths cannot encode this histogram (zxc_huffman.c:1042-1084, :1233-1249). */
__device__ u32 pivco_plan(const u32* freq, const u8* code_len, PivcoPlan* T, u32 lane) {
    u32 my_len[8];
    u32 kraft = 0, present = 0;
    bool bad = false;
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const u32 s = 32u * (u32)r + lane;
        const u32 l = code_len[s];
        my_len[r] = l;
        if (l > HUF_MAXLEN) bad = true;
        else if (l) {
            kraft += 1u << (HUF_MAXLEN - l);
            present++;
        } else if (freq[s] != 0) bad = true; /* a symbol of the histogram has no code */
    }
    if (__any_sync(FULL, bad)) return 0xFFFFFFFFu;
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
        kraft += __shfl_xor_sync(FULL, kraft, d);
        present += __shfl_xor_sync(FULL, present, d);
    }
    if (present == 0) return 0xFFFFFFFFu;
    u32 cnt[HUF_MAXLEN + 2], first[HUF_MAXLEN + 2], lbase[HUF_MAXLEN + 2], leafb[HUF_MAXLEN + 2];
#pragma unroll
    for (int l = 0; l <= HUF_MAXLEN + 1; l++) cnt[l] = 0;
    u32 base_l = 0;
    for (u32 l = 1; l <= HUF_MAXLEN; l++) {
        u32 c_l = 0;
#pragma unroll
        for (int r = 0; r < 8; r++) {
            const u32 m = __ballot_sync(FULL, my_len[r] == l);
            if (my_len[r] == l) T->sorted[base_l + c_l + __popc(m & ((1u << lane) - 1u))] = (u8)(32 * r + lane);
            c_l += __popc(m);
        }
        cnt[l] = c_l;
        base_l += c_l;
    }
    const bool single = (present == 1 && cnt[1] == 1 && kraft == (1u << (HUF_MAXLEN - 1)));
    if (kraft != (1u << HUF_MAXLEN) && !single) return 0xFFFFFFFFu;
    __syncwarp();
    if (single) {
        const u32 c = freq[T->sorted[0]];
        if (lane == 0) {
            T->single = 1;
            T->payload = (c + 7) >> 3;
        }
        __syncwarp();
        return (c + 7) >> 3;
    }
    {
        u32 code = 0, nodes = 1, leaves = 0;
        first[0] = 0;
        lbase[0] = 0;
        leafb[0] = 0;
        for (u32 l = 1; l <= HUF_MAXLEN; l++) {
            code = (code + cnt[l - 1]) << 1;
            first[l] = code;
            lbase[l] = nodes;
            leafb[l] = leaves;
            nodes += (1u << l) - code;
            leaves += cnt[l];
        }
        first[HUF_MAXLEN + 1] = 0;
        lbase[HUF_MAXLEN + 1] = nodes;
        leafb[HUF_MAXLEN + 1] = leaves;
        if (nodes > HUF_MAXNODES) return 0xFFFFFFFFu;
    }
    if (lane <= HUF_MAXLEN + 1) {
        T->first[lane] = first[lane];
        T->cnt[lane] = cnt[lane];
        T->lbase[lane] = lbase[lane];
        T->leafb[lane] = leafb[lane];
    }
    /* canonical code of every coded symbol: first[l] + its rank among the length-l symbols */
    for (u32 l = 1; l <= HUF_MAXLEN; l++)
        for (u32 t = lane; t < cnt[l]; t += 32) T->code[T->sorted[leafb[l] + t]] = (unsigned short)(first[l] + t);
    /* symbol counts, deepest level first */
    for (int l = HUF_MAXLEN; l >= 0; l--) {
        const u32 nn = (l == 0) ? 1u : (1u << l) - first[l];
        for (u32 t = lane; t < nn; t += 32) {
            const u32 id = lbase[l] + t;
            if (l > 0 && t < cnt[l]) T->count[id] = freq[T->sorted[leafb[l] + t]];
            else {
                const u32 v = first[l] + t;
                const u32 cid = lbase[l + 1] + (2u * v - first[l + 1]);
                T->count[id] = T->count[cid] + T->count[cid + 1];
            }
        }
        __syncwarp();
    }
    /* node kinds, parents before children (same rule as the decoder, zxc_huffman.cuh) */
    for (u32 l = 0; l <= HUF_MAXLEN; l++) {
        const u32 nn = (l == 0) ? 1u : (1u << l) - first[l];
        for (u32 t = lane; t < nn; t += 32) {
            const u32 v = first[l] + t;
            u32 kind;
            bool covered = false;
            if (l > 0) {
                const u32 pk = T->kind[lbase[l - 1] + (v >> 1) - first[l - 1]];
                covered = (pk >= 2 && pk <= HUF_MAXLEN) || pk == HUF_KIND_COVERED;
            }
            const bool leaf = (l > 0) && (t < cnt[l]);
            if (covered) kind = HUF_KIND_COVERED;
            else if (leaf) kind = HUF_KIND_LEAF;
            else {
                kind = HUF_KIND_BITMAP;
                for (u32 D = 1; l + D <= HUF_MAXLEN; D++) {
                    const u32 lo = v << D, hi = (v + 1) << D, ld = l + D;
                    const u32 leaf_end = first[ld] + cnt[ld];
                    if (hi <= leaf_end) {
                        if (D >= 2) kind = D;
                        break;
                    }
                    if (lo < leaf_end) break;
                }
            }
            T->kind[lbase[l] + t] = (u8)kind;
        }
        __syncwarp();
    }
    /* run offsets in BFS order */
    const u32 total_nodes = lbase[HUF_MAXLEN + 1];
    u32 roff = 0;
    for (u32 i0 = 0; i0 < total_nodes; i0 += 32) {
        const u32 id = i0 + lane;
        u32 bytes = 0;
        if (id < total_nodes) {
            const u32 kind = T->kind[id], c = T->count[id];
            if (kind == HUF_KIND_BITMAP) bytes = (c + 7) >> 3;
            else if (kind >= 2 && kind <= HUF_MAXLEN) bytes = (c * kind + 7) >> 3;
        }
        const u32 inc = warp_incl_scan(bytes, lane);
        if (id < total_nodes) {
            T->runoff[id] = roff + inc - bytes;
            T->wpos[id] = 0;
        }
        roff += __shfl_sync(FULL, inc, 31);
    }
    if (lane == 0) {
        T->single = 0;
        T->n_nodes = total_nodes;
        T->payload = roff;
    }
    __syncwarp();
    return roff;
}

/* ORs `bits` (<= 11 significant bits) into the little-endian bit stream at bit position bitpos of out */
__device__ __forceinline__ void or_bits(u8* out, u32 bitpos, u32 bits) {
    u8* a = out + (bitpos >> 3);
    const uintptr_t ua = reinterpret_cast<uintptr_t>(a);
    u32* w = reinterpret_cast<u32*>(ua & ~(uintptr_t)3);
    const u32 sh = (u32)(ua & 3u) * 8u + (bitpos & 7u);
    const u64 v = (u64)bits << sh;
    if ((u32)v) atomicOr(w, (u32)v);
    if ((u32)(v >> 32)) atomicOr(w + 1, (u32)(v >> 32));
}

/* Writes one PivCo section (optionally led by the 128-byte packed lengths) for a plan made by
 * pivco_plan with the same (freq, code_len).  Returns bytes written. */
__device__ u32 pivco_write(const u8* sym, u32 n, const u8* code_len, PivcoPlan* T, u8* dst, bool with_header, u32 lane) {
    u32 hdr = 0;
    if (with_header) {
        for (u32 k = lane; k < 128; k += 32) dst[k] = (u8)((code_len[2 * k] & 15u) | ((code_len[2 * k + 1] & 15u) << 4));
        hdr = 128;
    }
    u8* out = dst + hdr;
    const u32 payload = T->payload;
    for (u32 k = lane; k < payload; k += 32) out[k] = 0;
    __syncwarp();
    if (T->single) return hdr + payload; /* every symbol goes left at the root: all-zero bitmap */
    u32 first[HUF_MAXLEN + 2], lbase[HUF_MAXLEN + 2];
#pragma unroll
    for (int l = 0; l <= HUF_MAXLEN + 1; l++) {
        first[l] = T->first[l];
        lbase[l] = T->lbase[l];
    }
    for (u32 i0 = 0; i0 < n; i0 += 32) {
        const u32 i = i0 + lane;
        bool active = i < n;
        u32 l = 0, v = 0, d = 0;
        if (active) {
            const u32 s = sym[i];
            l = code_len[s];
            v = T->code[s];
        }
        for (;;) {
            const u32 am = __ballot_sync(FULL, active);
            if (!am) break;
            if (active) {
                const u32 id = lbase[d] + ((v >> (l - d)) - first[d]);
                const u32 kind = T->kind[id];
                const u32 grp = __match_any_sync(am, id);
                const u32 rank = __popc(grp & ((1u << lane) - 1u));
                const int leader = __ffs(grp) - 1;
                u32 base = 0;
                if ((int)lane == leader) {
                    ZXC_LANE_STAT(90, __popc(grp) > 1); /* lanes on one node take consecutive slots */
                    base = T->wpos[id];
                    T->wpos[id] = base + __popc(grp);
                }
                base = __shfl_sync(grp, base, leader);
                const u32 slot = base + rank;
                if (kind == HUF_KIND_BITMAP) {
                    const u32 bit = (v >> (l - d - 1)) & 1u;
                    if (bit) or_bits(out + T->runoff[id], slot, 1u);
                    d++;
                    if (d >= l) active = false;
                } else { /* flat root of depth `kind`: the remaining path, first branch in bit 0 */
                    ZXC_LANE_STAT(89, 1);
                    const u32 low = v & ((1u << kind) - 1u);
                    const u32 r = __brev(low) >> (32u - kind);
                    if (r) or_bits(out + T->runoff[id], slot * kind, r);
                    active = false;
                }
            }
            __syncwarp();
        }
    }
    __syncwarp();
    __threadfence_block();
    return hdr + payload;
}

/* byte histogram of sym[0..n) stepping by `step`, into hist[256] (shared memory, this warp's) */
__device__ __forceinline__ u32 warp_histogram(const u8* sym, u32 n, u32 step, u32* hist, u32 lane) {
    for (u32 k = lane; k < 256; k += 32) hist[k] = 0;
    __syncwarp();
    u32 cnt = 0;
    for (u32 i = lane * step; i < n; i += 32u * step) {
        atomicAdd(&hist[sym[i]], 1u);
        cnt++;
    }
    __syncwarp();
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) cnt += __shfl_xor_sync(FULL, cnt, d);
    return cnt;
}

/* extras cost of a match of length L in the DP (zxc_compress.c:904-950) */
__device__ __forceinline__ u32 opt_match_cost(u32 L) {
    const u32 ml = L - 5u;
    if (ml < 15u) return OPT_MATCH_COST_BASE;
    const u32 v = ml - 15u;
    return OPT_MATCH_COST_BASE + (v < 128u ? 8u : (v < 16384u ? 16u : 24u));
}

/* common prefix of src[a..] and src[b..] (b < a) with a + len <= iend, one lane on its own; the
 * first `known` bytes are already known equal */
__device__ __forceinline__ u32 lane_lcp(const u8* src, u32 a, u32 b, u32 iend, u32 known) {
    u32 len = known;
    while (a + len + 8u <= iend) {
        const u64 x = ldu64(src, a + len) ^ ldu64(src, b + len);
        if (x) return len + ((u32)(__ffsll((long long)x) - 1) >> 3);
        len += 8u;
    }
    while (a + len < iend && src[a + len] == src[b + len]) len++;
    return len;
}

/* The DP front lives in registers: lane j holds the entries of positions cbase + j (A) and
 * cbase + 32 + j (B) of the 32-aligned chunk being processed.  Transitions that land inside these 64
 * positions are register updates; longer ones go to the global array, which is also where chunks are
 * loaded from (already carrying those long transitions) and retired to for the backtrack. */
struct DpFront {
    u64 A, B;
    u32 cbase;
};
#define DP_INF 0xFFFFFFFF00000000ull

__device__ __forceinline__ void dp_front_init(DpFront& F, u64* dp, u32 n, u32 lane) {
    F.cbase = 0;
    F.A = lane <= n ? dp[lane] : DP_INF;
    F.B = 32 + lane <= n ? dp[32 + lane] : DP_INF;
}
__device__ __forceinline__ void dp_front_advance(DpFront& F, u64* dp, u32 n, u32 pi, u32 lane) {
    while (pi >= F.cbase + 32) {
        if (F.cbase + lane <= n) dp[F.cbase + lane] = F.A;
        F.A = F.B;
        F.cbase += 32;
        __syncwarp();
        F.B = F.cbase + 32 + lane <= n ? dp[F.cbase + 32 + lane] : DP_INF;
    }
}
__device__ __forceinline__ void dp_front_flush(DpFront& F, u64* dp, u32 n, u32 lane) {
    if (F.cbase + lane <= n) dp[F.cbase + lane] = F.A;
    if (F.cbase + 32 + lane <= n) dp[F.cbase + 32 + lane] = F.B;
    __syncwarp();
}
/* all transitions out of position pi (zxc_compress.c:879-951); found/L_max/offb are warp-uniform */
__device__ __forceinline__ void dp_front_step(DpFront& F, u64* dp, u32 n, u32 pi, u32 lit_cost, bool found, u32 L_max,
                                              u32 offb, u32 lane) {
    dp_front_advance(F, dp, n, pi, lane);
    const u32 i = pi - F.cbase;
    const u32 cur = __shfl_sync(FULL, (u32)(F.A >> 32), i);
    if (cur == 0xFFFFFFFFu) return;
    const u32 lit_next = cur + lit_cost;
    if (i < 31) {
        if (lane == i + 1 && lit_next < (u32)(F.A >> 32)) F.A = (u64)lit_next << 32;
    } else if (lane == 0 && lit_next < (u32)(F.B >> 32)) F.B = (u64)lit_next << 32;
    if (!found) return;
    const u32 span_end = i + L_max;          /* last target, relative to the chunk */
    const bool cheap = L_max < 20u;          /* every length up to L_max costs the base price (no extras byte) */
    {
        const u32 L = lane - i; /* target in A */
        if (lane >= i + 5 && L <= L_max) {
            const u32 nxt = cur + (cheap ? OPT_MATCH_COST_BASE : opt_match_cost(L));
            if (nxt < (u32)(F.A >> 32)) F.A = ((u64)nxt << 32) | (L << 16) | offb;
        }
    }
    if (span_end < 32) return;
    {
        const u32 L = lane + 32 - i; /* target in B */
        if (L >= 5 && L <= L_max) {
            const u32 nxt = cur + (cheap ? OPT_MATCH_COST_BASE : opt_match_cost(L));
            if (nxt < (u32)(F.B >> 32)) F.B = ((u64)nxt << 32) | (L << 16) | offb;
        }
    }
    if (span_end >= 64) { /* beyond the register front */
        ZXC_STAT(75, 1);
        for (u32 L = 64 - i + lane; L <= L_max; L += 32) {
            const u32 nxt = cur + opt_match_cost(L);
            if (nxt < (u32)(dp[pi + L] >> 32)) dp[pi + L] = ((u64)nxt << 32) | (L << 16) | offb;
        }
        __syncwarp();
    }
}

#ifdef ZXC_OPT_PROFILE
#define OPT_T(k) { const long long t_ = clock64(); prof[k] += t_ - tprev; tprev = t_; }
#else
#define OPT_T(k)
#endif

struct OptOut {
    u32 seq_c, lit_c, ext_c, max_off;
};

/* zxc_lz77_optimal_parse_glo: fills literals / tokens / offsets / extras for block bytes
 * src[base .. base+n).  dp: n+1 u64; ends: >= n/5 + 32 u32. */
__device__ OptOut optimal_parse(const u8* src, u32 base, u32 n, u32* head, unsigned short* chain, int level,
                                const LzParams& lzp, u64* dp, u32* ends, u8* literals, u8* tokens,
                                unsigned short* offsets, u8* extras, u32* hist, zxh_work_t* W, u8* cl_tmp, u32 lane) {
    OptOut R = {0, 0, 0, 0};
    const u8* blk = src + base;
    if (n < 9) {
        warp_bytes(literals, blk, n, lane);
        R.lit_c = n;
        return R;
    }
    /* literal price from a strided sample through the real code builder */
    u32 lit_cost = 8;
    if (n >= OPT_LIT_SAMPLE_MIN) {
        const u32 step = n > 4096 ? (n >> 12) : 1u;
        const u32 sampled = warp_histogram(blk, n, step, hist, lane);
        if (lane == 0) lit_cost = zxh_estimate_lit_bits(hist, sampled, cl_tmp, W);
        lit_cost = __shfl_sync(FULL, lit_cost, 0);
    }
    for (u32 k = lane; k <= n; k += 32) dp[k] = k ? 0xFFFFFFFF00000000ull : 0ull;
    __syncwarp();

    const u32 iend = base + n;
    const u32 slp = n - 8; /* positions >= slp are literal-only (ZXC_LZ_SEARCH_MARGIN) */
    unsigned short* oldc = reinterpret_cast<unsigned short*>(hist); /* chain slots displaced by the current batch */
    u32 p = 0, skip_until = 0, last_off = 0, rk_pos = 0, rk_len = 0;
#ifdef ZXC_OPT_PROFILE
    long long prof[8] = {0, 0, 0, 0, 0, 0, 0, 0}, tprev = clock64();
    u32 n_batches = 0, n_trunc = 0, n_arith = 0, n_spec = 0, n_load = 0, n_lcp = 0, n_far = 0;
#endif
    DpFront F;
    dp_front_init(F, dp, n, lane);
    while (p < n) {
        __syncwarp();
        if (p < skip_until || p >= slp) {
            /* literal-only stretch */
            const u32 end = p >= slp ? n : min(skip_until, slp);
            for (u32 q = p; q < end; q++) dp_front_step(F, dp, n, q, lit_cost, false, 0, 0, lane);
            p = end;
            OPT_T(0)
            continue;
        }
        /* ---- one batch: up to 32 * OPT_K consecutive searched positions, OPT_K per lane (position
         * p + 32k + lane is "index" 32k + lane); the OPT_K chain walks of a lane advance in lockstep
         * so their loads overlap ---- */
        const u32 nact = min(32u * OPT_K, slp - p);
        const u32 pos0 = base + p;
        u32 cur_val[OPT_K], hh[OPT_K], grp[OPT_K], midx[OPT_K];
        u64 nxt8[OPT_K]; /* bytes 4..11 after each position: the first step of every candidate compare */
        bool skip_head[OPT_K];
#pragma unroll
        for (int k = 0; k < OPT_K; k++) {
            const u32 my = 32u * k + lane;
            const bool act = my < nact;
            const u32 am = __ballot_sync(FULL, act);
            const u32 pos = pos0 + my;
            u64 cur8 = 0;
            hh[k] = 0;
            grp[k] = 0;
            midx[k] = 0;
            if (act) {
                cur8 = ldu64(src, pos);
                hh[k] = enc_hash(cur8, true);
                grp[k] = __match_any_sync(am, hh[k]);
                const u32 lower = grp[k] & ((1u << lane) - 1u);
                /* what head[h] holds once every lower position has inserted */
                midx[k] = lower ? pos0 + 32u * k + (31u - (u32)__clz(lower)) : head[hh[k]];
            }
            cur_val[k] = (u32)cur8;
            nxt8[k] = act ? ldu64(src, pos + 4) : 0;
            skip_head[k] = act && midx[k] && enc_tag(ldu32(src, midx[k])) != enc_tag(cur_val[k]);
            __syncwarp();
            if (act) {
                const u32 slot = pos & (ENC_WINDOW - 1);
                oldc[my] = chain[slot];
                const u32 dist = pos - midx[k];
                chain[slot] = (midx[k] != 0 && dist < ENC_WINDOW) ? (unsigned short)dist : 0;
                if (lane == 31u - (u32)__clz(grp[k])) { /* provisional: undone on truncation */
                    ZXC_LANE_STAT(70, __popc(grp[k]) > 1); /* insert groups of more than one lane */
                    head[hh[k]] = pos;
                }
            }
            __syncwarp();
        }
        OPT_T(1)
        /* lane-local chain walks (:256-437); a slot overwritten by a HIGHER index still reads as before */
        u32 c_len[OPT_K], c_ref[OPT_K], idx[OPT_K], tb[OPT_K]; /* tb: the byte a longer match must continue with */
        int att[OPT_K];
        bool c_found[OPT_K];
#define OPT_RDCHAIN(q, my, out)                                                              \
    {                                                                                        \
        const u32 jj = ((q) - pos0) & (ENC_WINDOW - 1);                                      \
        const u32 cv_ = chain[(q) & (ENC_WINDOW - 1)];                                       \
        ZXC_LANE_STAT(68, jj > (my) && jj < nact);                                           \
        out = (jj > (my) && jj < nact) ? (u32)oldc[jj] : cv_;                                \
    }
#pragma unroll
        for (int k = 0; k < OPT_K; k++) {
            c_len[k] = 4;
            tb[k] = (u32)nxt8[k] & 0xFFu;
            c_ref[k] = 0;
            c_found[k] = false;
            att[k] = lzp.search_depth;
            idx[k] = midx[k]; /* 0 for inactive lanes */
            if (skip_head[k]) {
                ZXC_LANE_STAT(92, 1);
                u32 delta;
                OPT_RDCHAIN(idx[k], 32u * k + lane, delta);
                idx[k] = delta ? idx[k] - delta : 0;
                att[k]--;
            }
        }
        for (;;) {
            bool live = false;
            u32 delta[OPT_K], oc[OPT_K], gb[OPT_K];
            /* issue every load of this step before anything consumes one: the chain link and the
             * reference's gate byte ref[best.len] (:281) -- two sectors per candidate */
#pragma unroll
            for (int k = 0; k < OPT_K; k++) {
                const u32 pos = pos0 + 32u * k + lane;
                ZXC_LANE_STAT(77, idx[k] > 0 && att[k] >= 0 && pos - idx[k] > ENC_MAX_DIST);
                if (idx[k] > 0 && (att[k]-- < 0 || pos - idx[k] > ENC_MAX_DIST)) idx[k] = 0;
                const u32 q = idx[k]; /* q == 0 reads slot 0 / byte c_len: harmless, ignored below */
                const u32 jj = (q - pos0) & (ENC_WINDOW - 1);
                delta[k] = chain[q & (ENC_WINDOW - 1)];
                gb[k] = src[q + c_len[k]];
                oc[k] = oldc[jj < 32u * OPT_K ? jj : 0u];
            }
#pragma unroll
            for (int k = 0; k < OPT_K; k++) {
                const u32 q = idx[k];
                const u32 jj = (q - pos0) & (ENC_WINDOW - 1);
                if (jj > 32u * k + lane && jj < nact) {
                    ZXC_LANE_STAT(69, q != 0); /* a link the batch has already overwritten */
                    delta[k] = oc[k];
                }
            }
#pragma unroll
            for (int k = 0; k < OPT_K; k++) {
                if (idx[k] == 0) continue;
                const u32 pos = pos0 + 32u * k + lane;
                bool stop = false;
                /* a candidate failing the gate cannot be longer than the best so far; one passing it is
                 * compared in full: first 4 bytes equal (:277-278), then the length */
                if (gb[k] == tb[k] && ldu32(src, idx[k]) == cur_val[k]) {
                    u32 mlen;
                    const u64 x = ldu64(src, idx[k] + 4) ^ nxt8[k];
                    if (pos + 12u > iend) mlen = lane_lcp(src, pos, idx[k], iend, 4);
                    else if (x) mlen = 4u + ((u32)(__ffsll((long long)x) - 1) >> 3);
                    else mlen = lane_lcp(src, pos, idx[k], iend, 12);
                    if (mlen > c_len[k]) {
                        c_len[k] = mlen;
                        c_ref[k] = idx[k];
                        c_found[k] = true;
                        /* next gate byte: from registers while it is within bytes 4..11 (padded past iend; unused
                         * once pos + mlen == iend, which stops the walk) */
                        tb[k] = mlen < 12u ? (u32)(nxt8[k] >> (8u * (mlen - 4u))) & 0xFFu : (u32)src[pos + mlen];
                    }
                    stop = c_len[k] >= (u32)lzp.sufficient_len || pos + c_len[k] >= iend;
                }
                idx[k] = (stop || delta[k] == 0) ? 0 : idx[k] - delta[k];
                live |= idx[k] > 0;
            }
            if (!live) break;
        }
#undef OPT_RDCHAIN
        __syncwarp();
        OPT_T(2)
        /* the repeat offset a position will most likely be probed with: the chain offset of the nearest
         * lower position that found a match (exact unless a repeat match won there) */
        bool spec_eq[OPT_K];
        u32 spec[OPT_K];
        {
            u32 carry = last_off;
#pragma unroll
            for (int k = 0; k < OPT_K; k++) {
                const u32 pos = pos0 + 32u * k + lane;
                const u32 fm = __ballot_sync(FULL, c_found[k]);
                const u32 lowerf = fm & ((1u << lane) - 1u);
                const int sl = lowerf ? 31 - __clz(lowerf) : 0;
                const u32 so = __shfl_sync(FULL, pos - c_ref[k], sl);
                spec[k] = lowerf ? so : carry;
                if (fm) carry = __shfl_sync(FULL, pos - c_ref[k], 31 - __clz(fm));
                spec_eq[k] = false;
                if (32u * k + lane < nact && spec[k] != 0 && spec[k] <= ENC_MAX_DIST && spec[k] <= pos)
                    spec_eq[k] = ldu32(src, pos - spec[k]) == cur_val[k];
            }
        }
        OPT_T(3)
        /* in order: repeat-offset probe (:233-254), then the DP transitions of each position */
        u32 valid = nact;
        bool truncated = false;
#pragma unroll
        for (int k = 0; k < OPT_K; k++) {
            if (truncated || 32u * k >= nact) break;
            const u32 gn = min(32u, nact - 32u * k);
            for (u32 i = 0; i < gn; i++) {
                const u32 pi = p + 32u * k + i, posi = pos0 + 32u * k + i;
                u32 len = __shfl_sync(FULL, c_found[k] ? c_len[k] : 0u, i);
                u32 ref = __shfl_sync(FULL, c_ref[k], i);
                bool found = len != 0;
                if (last_off != 0 && last_off <= ENC_MAX_DIST && last_off <= posi) {
                    /* lcp(posi, posi - last_off): known without touching memory while posi is still inside
                     * the last stretch measured at this offset (rk_len bytes from rk_pos) */
                    u32 rl = 0;
                    bool eq;
                    if (posi - rk_pos < rk_len) {
                        ZXC_STAT(71, 1);
                        rl = rk_len - (posi - rk_pos);
                        eq = rl >= 4;
#ifdef ZXC_OPT_PROFILE
                        n_arith++;
#endif
                    } else {
                        const u32 sp = __shfl_sync(FULL, spec[k], i);
                        ZXC_STAT(72, sp == last_off);
                        ZXC_STAT(73, sp != last_off);
#ifdef ZXC_OPT_PROFILE
                        if (sp == last_off) n_spec++; else n_load++;
#endif
                        if (sp == last_off) eq = __shfl_sync(FULL, (u32)spec_eq[k], i) != 0;
                        else eq = ldu32(src, posi - last_off) == __shfl_sync(FULL, cur_val[k], i);
                        if (eq) rl = warp_lcp(src, posi, posi - last_off, iend, 4, 0xFFFFFFFFu, lane);
#ifdef ZXC_OPT_PROFILE
                        n_lcp += eq;
#endif
                    }
                    if (eq) {
                        const bool fin = rl >= (u32)lzp.sufficient_len || posi + rl >= iend;
                        if (fin || !found || len <= rl) { /* ties go to the repeat offset */
                            ZXC_STAT(74, found && len == rl);
                            found = true;
                            len = rl;
                            ref = posi - last_off;
                        }
                    }
                }
                u32 L_max = 0, offb = 0;
                if (found) {
                    const u32 off = posi - ref;
                    last_off = off;
                    rk_pos = posi; /* len is the full common prefix at this offset */
                    rk_len = len;
                    L_max = len > n - pi ? n - pi : len;
                    if (L_max > 65535u) {
                        ZXC_STAT(76, 1);
                        L_max = 65535u;
                    }
                    offb = (off - 1u) & 0xFFFFu;
                }
#ifdef ZXC_OPT_PROFILE
                const long long t_a = clock64();
#endif
                dp_front_step(F, dp, n, pi, lit_cost, found, L_max, offb, lane);
#ifdef ZXC_OPT_PROFILE
                prof[6] += clock64() - t_a;
                n_far += found && L_max >= 64 - ((pi) & 31u);
#endif
                if (L_max >= OPT_LONG_MATCH_SKIP) { /* positions inside a long match are neither searched nor inserted */
                    skip_until = pi + L_max - 1;
                    valid = 32u * k + i + 1;
                    truncated = true;
                    break;
                }
            }
        }
        __syncwarp();
        OPT_T(4)
        ZXC_STAT(64, 1);
        ZXC_STAT(65, valid != nact);
        if (valid != nact) {
            /* undo the inserts past `valid`, highest first: each hash ends up pointing at what its lowest
             * undone position had found there */
#pragma unroll
            for (int k = OPT_K - 1; k >= 0; k--) {
                const u32 my = 32u * k + lane;
                const bool inv = my >= valid && my < nact;
                const u32 invm = __ballot_sync(FULL, inv);
                if (inv) {
                    chain[(pos0 + my) & (ENC_WINDOW - 1)] = oldc[my];
                    ZXC_LANE_STAT(67, 1);
                    if ((grp[k] & invm & ((1u << lane) - 1u)) == 0) {
                        ZXC_LANE_STAT(66, 1); /* the lowest undone position of its hash restores the head */
                        head[hh[k]] = midx[k];
                    }
                }
                __syncwarp();
            }
        }
        p += valid;
        OPT_T(5)
#ifdef ZXC_OPT_PROFILE
        n_batches++;
        n_trunc += valid != nact;
#endif
    }
#ifdef ZXC_OPT_PROFILE
    if (lane == 0)
        printf("opt profile n=%u batches=%u trunc=%u | cycles: litonly %lld insert %lld walk %lld spec %lld fixup+dp %lld commit %lld | rep arith %u spec %u load %u lcp %u far %u dpstep %lld\n", n,
               n_batches, n_trunc, prof[0], prof[1], prof[2], prof[3], prof[4], prof[5], n_arith, n_spec, n_load, n_lcp, n_far, prof[6]);
#endif
    dp_front_flush(F, dp, n, lane);

    /* backtrack: match ends, newest first */
    u32 count = 0;
    {
        u32 pos = n;
        while (pos > 0) {
            const bool in = pos > lane;
            const u32 q = pos - lane;
            const u32 L = in ? (((u32)dp[q]) >> 16) : 0u;
            const u32 hit = __ballot_sync(FULL, !in || L != 0);
            if (!hit) {
                pos -= 32;
                continue;
            }
            const int f = __ffs(hit) - 1;
            const u32 fin = __shfl_sync(FULL, (u32)in, f);
            if (!fin) break; /* ran off the front through literals */
            const u32 fq = pos - (u32)f;
            const u32 fL = __shfl_sync(FULL, L, f);
            if (lane == 0) ends[count] = fq;
            count++;
            pos = fq - fL;
        }
    }
    __syncwarp();

    /* forward emission, 32 sequences per step */
    u32 lit_c = 0, ext_c = 0, max_off = 0;
    for (u32 k0 = 0; k0 < count; k0 += 32) {
        const u32 k = k0 + lane;
        const bool on = k < count;
        u32 e = 0, prev_e = 0, L = 5, offb = 0;
        if (on) {
            e = ends[count - 1 - k];
            prev_e = k ? ends[count - k] : 0u;
            const u32 lo = (u32)dp[e];
            L = lo >> 16;
            offb = lo & 0xFFFFu;
        }
        const u32 ms = e - L;
        const u32 ll = on ? ms - prev_e : 0u;
        const u32 ml = L - 5u;
        u32 nb = 0;
        if (on) {
            if (ll >= 15u) {
                const u32 v = ll - 15u;
                nb += v < 128u ? 1u : (v < 16384u ? 2u : 3u);
            }
            if (ml >= 15u) {
                const u32 v = ml - 15u;
                nb += v < 128u ? 1u : (v < 16384u ? 2u : 3u);
            }
        }
        const u32 s_ll = warp_incl_scan(ll, lane);
        const u32 s_nb = warp_incl_scan(nb, lane);
        const u32 my_lit = lit_c + s_ll - ll;
        if (on) {
            tokens[k] = (u8)(((ll >= 15u ? 15u : ll) << 4) | (ml >= 15u ? 15u : ml));
            offsets[k] = (unsigned short)offb;
            u8* x = extras + ext_c + s_nb - nb;
            if (ll >= 15u) x += put_varint(x, ll - 15u);
            if (ml >= 15u) put_varint(x, ml - 15u);
        }
        u32 mo = on ? offb : 0u;
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) mo = max(mo, __shfl_xor_sync(FULL, mo, d));
        max_off = max(max_off, mo);
        const u32 nseq = min(32u, count - k0);
        for (u32 j = 0; j < nseq; j++) {
            const u32 j_ll = __shfl_sync(FULL, ll, j);
            if (j_ll == 0) continue;
            const u32 j_src = __shfl_sync(FULL, prev_e, j);
            const u32 j_dst = __shfl_sync(FULL, my_lit, j);
            warp_bytes(literals + j_dst, blk + j_src, j_ll, lane);
        }
        lit_c += __shfl_sync(FULL, s_ll, 31);
        ext_c += __shfl_sync(FULL, s_nb, 31);
    }
    const u32 lit_start = count ? ends[0] : 0u;
    if (lit_start < n) {
        warp_bytes(literals + lit_c, blk + lit_start, n - lit_start, lane);
        lit_c += n - lit_start;
    }
    __syncwarp();
    R.seq_c = count;
    R.lit_c = lit_c;
    R.ext_c = ext_c;
    R.max_off = max_off;
    return R;
}

/* The nudge's grouped DP (zxh_dp_solve) with the destinations of each level spread over the lanes;
 * zxh_dp_pull visits a destination's sources in the reference's order, so ties resolve identically. */
__device__ int warp_dp_solve(const u64* pfg, int m, int cap_c, int lu, int g_log2, u32* out_cblc, zxh_work_t* W, u32 lane) {
    if (m < 2 || cap_c < 1 || m > ZXH_DP_M) return 0;
    const u32 row = (u32)(m + 1), plane = row * row;
    u64* jcur = W->dp_a;
    u64* jnxt = W->dp_b;
    for (u32 i = lane; i < plane; i += 32) jcur[i] = (i == 2) ? 0ull : ZXH_U64MAX;
    __syncwarp();
    zxh_dp_best_t B;
    B.j = ZXH_U64MAX;
    B.l = B.k = B.s = 0;
    const u32 hm = (u32)m / 2, ndest = row * hm;
    for (int lc = 1; lc <= cap_c; lc++) {
        u64 bj = ZXH_U64MAX;
        u32 bk = 0;
        for (u32 k = lane; k < (u32)m; k += 32) {
            const u64 j = zxh_dp_finish(pfg, jcur, m, lu, g_log2, lc, k);
            if (j < bj) {
                bj = j;
                bk = k;
            }
        }
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) { /* lowest cost, then lowest row: the first one a serial scan keeps */
            const u64 oj = __shfl_xor_sync(FULL, bj, d);
            const u32 ok = __shfl_xor_sync(FULL, bk, d);
            if (oj < bj || (oj == bj && ok < bk)) {
                bj = oj;
                bk = ok;
            }
        }
        if (bj < B.j) {
            B.j = bj;
            B.l = lc;
            B.k = (int)bk;
            B.s = m - (int)bk;
        }
        if (lc == cap_c) break;
        for (u32 i = lane; i < plane; i += 32) jnxt[i] = ZXH_U64MAX;
        __syncwarp();
        for (u32 d = lane; d < ndest; d += 32) {
            const u32 kd = d / hm, sd = 2u * (d % hm + 1u);
            u32 c;
            const u64 j = zxh_dp_pull(pfg, jcur, m, cap_c, lu, g_log2, lc, kd, sd, &c);
            if (j != ZXH_U64MAX) {
                jnxt[kd * row + sd] = j;
                W->arrive[(u32)(lc + 1) * plane + kd * row + sd] = (unsigned short)c;
            }
        }
        __syncwarp();
        u64* t = jcur;
        jcur = jnxt;
        jnxt = t;
    }
    int ok = 0;
    if (lane == 0) ok = zxh_dp_backtrack(W->arrive, m, &B, out_cblc);
    __syncwarp();
    return __shfl_sync(FULL, ok, 0);
}

/* code lengths for one section at level >= 6: package-merge, then the nudge (serial parts on lane 0,
 * its grouped DP warp-wide; the result is in global memory for every lane after the trailing
 * barrier).  false when no code could be built. */
__device__ bool build_section_lengths(const u32* freq, u8* code_len, int cap, zxh_work_t* W, u32 lane) {
    int ok = 0, go = 0;
    zxh_nudge_t S;
    S.do_dp = S.m = S.cap_c = S.g_log2 = 0;
    if (lane == 0) {
        ok = zxh_build_code_lengths(freq, code_len, cap, W) == 0;
        if (ok) go = zxh_nudge_begin(freq, code_len, cap, W, &S);
    }
    __syncwarp();
    ok = __shfl_sync(FULL, ok, 0);
    go = __shfl_sync(FULL, go, 0);
    if (ok && go) {
        const int do_dp = __shfl_sync(FULL, S.do_dp, 0), m = __shfl_sync(FULL, S.m, 0);
        const int cap_c = __shfl_sync(FULL, S.cap_c, 0), g_log2 = __shfl_sync(FULL, S.g_log2, 0);
        int dp_ok = 0;
        if (do_dp) dp_ok = warp_dp_solve(W->pfg, m, cap_c, ZXH_LU - g_log2, g_log2, W->cblc, W, lane);
        if (lane == 0) (void)zxh_nudge_end(freq, code_len, W, &S, dp_ok, W->cblc);
    }
    __syncwarp();
    return ok != 0;
}
