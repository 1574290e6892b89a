/*
 * zxc_huffman.cuh -- PivCo (level-ordered canonical Huffman) section decode, one warp per section.
 *
 * Wire format: docs/FORMAT.md:246-343.  Reference decoder: src/lib/zxc_huffman.c:1042-1170 (tree,
 * flat roots), :2271-2430 (popcount pass + bottom-up merges).  The reference merges child
 * sequences bottom-up with SIMD shuffles; here every output symbol walks the tree top-down with
 * rank queries (SURVEY.md Appendix D point 6), which needs no ping-pong buffers:
 *
 *   at a bitmap node with local index i: bit = run[i]; child index = rank_bit(i)
 *   at a flat root with local index i:   the D-bit path at bit i*D names the leaf
 *
 * A canonical, Kraft-complete code needs no explicit trie: at depth l the existing nodes are the
 * l-bit prefixes v in [first[l], 2^l), the first cnt[l] of them leaves (in symbol order), the rest
 * internal with children 2v and 2v+1; BFS order inside a level is increasing v.  So a node is just
 * (l, v) and its BFS index is level_base[l] + v - first[l].
 *
 * Work area (per warp, global scratch): node table (count, run offset, rank-table offset, kind)
 * for <= 511 nodes, the symbols sorted by (length, value), and one cumulative popcount per 32 run
 * bits of every bitmap node.
 */
#pragma once

#ifndef ZXC_STAT
#define ZXC_STAT(i, v) /* tests/simt counts events here (lane 0 only); nothing in the product build */
#endif
/* emulator counters of this file (tests/simt): 32 single-symbol sections, 33 lanes that took a bitmap step, 34 rank
 * words filled, 35 verdicts, 40 + D symbols read from a flat root of depth D */
#define HUF_FAIL()                   \
    do {                             \
        ZXC_STAT(35, 1);             \
        return ZXC_ERROR_CORRUPT_DATA; \
    } while (0)

#define HUF_MAXLEN 11
#define HUF_MAXNODES 512
#define HUF_KIND_LEAF 0u
#define HUF_KIND_BITMAP 1u
#define HUF_KIND_COVERED 255u /* strict descendant of a flat root: emits no run */
/* kind >= 2 && kind <= 11: flat root of that depth */

struct HufWork {
    u32 count[HUF_MAXNODES];
    u32 runoff[HUF_MAXNODES];
    u32 cumoff[HUF_MAXNODES];
    u8 kind[HUF_MAXNODES];
    u8 sorted[256];
    u32 first[HUF_MAXLEN + 2], cnt[HUF_MAXLEN + 2], level_base[HUF_MAXLEN + 2], leaf_base[HUF_MAXLEN + 2];
};
#define HUF_WORK_BYTES ((sizeof(HufWork) + 255u) & ~255u)

/* byte k of the run area, 0 past its end: the 4-byte bitmap word and the 3-byte flat path of a symbol in the last
 * node's run may reach past the section, which can be the end of the source buffer */
__device__ __forceinline__ u32 huf_byte(const u8* runs, u32 rsz, u32 k) { return k < rsz ? (u32)runs[k] : 0u; }
__device__ __forceinline__ u32 huf_bits32(const u8* runs, u32 rsz, u32 k) { /* 32 run bits starting at byte k */
    return huf_byte(runs, rsz, k) | (huf_byte(runs, rsz, k + 1) << 8) | (huf_byte(runs, rsz, k + 2) << 16) |
           (huf_byte(runs, rsz, k + 3) << 24);
}

/* Decodes n symbols.  lens128: 128 packed nibbles; runs/rsz: the run area; cum: cum_words rank words.
 * Every symbol sits in at most one bitmap node per level, so a well-formed section needs at most
 * HUF_MAXLEN * n / 32 + HUF_MAXNODES rank words (scr_cum_cap); a crafted one that asks for more is
 * rejected before the table is written. */
__device__ __noinline__ int pivco_decode(const u8* lens128, const u8* runs, u32 rsz, u8* out, u32 n, HufWork* W,
                                         u32* cum, u32 cum_words, u32 lane) {
    /* ---- code lengths: validate, count, Kraft (zxc_huffman.c:1055-1064) ---- */
    u32 my_len[8];
    u32 kraft = 0, present = 0;
    bool bad = false;
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const u32 s = 32u * (u32)r + lane;
        const u32 byte = lens128[s >> 1];
        const u32 l = (s & 1u) ? (byte >> 4) : (byte & 15u);
        my_len[r] = l;
        if (l > HUF_MAXLEN) bad = true;
        else if (l) {
            kraft += 1u << (HUF_MAXLEN - l);
            present++;
        }
    }
    if (__any_sync(FULL, bad)) HUF_FAIL();
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
        kraft += __shfl_xor_sync(FULL, kraft, d);
        present += __shfl_xor_sync(FULL, present, d);
    }
    if (present == 0) HUF_FAIL();
    u32 cnt[HUF_MAXLEN + 2];
#pragma unroll
    for (int l = 0; l <= HUF_MAXLEN + 1; l++) cnt[l] = 0;
    /* per-length counts + the (length, symbol)-sorted symbol table by counting sort */
    u32 base_l = 0;
    for (u32 l = 1; l <= HUF_MAXLEN; l++) {
        u32 c_l = 0;
#pragma unroll
        for (int r = 0; r < 8; r++) {
            const u32 m = __ballot_sync(FULL, my_len[r] == l);
            if (my_len[r] == l) W->sorted[base_l + c_l + __popc(m & ((1u << lane) - 1u))] = (u8)(32 * r + lane);
            c_l += __popc(m);
        }
        cnt[l] = c_l;
        base_l += c_l;
    }
    const bool single = (present == 1 && cnt[1] == 1 && kraft == (1u << (HUF_MAXLEN - 1)));
    if (kraft != (1u << HUF_MAXLEN) && !single) HUF_FAIL();
    __syncwarp();
    if (single) {
        /* one symbol of length 1: the root's bitmap must route every symbol left */
        const u32 bytes = (n + 7) >> 3;
        if (bytes > rsz) HUF_FAIL();
        u32 nz = 0;
        for (u32 k = lane; k < bytes; k += 32) {
            u32 b = runs[k];
            if (k == bytes - 1 && (n & 7u)) b &= (1u << (n & 7u)) - 1u;
            nz |= b;
        }
        if (__any_sync(FULL, nz != 0)) HUF_FAIL();
        ZXC_STAT(32, 1);
        const u8 sym = W->sorted[0];
        for (u32 k = lane; k < n; k += 32) out[k] = sym;
        return ZXC_OK;
    }

    /* ---- level geometry ---- */
    u32 first[HUF_MAXLEN + 2], lbase[HUF_MAXLEN + 2], leafb[HUF_MAXLEN + 2];
    {
        u32 code = 0, nodes = 0, leaves = 0;
        first[0] = 0;
        lbase[0] = 0;
        leafb[0] = 0;
        nodes = 1;
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
        if (nodes > HUF_MAXNODES) HUF_FAIL();
    }
    if (lane <= HUF_MAXLEN + 1) {
        W->first[lane] = first[lane];
        W->cnt[lane] = cnt[lane];
        W->level_base[lane] = lbase[lane];
        W->leaf_base[lane] = leafb[lane];
    }

    /* ---- node kinds, level by level (parents before children): flat roots and coverage ---- */
    if (lane == 0) W->kind[0] = HUF_KIND_BITMAP; /* root: provisional, fixed below */
    __syncwarp();
    for (u32 l = 0; l <= HUF_MAXLEN; l++) {
        const u32 nn = (l == 0) ? 1u : (1u << l) - first[l];
        for (u32 t = lane; t < nn; t += 32) {
            const u32 v = first[l] + t;
            const u32 id = lbase[l] + t;
            u32 kind;
            bool covered = false;
            if (l > 0) {
                const u32 pk = W->kind[lbase[l - 1] + (v >> 1) - first[l - 1]];
                covered = (pk >= 2 && pk <= HUF_MAXLEN) || pk == HUF_KIND_COVERED;
            }
            const bool leaf = (l > 0) && (v < first[l] + cnt[l]);
            if (covered) kind = HUF_KIND_COVERED;
            else if (leaf) kind = HUF_KIND_LEAF;
            else {
                /* perfect subtree of depth D: all of [v<<d, (v+1)<<d) internal for d < D, all leaves at D */
                kind = HUF_KIND_BITMAP;
                for (u32 D = 1; l + D <= HUF_MAXLEN; D++) {
                    const u32 lo = v << D, hi = (v + 1) << D, ld = l + D;
                    const u32 leaf_end = first[ld] + cnt[ld];
                    if (hi <= leaf_end) { /* every descendant at this depth is a leaf */
                        if (D >= 2) kind = D;
                        break;
                    }
                    if (lo < leaf_end) break; /* mixed depth: not flat */
                }
            }
            W->kind[id] = (u8)kind;
        }
        __syncwarp();
    }

    /* ---- counts, run offsets, rank tables: one emitting node at a time in BFS order ---- */
    if (lane == 0) W->count[0] = n;
    __syncwarp();
    u32 roff = 0, coff = 0;
    const u32 total_nodes = lbase[HUF_MAXLEN + 1];
    u32 l = 0;
    for (u32 id = 0; id < total_nodes; id++) {
        while (id >= lbase[l + 1]) l++;
        const u32 kind = W->kind[id];
        if (kind == HUF_KIND_LEAF || kind == HUF_KIND_COVERED) continue;
        const u32 c = W->count[id];
        const u32 v = first[l] + (id - lbase[l]);
        if (kind >= 2) { /* flat root: c paths of `kind` bits */
            const u32 bytes = (c * kind + 7) >> 3;
            if (bytes > rsz - roff) HUF_FAIL();
            if (lane == 0) W->runoff[id] = roff;
            roff += bytes;
            continue;
        }
        const u32 bytes = (c + 7) >> 3;
        if (bytes > rsz - roff) HUF_FAIL();
        const u8* run = runs + roff;
        const u32 words = (c + 31) >> 5;
        if (words > cum_words - coff) HUF_FAIL();
        ZXC_STAT(34, words);
        u32 ones = 0;
        for (u32 w0 = 0; w0 < words; w0 += 32) {
            const u32 wi = w0 + lane;
            u32 pc = 0;
            if (wi < words) {
                u32 bits = 0;
                const u32 b0 = 4u * wi;
                for (u32 q = 0; q < 4 && b0 + q < bytes; q++) bits |= (u32)run[b0 + q] << (8u * q);
                if (wi == words - 1 && (c & 31u)) bits &= (1u << (c & 31u)) - 1u;
                pc = __popc(bits);
            }
            const u32 inc = warp_incl_scan(pc, lane);
            if (wi < words) cum[coff + wi] = ones + inc - pc; /* ones before this word */
            ones += __shfl_sync(FULL, inc, 31);
        }
        if (lane == 0) {
            W->runoff[id] = roff;
            W->cumoff[id] = coff;
            /* children live at depth l+1 with values 2v, 2v+1 */
            const u32 cid = lbase[l + 1] + (2u * v - first[l + 1]);
            W->count[cid] = c - ones;
            W->count[cid + 1] = ones;
        }
        roff += bytes;
        coff += words;
        __syncwarp();
    }

    __syncwarp();
    /* ---- every output symbol walks down from the root ---- */
    for (u32 k0 = 0; k0 < n; k0 += 32) {
        const u32 k = k0 + lane;
        u32 flat_seen = 0, steps = 0; /* emulator counters only */
        if (k < n) {
            u32 lv = 0, v = 0, idx = k;
            for (;;) {
                const u32 id = lbase[lv] + (v - first[lv]);
                const u32 kind = W->kind[id];
                if (kind == HUF_KIND_LEAF) break;
                const u32 ro = W->runoff[id];
                if (kind >= 2) {
                    const u32 bp = idx * kind, b = ro + (bp >> 3);
                    u32 bits = huf_byte(runs, rsz, b) | (huf_byte(runs, rsz, b + 1) << 8) | (huf_byte(runs, rsz, b + 2) << 16);
                    bits >>= (bp & 7u);
                    for (u32 j = 0; j < kind; j++) v = (v << 1) | ((bits >> j) & 1u);
                    lv += kind;
                    flat_seen |= 1u << kind;
                    break;
                }
                steps++;
                const u32 word = huf_bits32(runs, rsz, ro + 4u * (idx >> 5));
                const u32 bit = (word >> (idx & 31u)) & 1u;
                const u32 before = cum[W->cumoff[id] + (idx >> 5)] + __popc(word & ((1u << (idx & 31u)) - 1u));
                idx = bit ? before : idx - before;
                v = (v << 1) | bit;
                lv++;
            }
            out[k] = W->sorted[leafb[lv] + (v - first[lv])];
        }
        ZXC_STAT(33, __popc(__ballot_sync(FULL, steps != 0)));
#pragma unroll
        for (u32 D = 2; D <= HUF_MAXLEN; D++) ZXC_STAT(40 + D, __popc(__ballot_sync(FULL, (flat_seen >> D) & 1u)));
        (void)flat_seen;
        (void)steps;
    }
    return ZXC_OK;
}
