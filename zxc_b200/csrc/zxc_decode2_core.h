/*
 * zxc_decode2_core.h -- integer helpers shared by the decode kernels (zxc_decode.cuh, zxc_decode_units.cuh):
 *
 *   - the extras-section segment-map scan, which resolves every varint of a block's extras section in one
 *     warp-wide prefix scan instead of a serial walk;
 *   - the 8-byte per-sequence record of the output-centric body (zxc_decode_units.cuh), which answers "which
 *     sequence covers output position q, and where do its bytes come from":
 *
 *     w0 = (E - 1) | md << 16        E  = output position one past the sequence's last byte
 *                                    md = output position of its first match byte (literals end)
 *     w1 = (off - 1) | M << 16       off = match distance, M = sum of the match lengths before it
 *                                    (literal k of the run sits at literal-stream index q - M for
 *                                    output position q, so one delta serves the whole run)
 *
 *     Self-overlapping matches (off < ml, :197-413 in the reference) read `md - off + (k mod off)`, i.e. only
 *     bytes in front of the match.
 */
#ifndef ZXC_DECODE2_CORE_H
#define ZXC_DECODE2_CORE_H

#include <stdint.h>

#ifdef __CUDACC__
#define Z2_HD __host__ __device__ __forceinline__
#else
#define Z2_HD static inline
#endif

#define Z2_MD_INF 0x100000 /* "literals never end" for the virtual trailing-literal record */

typedef struct {
    uint32_t w0, w1;
} z2_rec_t;

typedef struct {
    int32_t E;   /* end of the sequence (exclusive) */
    int32_t md;  /* first match byte */
    int32_t off; /* match distance, >= 1 */
    int32_t M;   /* match bytes before this sequence */
} z2_seq_t;

Z2_HD z2_rec_t z2_pack(uint32_t E, uint32_t md, uint32_t off, uint32_t M) {
    z2_rec_t r;
    r.w0 = ((E - 1u) & 0xFFFFu) | (md << 16);
    r.w1 = ((off - 1u) & 0xFFFFu) | (M << 16);
    return r;
}

Z2_HD z2_seq_t z2_unpack(z2_rec_t r) {
    z2_seq_t s;
    s.E = (int32_t)(r.w0 & 0xFFFFu) + 1;
    s.md = (int32_t)(r.w0 >> 16);
    s.off = (int32_t)(r.w1 & 0xFFFFu) + 1;
    s.M = (int32_t)(r.w1 >> 16);
    return s;
}

/* k mod off for 0 <= k < 2^17, 1 <= off <= 65536 without an integer divide */
Z2_HD uint32_t z2_mod(uint32_t k, uint32_t off) {
#ifdef __CUDA_ARCH__
    uint32_t q = (uint32_t)__float2uint_rz(__fdividef((float)k, (float)off));
#else
    uint32_t q = (uint32_t)((float)k / (float)off);
#endif
    int32_t r = (int32_t)k - (int32_t)(q * off);
    if (r < 0) r += (int32_t)off;
    if (r >= (int32_t)off) r -= (int32_t)off;
    return (uint32_t)r;
}

/* ---- extras section: segment maps ----------------------------------------------------------------
 * The extras section is a chain of prefix varints (zxc_decompress.c:51-88) whose start positions
 * depend on all earlier lengths.  It is cut into segments; a map says, for each way the cursor can
 * enter a segment (0, 1 or 2 bytes past its start), how many varints start inside the segment and
 * how the cursor leaves it (0..2 bytes past the end, or 3 = jammed: invalid lead byte or a varint
 * running past the section -- the reference then returns 0 for this and every later read).  Maps
 * compose associatively, so a prefix scan over the segments gives every segment its entry phase and
 * the ordinal of its first varint.
 * Packed: count of entry s in bits [19s, 19s+17), exit of entry s in bits [57+2s, 59+2s). */
Z2_HD uint64_t z2_map_make(uint32_t c0, uint32_t e0, uint32_t c1, uint32_t e1, uint32_t c2, uint32_t e2) {
    return (uint64_t)c0 | ((uint64_t)c1 << 19) | ((uint64_t)c2 << 38) | ((uint64_t)e0 << 57) | ((uint64_t)e1 << 59) |
           ((uint64_t)e2 << 61);
}
Z2_HD uint32_t z2_map_cnt(uint64_t m, uint32_t s) { return (uint32_t)(m >> (19u * s)) & 0x1FFFFu; }
Z2_HD uint32_t z2_map_exit(uint64_t m, uint32_t s) { return (uint32_t)(m >> (57u + 2u * s)) & 3u; }
#define Z2_MAP_ID z2_map_make(0, 0, 0, 1, 0, 2)
Z2_HD uint64_t z2_map_compose(uint64_t a, uint64_t b) { /* a first, then b */
    uint32_t c[3], e[3];
    for (uint32_t s = 0; s < 3; s++) {
        const uint32_t ea = z2_map_exit(a, s);
        const uint32_t ca = z2_map_cnt(a, s);
        if (ea == 3u) {
            c[s] = ca;
            e[s] = 3u;
        } else {
            c[s] = ca + z2_map_cnt(b, ea);
            e[s] = z2_map_exit(b, ea);
        }
    }
    return z2_map_make(c[0], e[0], c[1], e[1], c[2], e[2]);
}
/* walk segment [lo, hi) of an extras section of `len` bytes from entry phase s */
Z2_HD void z2_seg_walk(const uint8_t* x, uint32_t lo, uint32_t hi, uint32_t len, uint32_t s, uint32_t* cnt,
                       uint32_t* ex) {
    uint32_t pos = lo + s, c = 0;
    int jam = 0;
    while (pos < hi) {
        const uint32_t b0 = x[pos];
        const uint32_t l = 1u + (b0 >> 7) + ((b0 & 0xC0u) == 0xC0u ? 1u : 0u);
        if (b0 >= 0xE0u || pos + l > len) {
            jam = 1;
            break;
        }
        pos += l;
        c++;
    }
    *cnt = c;
    *ex = jam ? 3u : (pos - hi);
}
Z2_HD uint64_t z2_seg_map(const uint8_t* x, uint32_t lo, uint32_t hi, uint32_t len) {
    uint32_t c0, e0, c1, e1, c2, e2;
    z2_seg_walk(x, lo, hi, len, 0, &c0, &e0);
    z2_seg_walk(x, lo, hi, len, 1, &c1, &e1);
    z2_seg_walk(x, lo, hi, len, 2, &c2, &e2);
    return z2_map_make(c0, e0, c1, e1, c2, e2);
}
/* values of the varints that start in [lo, hi) when the cursor enters at phase `ent` (not 3) */
Z2_HD void z2_seg_values(const uint8_t* x, uint32_t lo, uint32_t hi, uint32_t len, uint32_t ent, uint32_t ord,
                         uint32_t* vals) {
    uint32_t pos = lo + ent;
    while (pos < hi) {
        const uint32_t b0 = x[pos];
        const uint32_t l = 1u + (b0 >> 7) + ((b0 & 0xC0u) == 0xC0u ? 1u : 0u);
        if (b0 >= 0xE0u || pos + l > len) break;
        uint32_t v = b0;
        if (l == 2) v = (b0 & 0x3Fu) | ((uint32_t)x[pos + 1] << 6);
        else if (l == 3) v = (b0 & 0x1Fu) | ((uint32_t)x[pos + 1] << 5) | ((uint32_t)x[pos + 2] << 13);
        vals[ord++] = v;
        pos += l;
    }
}

#endif /* ZXC_DECODE2_CORE_H */
