/*
 * zxc_oracle.c -- TEST INFRASTRUCTURE ONLY (see zxc_oracle.h).
 *
 * Scalar restatement of the ZXC wire format v8 decoder.  Byte-serial on
 * purpose: it is the executable form of docs/FORMAT.md sections 3-8 and of the
 * semantics of src/lib/zxc_decompress.c, written without any of the
 * reference's wild-copy / SIMD machinery.  Each function cites what it follows.
 */
#include "zxc_oracle.h"

#include <stdlib.h>
#include <string.h>

/* ---- wire constants (src/lib/zxc_internal.h:331-547, include/zxc_constants.h) ---- */
#define MAGIC 0x9CB02EF5u
#define VERSION 8
#define FILE_HDR 16
#define FILE_FTR 12
#define BLK_HDR 8
#define BLK_CKS 4
#define SUB_HDR 12
#define LIT_SLACK 32
#define TAIL_PAD 2112 /* ZXC_DECOMPRESS_TAIL_PAD = 32*66 */
#define MIN_MATCH 5
#define BT_RAW 0
#define BT_GLO 1
#define BT_GHI 2
#define BT_SEK 254
#define BT_EOF 255
#define FLAG_CKS 0x80u
#define FLAG_DICT 0x40u

static uint32_t le16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
static uint32_t le32(const uint8_t* p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
static uint64_t le64(const uint8_t* p) { return (uint64_t)le32(p) | ((uint64_t)le32(p + 4) << 32); }

/* ------------------------------------------------------------------------- */
/* header hashes: xorshift of the LE words (zxc_internal.h:1188-1214)        */
/* ------------------------------------------------------------------------- */
static uint64_t xs64(uint64_t h) {
    h ^= h << 13;
    h ^= h >> 7;
    h ^= h << 17;
    return h;
}

uint8_t zxo_hash8(const uint8_t* p) {
    const uint64_t h = xs64(le64(p) ^ 0x9E3779B97F4A7C15ull);
    return (uint8_t)((h >> 32) ^ h);
}

uint16_t zxo_hash16(const uint8_t* p) {
    const uint64_t h = xs64(le64(p) ^ le64(p + 8) ^ 0xD2D84A61D2D84A61ull);
    const uint32_t r = (uint32_t)((h >> 32) ^ h);
    return (uint16_t)((r >> 16) ^ r);
}

/* ------------------------------------------------------------------------- */
/* rapidhash V3 (vendored third-party algorithm, src/lib/vendors/rapidhash.h  */
/* :130-345): 7 independent 16-byte lanes per 112-byte stripe, then a <=112   */
/* byte tail of chained mixes, then a finaliser over the last 16 bytes.       */
/* ------------------------------------------------------------------------- */
static const uint64_t RS[8] = {0x2d358dccaa6c78a5ull, 0x8bb84b93962eacc9ull, 0x4b33a62ed433d4a3ull,
                               0x4d5a2da51de1aa47ull, 0xa0761d6478bd642full, 0xe7037ed1a0b428dbull,
                               0x90ed1765281c388cull, 0xaaaaaaaaaaaaaaaaull};

static void mum(uint64_t* a, uint64_t* b) {
    const __uint128_t r = (__uint128_t)(*a) * (*b);
    *a = (uint64_t)r;
    *b = (uint64_t)(r >> 64);
}
static uint64_t mix(uint64_t a, uint64_t b) {
    mum(&a, &b);
    return a ^ b;
}

uint64_t zxo_rapidhash(const void* key, size_t len, uint64_t seed) {
    const uint8_t* p = (const uint8_t*)key;
    uint64_t a = 0, b = 0;
    size_t i = len;
    seed ^= mix(seed ^ RS[2], RS[1]);
    if (len <= 16) {
        if (len >= 4) {
            seed ^= len;
            if (len >= 8) {
                a = le64(p);
                b = le64(p + len - 8);
            } else {
                a = le32(p);
                b = le32(p + len - 4);
            }
        } else if (len > 0) {
            a = ((uint64_t)p[0] << 45) | p[len - 1];
            b = p[len >> 1];
        }
    } else {
        if (len > 112) {
            uint64_t s[7];
            for (int k = 0; k < 7; k++) s[k] = seed;
            while (i > 112) {
                for (int k = 0; k < 7; k++)
                    s[k] = mix(le64(p + 16 * k) ^ RS[k], le64(p + 16 * k + 8) ^ s[k]);
                p += 112;
                i -= 112;
            }
            /* fold order: rapidhash.h:306-311 */
            s[0] ^= s[1];
            s[2] ^= s[3];
            s[4] ^= s[5];
            s[0] ^= s[6];
            s[2] ^= s[4];
            s[0] ^= s[2];
            seed = s[0];
        }
        if (i > 16) {
            static const int sec[6] = {2, 2, 1, 1, 2, 1};
            for (int k = 0; k < 6 && i > (size_t)(16 * (k + 1)); k++)
                seed = mix(le64(p + 16 * k) ^ RS[sec[k]], le64(p + 16 * k + 8) ^ seed);
        }
        a = le64(p + i - 16) ^ i;
        b = le64(p + i - 8);
    }
    a ^= RS[1];
    b ^= seed;
    mum(&a, &b);
    return mix(a ^ RS[7], b ^ RS[1] ^ i);
}

/* zxc_checksum / zxc_checksum_seed: fold to 32 bits (zxc_internal.h:1353-1378) */
uint32_t zxo_checksum(const void* p, size_t len) {
    const uint64_t h = zxo_rapidhash(p, len, 0);
    return (uint32_t)(h ^ (h >> 32));
}
uint32_t zxo_checksum_seed(const void* p, size_t len, uint32_t seed) {
    const uint64_t h = zxo_rapidhash(p, len, seed);
    return (uint32_t)(h ^ (h >> 32));
}

/* zxc_dict_id (src/lib/zxc_dict.c:35-44) */
uint32_t zxo_dict_id(const void* dict, size_t dict_size, const void* huf128) {
    if (!dict || dict_size == 0) return 0;
    const uint32_t base = zxo_checksum(dict, dict_size);
    return huf128 ? zxo_checksum_seed(huf128, 128, base) : base;
}

/* ------------------------------------------------------------------------- */
/* prefix varint (zxc_decompress.c:51-88).  Mirrors the reference exactly,    */
/* including its failure behaviour: value 0, and the cursor jams to `end`     */
/* (except when already at/after end, where it is left alone).                */
/* ------------------------------------------------------------------------- */
static uint32_t varint(const uint8_t** pp, const uint8_t* end) {
    const uint8_t* p = *pp;
    if (p >= end) return 0;
    const uint32_t b0 = p[0];
    if (b0 < 0x80) {
        *pp = p + 1;
        return b0;
    }
    if (b0 < 0xC0) {
        if (p + 1 >= end) {
            *pp = end;
            return 0;
        }
        *pp = p + 2;
        return (b0 & 0x3F) | ((uint32_t)p[1] << 6);
    }
    if (b0 < 0xE0) {
        if (p + 2 >= end) {
            *pp = end;
            return 0;
        }
        *pp = p + 3;
        return (b0 & 0x1F) | ((uint32_t)p[1] << 5) | ((uint32_t)p[2] << 13);
    }
    *pp = end;
    return 0;
}

/* ------------------------------------------------------------------------- */
/* RLE literal section (zxc_decompress.c:906-978, FORMAT.md 5.2)              */
/* ------------------------------------------------------------------------- */
static int rle_expand(const uint8_t* r, size_t rsz, uint8_t* w, size_t wsz) {
    const uint8_t* const r_end = r + rsz;
    uint8_t* const w_end = w + wsz;
    while (r < r_end && w < w_end) {
        const uint8_t t = *r++;
        if (!(t & 0x80)) {
            const uint32_t len = (uint32_t)t + 1;
            if ((size_t)(w_end - w) < len || (size_t)(r_end - r) < len) return ZXO_E_CORRUPT_DATA;
            memcpy(w, r, len);
            w += len;
            r += len;
        } else {
            const uint32_t len = (uint32_t)(t & 0x7F) + 4;
            if ((size_t)(w_end - w) < len || r >= r_end) return ZXO_E_CORRUPT_DATA;
            memset(w, *r++, len);
            w += len;
        }
    }
    return (w == w_end) ? ZXO_OK : ZXO_E_CORRUPT_DATA;
}

/* ------------------------------------------------------------------------- */
/* PivCo (level-ordered canonical Huffman) section decode.                    */
/* Follows docs/FORMAT.md:246-343 and the scalar semantics of                 */
/* src/lib/zxc_huffman.c:1042-1170 (tree + flat roots), :2271-2430 (decode),  */
/* in the top-down "rank" form: symbol k walks from the root; at a bitmap     */
/* node with local index i it takes bit i and continues in that child with    */
/* index rank(i); at a flat root it reads its D-bit path.                     */
/* ------------------------------------------------------------------------- */
#define HUF_MAX_LEN 11
#define HUF_MAX_NODES 512 /* complete binary tree over <= 256 leaves */

typedef struct {
    int left, right; /* child node ids, -1 if absent */
    int sym;         /* >= 0 for leaves */
    int depth;
    int flat_d;  /* D if this node is a flat root, else 0 */
    int covered; /* strict descendant of a flat root */
    size_t count;
    const uint8_t* run; /* this node's run on the wire */
} hnode_t;

typedef struct {
    hnode_t n[HUF_MAX_NODES];
    int n_nodes;
    int bfs[HUF_MAX_NODES];
    int single; /* single-symbol degenerate code */
} htree_t;

static int huf_subtree_uniform_depth(const htree_t* t, int id) {
    /* returns relative depth D if all leaves below id sit at the same depth, else -1 */
    const hnode_t* nd = &t->n[id];
    if (nd->sym >= 0) return 0;
    if (nd->left < 0 || nd->right < 0) return -1;
    const int a = huf_subtree_uniform_depth(t, nd->left);
    const int b = huf_subtree_uniform_depth(t, nd->right);
    if (a < 0 || b < 0 || a != b) return -1;
    return a + 1;
}

static void huf_mark_covered(htree_t* t, int id) {
    hnode_t* nd = &t->n[id];
    if (nd->left >= 0) {
        t->n[nd->left].covered = 1;
        huf_mark_covered(t, nd->left);
    }
    if (nd->right >= 0) {
        t->n[nd->right].covered = 1;
        huf_mark_covered(t, nd->right);
    }
}

static int huf_build(htree_t* t, const uint8_t* lens128) {
    uint8_t len[256];
    int cnt[HUF_MAX_LEN + 2] = {0};
    int present = 0;
    for (int i = 0; i < 128; i++) {
        len[2 * i] = lens128[i] & 0x0F;
        len[2 * i + 1] = lens128[i] >> 4;
    }
    for (int s = 0; s < 256; s++) {
        if (len[s] > HUF_MAX_LEN) return ZXO_E_CORRUPT_DATA;
        if (len[s]) {
            cnt[len[s]]++;
            present++;
        }
    }
    if (present == 0) return ZXO_E_CORRUPT_DATA;
    uint32_t kraft = 0;
    for (int l = 1; l <= HUF_MAX_LEN; l++) kraft += (uint32_t)cnt[l] << (HUF_MAX_LEN - l);
    t->single = 0;
    if (kraft != (1u << HUF_MAX_LEN)) {
        if (present == 1 && cnt[1] == 1 && kraft == (1u << (HUF_MAX_LEN - 1)))
            t->single = 1;
        else
            return ZXO_E_CORRUPT_DATA;
    }
    /* canonical codes */
    uint32_t next[HUF_MAX_LEN + 2] = {0};
    uint32_t code = 0;
    for (int l = 1; l <= HUF_MAX_LEN; l++) {
        code = (code + (uint32_t)cnt[l - 1]) << 1;
        next[l] = code;
    }
    memset(t->n, 0, sizeof(t->n));
    t->n_nodes = 1;
    t->n[0].left = t->n[0].right = -1;
    t->n[0].sym = -1;
    for (int l = 1; l <= HUF_MAX_LEN; l++) {
        for (int s = 0; s < 256; s++) {
            if (len[s] != l) continue;
            const uint32_t c = next[l]++;
            int cur = 0;
            for (int d = 0; d < l; d++) {
                const int bit = (c >> (l - 1 - d)) & 1;
                int* child = bit ? &t->n[cur].right : &t->n[cur].left;
                if (*child < 0) {
                    if (t->n_nodes >= HUF_MAX_NODES) return ZXO_E_CORRUPT_DATA;
                    const int id = t->n_nodes++;
                    t->n[id].left = t->n[id].right = -1;
                    t->n[id].sym = -1;
                    t->n[id].depth = d + 1;
                    *child = id;
                }
                cur = *child;
            }
            t->n[cur].sym = s;
        }
    }
    /* BFS order + flat-root classification (parents first) */
    int head = 0, tail = 0;
    t->bfs[tail++] = 0;
    while (head < tail) {
        const int id = t->bfs[head++];
        hnode_t* nd = &t->n[id];
        if (nd->sym < 0 && !nd->covered) {
            const int D = huf_subtree_uniform_depth(t, id);
            if (D >= 2) {
                nd->flat_d = D;
                huf_mark_covered(t, id);
            }
        }
        if (nd->left >= 0) t->bfs[tail++] = nd->left;
        if (nd->right >= 0) t->bfs[tail++] = nd->right;
    }
    return ZXO_OK;
}

static size_t popcount_prefix(const uint8_t* bits, size_t nbits) {
    size_t c = 0;
    size_t full = nbits >> 3;
    for (size_t i = 0; i < full; i++) c += (size_t)__builtin_popcount(bits[i]);
    const unsigned rem = (unsigned)(nbits & 7);
    if (rem) c += (size_t)__builtin_popcount(bits[full] & ((1u << rem) - 1));
    return c;
}

/* payload excludes the 128-byte lengths header */
static int huf_decode_runs(htree_t* t, const uint8_t* payload, size_t psize, uint8_t* out, size_t n) {
    if (n == 0) return ZXO_E_CORRUPT_DATA; /* zxc_pivco_decode_core rejects an empty section (zxc_huffman.c:2276) */
    /* pass 1: walk the BFS order, assign runs and counts (zxc_huffman.c:2297-2328) */
    const uint8_t* p = payload;
    const uint8_t* const pend = payload + psize;
    for (int i = 0; i < t->n_nodes; i++) {
        t->n[i].count = 0;
        t->n[i].run = NULL;
    }
    t->n[0].count = n;
    if (t->single) {
        /* one symbol of length 1: the root is a bitmap node with a single (left) child */
    }
    for (int qi = 0; qi < t->n_nodes; qi++) {
        hnode_t* nd = &t->n[t->bfs[qi]];
        if (nd->sym >= 0 || nd->covered) continue;
        const size_t c = nd->count;
        if (nd->flat_d) {
            const size_t bytes = (c * (size_t)nd->flat_d + 7) >> 3;
            if ((size_t)(pend - p) < bytes) return ZXO_E_CORRUPT_DATA;
            nd->run = p;
            p += bytes;
        } else {
            const size_t bytes = (c + 7) >> 3;
            if ((size_t)(pend - p) < bytes) return ZXO_E_CORRUPT_DATA;
            nd->run = p;
            p += bytes;
            const size_t ones = popcount_prefix(nd->run, c);
            if (ones > c) return ZXO_E_CORRUPT_DATA;
            const size_t zeros = c - ones;
            if (nd->right >= 0)
                t->n[nd->right].count = ones;
            else if (ones)
                return ZXO_E_CORRUPT_DATA;
            if (nd->left >= 0)
                t->n[nd->left].count = zeros;
            else if (zeros)
                return ZXO_E_CORRUPT_DATA;
        }
    }
    /* pass 2: per-symbol top-down walk; a node's run is read in order by the symbols that pass through it, so the
     * index of a symbol at a node is the number that passed before it */
    size_t* seen = (size_t*)calloc((size_t)t->n_nodes, sizeof(size_t));
    if (!seen) return ZXO_E_MEMORY;
    for (size_t k = 0; k < n; k++) {
        int id = 0;
        for (;;) {
            const hnode_t* nd = &t->n[id];
            if (nd->sym >= 0) {
                out[k] = (uint8_t)nd->sym;
                break;
            }
            const size_t idx = seen[id]++;
            if (nd->flat_d) {
                const size_t bitpos = idx * (size_t)nd->flat_d;
                int cur = id;
                for (int j = 0; j < nd->flat_d; j++) {
                    const size_t bp = bitpos + (size_t)j;
                    const int bit = (nd->run[bp >> 3] >> (bp & 7)) & 1;
                    cur = bit ? t->n[cur].right : t->n[cur].left;
                }
                out[k] = (uint8_t)t->n[cur].sym;
                break;
            }
            const int bit = (nd->run[idx >> 3] >> (idx & 7)) & 1;
            id = bit ? nd->right : nd->left;
            if (id < 0) {
                free(seen);
                return ZXO_E_CORRUPT_DATA;
            }
        }
    }
    free(seen);
    return ZXO_OK;
}

/* section = [128-byte lengths][runs] when lens128 == NULL, else [runs] with external lengths */
static int huf_decode_section(const uint8_t* sec, size_t ssz, const uint8_t* lens128, uint8_t* out,
                              size_t n) {
    htree_t* t = (htree_t*)malloc(sizeof(htree_t));
    if (!t) return ZXO_E_MEMORY;
    int rc;
    if (!lens128) {
        if (ssz < 128) {
            free(t);
            return ZXO_E_CORRUPT_DATA;
        }
        lens128 = sec;
        sec += 128;
        ssz -= 128;
    }
    rc = huf_build(t, lens128);
    if (rc == ZXO_OK) rc = huf_decode_runs(t, sec, ssz, out, n);
    free(t);
    return rc;
}

/* ------------------------------------------------------------------------- */
/* LZ sequence execution shared by GLO and GHI (SURVEY Appendix A;            */
/* zxc_decompress.c:1168-1208 "safe path" is the byte-exact semantics, the    */
/* unrolled loops before it are an optimisation of the same thing).           */
/* ------------------------------------------------------------------------- */
typedef struct {
    uint8_t* dst;
    size_t cap;
    size_t o; /* output cursor */
    const uint8_t* lit;
    size_t n_lit;
    size_t l; /* literal cursor */
    const uint8_t* dict;
    size_t dict_size;
} lz_t;

static int lz_emit(lz_t* z, uint64_t ll, uint64_t ml, uint32_t off) {
    if (ll + ml > (uint64_t)(z->cap - z->o) || ll > (uint64_t)(z->n_lit - z->l)) return ZXO_E_OVERFLOW;
    memcpy(z->dst + z->o, z->lit + z->l, (size_t)ll);
    z->o += (size_t)ll;
    z->l += (size_t)ll;
    if ((uint64_t)z->o + z->dict_size < off) return ZXO_E_BAD_OFFSET;
    for (uint64_t k = 0; k < ml; k++) {
        const size_t pos = z->o + (size_t)k;
        uint8_t v;
        if (pos >= off)
            v = z->dst[pos - off];
        else
            v = z->dict[z->dict_size - (off - pos)];
        z->dst[pos] = v;
    }
    z->o += (size_t)ml;
    return ZXO_OK;
}

static int lz_finish(lz_t* z) {
    const size_t rem = z->n_lit - z->l;
    if (rem > z->cap - z->o) return ZXO_E_OVERFLOW;
    memcpy(z->dst + z->o, z->lit + z->l, rem);
    z->o += rem;
    return (int)z->o;
}

/* GLO payload (zxc_decompress.c:847-1209, zxc_common.c:773-795) */
/* block_size: the frame's block size, the reference's chunk_size; its token buffer holds block_size / 5 + 16 sequences
 * (zxc_common.c:142-156, zxc_decompress.c:801) */
static int decode_glo(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, const uint8_t* dict,
                      size_t dict_size, const uint8_t* dict_huf, size_t block_size) {
    if (n < SUB_HDR) return ZXO_E_BAD_HEADER;
    const uint32_t n_seq = le32(src), n_lit = le32(src + 4);
    const uint8_t enc_lit = src[8], enc_tok = src[9], enc_off = src[11];
    const size_t desc = (enc_lit != 0 ? 4u : 0u) + (enc_tok == 2 ? 4u : 0u);
    if (n < SUB_HDR + desc) return ZXO_E_BAD_HEADER;
    const uint8_t* dp = src + SUB_HDR;
    uint32_t lit_comp = n_lit, tok_comp = n_seq;
    if (enc_lit != 0) {
        lit_comp = le32(dp);
        dp += 4;
    }
    if (enc_tok == 2) tok_comp = le32(dp);
    if (enc_off > 1) return ZXO_E_CORRUPT_DATA; /* :863 */

    const uint8_t* const p_data = src + SUB_HDR + desc;
    const size_t avail = n - SUB_HDR - desc;
    uint8_t* lit_buf = NULL;
    uint8_t* tok_buf = NULL;
    const uint8_t* lit;
    int rc = ZXO_OK;

    if (enc_lit == 2 || enc_lit == 3) { /* :888-905 */
        if (lit_comp > avail) return ZXO_E_CORRUPT_DATA;
        if (n_lit == 0) {
            lit = p_data;
        } else {
            if (n_lit > cap) return ZXO_E_DST_TOO_SMALL;
            if (enc_lit == 3 && !dict_huf) return ZXO_E_DICT_REQUIRED;
            if (n_lit > block_size) return ZXO_E_CORRUPT_DATA; /* lit_buffer_cap (:774) */
            lit_buf = (uint8_t*)malloc((size_t)n_lit + 1);
            if (!lit_buf) return ZXO_E_MEMORY;
            rc = huf_decode_section(p_data, lit_comp, enc_lit == 3 ? dict_huf : NULL, lit_buf, n_lit);
            if (rc != ZXO_OK) goto done;
            lit = lit_buf;
        }
    } else if (enc_lit == 1) { /* :906-978 */
        if (n_lit > 0) {
            if (n_lit > cap) return ZXO_E_DST_TOO_SMALL;
            if (n_lit > block_size) return ZXO_E_CORRUPT_DATA; /* lit_buffer_cap (:914) */
            if (lit_comp > avail) return ZXO_E_CORRUPT_DATA;
            lit_buf = (uint8_t*)malloc((size_t)n_lit + 1);
            if (!lit_buf) return ZXO_E_MEMORY;
            rc = rle_expand(p_data, lit_comp, lit_buf, n_lit);
            if (rc != ZXO_OK) goto done;
            lit = lit_buf;
        } else {
            lit = p_data;
        }
    } else if (enc_lit == 0) {
        lit = p_data;
    } else {
        return ZXO_E_CORRUPT_DATA; /* :983 */
    }

    {
        const uint64_t sz_off = enc_off ? (uint64_t)n_seq : (uint64_t)n_seq * 2;
        const uint64_t consumed = (uint64_t)lit_comp + tok_comp + sz_off;
        if (consumed > avail) { /* :996 */
            rc = ZXO_E_CORRUPT_DATA;
            goto done;
        }
        if (avail - lit_comp < LIT_SLACK) { /* :1003 */
            rc = ZXO_E_CORRUPT_DATA;
            goto done;
        }
        const uint8_t* tok = p_data + lit_comp;
        const uint8_t* offs = tok + tok_comp;
        const uint8_t* ext = offs + sz_off;
        const uint8_t* const ext_end = p_data + avail;
        if (enc_tok == 2) { /* :1019-1022 */
            if ((size_t)n_seq > block_size / MIN_MATCH + 16) {
                rc = ZXO_E_CORRUPT_DATA;
                goto done;
            }
            tok_buf = (uint8_t*)malloc((size_t)n_seq + 1);
            if (!tok_buf) {
                rc = ZXO_E_MEMORY;
                goto done;
            }
            rc = huf_decode_section(tok, tok_comp, NULL, tok_buf, n_seq);
            if (rc != ZXO_OK) goto done;
            tok = tok_buf;
        } else if (enc_tok != 0) {
            rc = ZXO_E_CORRUPT_DATA; /* :1016 */
            goto done;
        }
        /* a RAW literal section longer than the payload cannot occur: lit_comp <= consumed <= avail */
        lz_t z = {dst, cap, 0, lit, (enc_lit == 0) ? lit_comp : n_lit, 0, dict, dict_size};
        for (uint32_t i = 0; i < n_seq; i++) {
            uint64_t ll = tok[i] >> 4, ml = tok[i] & 15;
            const uint32_t off = (enc_off ? offs[i] : le16(offs + 2 * (size_t)i)) + 1;
            if (ll == 15) ll += varint(&ext, ext_end);
            if (ml == 15) ml += varint(&ext, ext_end);
            ml += MIN_MATCH;
            rc = lz_emit(&z, ll, ml, off);
            if (rc != ZXO_OK) goto done;
        }
        rc = lz_finish(&z);
    }
done:
    free(lit_buf);
    free(tok_buf);
    return rc;
}

/* GHI payload (zxc_decompress.c:1231-1469) */
static int decode_ghi(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, const uint8_t* dict,
                      size_t dict_size) {
    if (n < SUB_HDR) return ZXO_E_BAD_HEADER;
    const uint32_t n_seq = le32(src), n_lit = le32(src + 4);
    if (src[8] != 0 || src[9] != 0) return ZXO_E_CORRUPT_DATA; /* :1242 */
    const size_t avail = n - SUB_HDR;
    const uint64_t consumed = (uint64_t)n_lit + (uint64_t)n_seq * 4;
    if (consumed > avail) return ZXO_E_CORRUPT_DATA;       /* :1256 */
    if (avail - n_lit < LIT_SLACK) return ZXO_E_CORRUPT_DATA; /* :1261 */
    const uint8_t* lit = src + SUB_HDR;
    const uint8_t* seq = lit + n_lit;
    const uint8_t* ext = seq + (size_t)n_seq * 4;
    const uint8_t* const ext_end = src + n;
    lz_t z = {dst, cap, 0, lit, n_lit, 0, dict, dict_size};
    for (uint32_t i = 0; i < n_seq; i++) {
        const uint32_t w = le32(seq + 4 * (size_t)i);
        uint64_t ll = w >> 24, ml = (w >> 16) & 0xFF;
        const uint32_t off = (w & 0xFFFF) + 1;
        if (ll == 255) ll += varint(&ext, ext_end);
        if (ml == 255) ml += varint(&ext, ext_end);
        ml += MIN_MATCH;
        const int rc = lz_emit(&z, ll, ml, off);
        if (rc != ZXO_OK) return rc;
    }
    return lz_finish(&z);
}

/* zxc_decompress_chunk_wrapper_body (zxc_decompress.c:1646-1695) */
int zxo_decode_block_bs(const uint8_t* blk, size_t blk_size, uint8_t* dst, size_t dst_cap,
                        const uint8_t* dict, size_t dict_size, const uint8_t* dict_huf,
                        int verify_checksum, size_t block_size) {
    if (blk_size < BLK_HDR) return ZXO_E_SRC_TOO_SMALL;
    const uint8_t type = blk[0];
    const uint32_t comp = le32(blk + 3);
    const size_t need = (size_t)BLK_HDR + comp + (verify_checksum ? BLK_CKS : 0);
    if (blk_size < need) return ZXO_E_SRC_TOO_SMALL;
    const uint8_t* data = blk + BLK_HDR;
    if (verify_checksum && le32(data + comp) != zxo_checksum(data, comp)) return ZXO_E_BAD_CHECKSUM;
    switch (type) {
        case BT_GLO:
            return decode_glo(data, comp, dst, dst_cap, dict, dict_size, dict_huf, block_size);
        case BT_GHI:
            return decode_ghi(data, comp, dst, dst_cap, dict, dict_size);
        case BT_RAW:
            if (comp > dst_cap) return ZXO_E_DST_TOO_SMALL;
            memcpy(dst, data, comp);
            return (int)comp;
        case BT_EOF:
            return ZXO_E_CORRUPT_DATA;
        default:
            return ZXO_E_BAD_BLOCK_TYPE;
    }
}

/* the block API (zxc_decompress_block, zxc_dispatch.c:1742): the block size is dst_cap rounded up to a power of two,
 * at least the smallest block size */
int zxo_decode_block(const uint8_t* blk, size_t blk_size, uint8_t* dst, size_t dst_cap,
                     const uint8_t* dict, size_t dict_size, const uint8_t* dict_huf,
                     int verify_checksum) {
    size_t bs = (size_t)1 << 12;
    while (bs < dst_cap) bs <<= 1;
    return zxo_decode_block_bs(blk, blk_size, dst, dst_cap, dict, dict_size, dict_huf, verify_checksum, bs);
}

/* zxc_read_file_header (zxc_common.c:574-603) */
static int read_file_header(const uint8_t* src, size_t n, size_t* bs, int* has_cks, uint32_t* did) {
    if (n < FILE_HDR) return ZXO_E_SRC_TOO_SMALL;
    if (le32(src) != MAGIC) return ZXO_E_BAD_MAGIC;
    if (src[4] != VERSION) return ZXO_E_BAD_VERSION;
    uint8_t tmp[FILE_HDR];
    memcpy(tmp, src, FILE_HDR);
    tmp[14] = tmp[15] = 0;
    if (le16(src + 14) != zxo_hash16(tmp) || (src[6] & 0x0F) != 0) return ZXO_E_BAD_HEADER;
    if (src[5] < 12 || src[5] > 21) return ZXO_E_BAD_BLOCK_SIZE;
    *bs = (size_t)1 << src[5];
    *has_cks = (src[6] & FLAG_CKS) ? 1 : 0;
    *did = (src[6] & FLAG_DICT) ? le32(src + 7) : 0;
    return ZXO_OK;
}

static int block_header_ok(const uint8_t* p) {
    uint8_t tmp[BLK_HDR];
    memcpy(tmp, p, BLK_HDR);
    tmp[7] = 0;
    return p[7] == zxo_hash8(tmp);
}

/* zxc_decompress + zxc_decompress_frame (zxc_dispatch.c:842-1005) */
int64_t zxo_decompress(const uint8_t* src, size_t src_size, uint8_t* dst, size_t dst_cap,
                       int checksum_enabled, const uint8_t* dict, size_t dict_size,
                       const uint8_t* dict_huf) {
    if (!src || (!dst && dst_cap != 0)) return ZXO_E_NULL_INPUT;
    if (src_size < FILE_HDR + FILE_FTR) return ZXO_E_SRC_TOO_SMALL;
    if (!dst || dst_cap == 0) {
        if (le32(src) != MAGIC) return ZXO_E_BAD_MAGIC;
        return le64(src + src_size - FILE_FTR) == 0 ? 0 : ZXO_E_DST_TOO_SMALL;
    }
    size_t bs = 0;
    int file_cks = 0;
    uint32_t did = 0;
    const int hrc = read_file_header(src, src_size, &bs, &file_cks, &did);
    if (hrc != ZXO_OK) return hrc;
    if (!dict) dict_size = 0;
    if (did != 0) {
        if (!dict || dict_size == 0) return ZXO_E_DICT_REQUIRED;
        if (zxo_dict_id(dict, dict_size, dict_huf) != did) return ZXO_E_DICT_MISMATCH;
    }
    if (dict_size && dict_huf) { /* zxc_cctx_attach_dict_huf (zxc_common.c:490-512) */
        int any = 0;
        for (int i = 0; i < 128; i++) any |= dict_huf[i];
        if (!any) {
            dict_huf = NULL; /* an all-zero table is no table */
        } else {
            htree_t* t = (htree_t*)malloc(sizeof(htree_t));
            if (!t) return ZXO_E_MEMORY;
            const int brc = huf_build(t, dict_huf);
            free(t);
            if (brc != ZXO_OK) return ZXO_E_CORRUPT_DATA;
        }
    }
    const int verify = file_cks && checksum_enabled;
    const size_t work_sz = bs + TAIL_PAD;
    uint8_t* work = (uint8_t*)malloc(work_sz);
    if (!work) return ZXO_E_MEMORY;
    const uint8_t* ip = src + FILE_HDR;
    const uint8_t* const ip_end = src + src_size;
    size_t op = 0;
    uint32_t ghash = 0;
    int64_t ret = 0;
    for (;;) {
        if (ip >= ip_end) {
            ret = (int64_t)op; /* ran off the end without EOF: the loop simply ends (:912) */
            break;
        }
        const size_t rem = (size_t)(ip_end - ip);
        if (rem < BLK_HDR || !block_header_ok(ip)) {
            ret = ZXO_E_BAD_HEADER;
            break;
        }
        const uint8_t type = ip[0];
        const uint32_t comp = le32(ip + 3);
        if (type == BT_EOF) {
            if (comp != 0) {
                ret = ZXO_E_BAD_HEADER;
                break;
            }
            const uint8_t* f = src + src_size - FILE_FTR;
            if (le64(f) != (uint64_t)op) {
                ret = ZXO_E_CORRUPT_DATA;
                break;
            }
            if (verify && le32(f + 8) != ghash) {
                ret = ZXO_E_BAD_CHECKSUM;
                break;
            }
            ret = (int64_t)op;
            break;
        }
        const int res = zxo_decode_block_bs(ip, rem, work, work_sz, dict, dict_size, dict_huf, verify, bs);
        if (res < 0) {
            ret = res;
            break;
        }
        if ((size_t)res > dst_cap - op) {
            ret = ZXO_E_DST_TOO_SMALL;
            break;
        }
        memcpy(dst + op, work, (size_t)res);
        if (verify) {
            const uint32_t bh = le32(ip + BLK_HDR + comp);
            ghash = ((ghash << 1) | (ghash >> 31)) ^ bh;
        }
        ip += (size_t)BLK_HDR + comp + (file_cks ? BLK_CKS : 0);
        op += (size_t)res;
    }
    free(work);
    return ret;
}

/* zxc_seekable_parse (zxc_seekable.c:270-396) */
int64_t zxo_seek_parse(const uint8_t* src, size_t n, uint32_t* block_size, uint64_t* total,
                       uint32_t* comp_sizes, size_t cap) {
    if (n < FILE_HDR + BLK_HDR + BLK_HDR + FILE_FTR) return ZXO_E_SRC_TOO_SMALL;
    size_t bs = 0;
    int cks = 0;
    uint32_t did = 0;
    const int hrc = read_file_header(src, n, &bs, &cks, &did);
    if (hrc != ZXO_OK) return hrc;
    const uint64_t tot = le64(src + n - FILE_FTR);
    if (tot == 0) return ZXO_E_CORRUPT_DATA;
    const uint64_t nb = (tot + bs - 1) / bs;
    if (nb > 0xFFFFFFFFull) return ZXO_E_CORRUPT_DATA;
    const uint64_t sek_total = BLK_HDR + nb * 4;
    if (sek_total + FILE_FTR > n) return ZXO_E_CORRUPT_DATA;
    const uint8_t* sek = src + n - FILE_FTR - sek_total;
    if (!block_header_ok(sek) || sek[0] != BT_SEK || le32(sek + 3) != (uint32_t)(nb * 4))
        return ZXO_E_CORRUPT_DATA;
    uint64_t acc = FILE_HDR;
    for (uint64_t i = 0; i < nb; i++) {
        const uint32_t c = le32(sek + BLK_HDR + 4 * i);
        if (c < BLK_HDR || c > n) return ZXO_E_CORRUPT_DATA;
        acc += c;
        if (acc > n) return ZXO_E_CORRUPT_DATA;
        if (comp_sizes && i < cap) comp_sizes[i] = c;
    }
    if (acc != (uint64_t)(sek - src) - BLK_HDR) return ZXO_E_CORRUPT_DATA;
    if (!block_header_ok(src + acc) || src[acc] != BT_EOF) return ZXO_E_CORRUPT_DATA;
    *block_size = (uint32_t)bs;
    *total = tot;
    return (int64_t)nb;
}

/* sequence statistics over a frame (not a reference function; kernel-sizing aid) */
int zxo_frame_stats(const uint8_t* src, size_t n, zxo_stats_t* st) {
    memset(st, 0, sizeof(*st));
    size_t bs = 0;
    int cks = 0;
    uint32_t did = 0;
    const int hrc = read_file_header(src, n, &bs, &cks, &did);
    if (hrc != ZXO_OK) return hrc;
    const uint8_t* ip = src + FILE_HDR;
    const uint8_t* const end = src + n;
    while (ip + BLK_HDR <= end) {
        if (!block_header_ok(ip)) return ZXO_E_BAD_HEADER;
        const uint8_t type = ip[0];
        const uint32_t comp = le32(ip + 3);
        if (type == BT_EOF) break;
        const uint8_t* d = ip + BLK_HDR;
        st->blocks++;
        st->comp_bytes += (uint64_t)BLK_HDR + comp + (cks ? BLK_CKS : 0);
        if (type == BT_RAW) {
            st->raw_blocks++;
            st->decoded_bytes += comp;
        } else if ((type == BT_GLO || type == BT_GHI) && comp >= SUB_HDR) {
            const uint32_t n_seq = le32(d), n_lit = le32(d + 4);
            const uint8_t enc_lit = d[8], enc_tok = d[9], enc_off = d[11];
            st->sequences += n_seq;
            st->literals += n_lit;
            if (n_seq > st->max_seq_per_block) st->max_seq_per_block = n_seq;
            uint64_t out = n_lit;
            if (type == BT_GLO) {
                st->glo_blocks++;
                if (enc_lit == 1) st->rle_blocks++;
                if (enc_lit >= 2) st->huf_blocks++;
                if (enc_off) st->off8_blocks++;
                const size_t desc = (enc_lit ? 4u : 0u) + (enc_tok == 2 ? 4u : 0u);
                const uint32_t lit_comp = enc_lit ? le32(d + SUB_HDR) : n_lit;
                if (enc_tok == 0) {
                    const uint8_t* tok = d + SUB_HDR + desc + lit_comp;
                    const uint8_t* offs = tok + n_seq;
                    const uint8_t* ext = offs + (size_t)n_seq * (enc_off ? 1 : 2);
                    const uint8_t* ext0 = ext;
                    const uint8_t* ext_end = d + comp;
                    for (uint32_t i = 0; i < n_seq; i++) {
                        uint64_t ll = tok[i] >> 4, ml = tok[i] & 15;
                        const uint32_t off = (enc_off ? offs[i] : le16(offs + 2 * (size_t)i)) + 1;
                        if (ll == 15) {
                            ll += varint(&ext, ext_end);
                            st->ll_escapes++;
                        }
                        if (ml == 15) {
                            ml += varint(&ext, ext_end);
                            st->ml_escapes++;
                        }
                        ml += MIN_MATCH;
                        if (off < 32) st->off_lt32++;
                        if (off < ml) st->off_lt_ml++;
                        st->ml_sum += ml;
                        out += ml;
                    }
                    st->extras_bytes += (uint64_t)(ext - ext0);
                }
            } else {
                st->ghi_blocks++;
                const uint8_t* seq = d + SUB_HDR + n_lit;
                const uint8_t* ext = seq + (size_t)n_seq * 4;
                const uint8_t* ext0 = ext;
                const uint8_t* ext_end = d + comp;
                for (uint32_t i = 0; i < n_seq; i++) {
                    const uint32_t w = le32(seq + 4 * (size_t)i);
                    uint64_t ll = w >> 24, ml = (w >> 16) & 0xFF;
                    const uint32_t off = (w & 0xFFFF) + 1;
                    if (ll == 255) {
                        ll += varint(&ext, ext_end);
                        st->ll_escapes++;
                    }
                    if (ml == 255) {
                        ml += varint(&ext, ext_end);
                        st->ml_escapes++;
                    }
                    ml += MIN_MATCH;
                    if (off < 32) st->off_lt32++;
                    if (off < ml) st->off_lt_ml++;
                    st->ml_sum += ml;
                    out += ml;
                }
                st->extras_bytes += (uint64_t)(ext - ext0);
            }
            st->decoded_bytes += out;
        }
        ip += (size_t)BLK_HDR + comp + (cks ? BLK_CKS : 0);
    }
    return ZXO_OK;
}
