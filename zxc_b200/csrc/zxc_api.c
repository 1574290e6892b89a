/*
 * zxc_api.c -- the reference's public C API, re-hosted on the GPU block codec.
 *
 * Host code stays C (north_star).  Every function here does argument checks in
 * the reference's order, O(blocks) header arithmetic, staging copies, and one
 * call into the CUDA shim (zxc_gpu.cu) per frame / range / block.  There is no
 * CPU codec in this library: without a usable CUDA device the codec entry
 * points return ZXC_B200_ERROR_NO_DEVICE.
 *
 * Reference code paths mirrored (file:line in /root/reference/src/lib):
 *   zxc_decompress / frame loop      zxc_dispatch.c:842-1005
 *   size / dict-id probes            zxc_dispatch.c:1203-1241
 *   dctx / cctx wrappers             zxc_dispatch.c:1260-1601
 *   block API                        zxc_dispatch.c:1627-1858
 *   seekable                         zxc_seekable.c:172-214, 270-785, 999-1174
 *   dict id / .zxd                   zxc_dict.c:35-205
 *   bounds, names                    zxc_common.c:850-1017
 */
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/types.h>
#include <unistd.h>

#include "zxc.h"
#include "zxc_b200.h"
#include "zxc_format.h"
#include "zxc_frame.h"
#include "zxc_gpu.h"
#include "zxc_hufenc.h" /* zxh_geometry: validates a dictionary's shared literal table */
#include "zxc_seekable.h"
#include "zxc_stream.h"

/* ------------------------------------------------------------------------- */
/* info, options, names, bounds                                              */
/* ------------------------------------------------------------------------- */
int zxc_min_level(void) { return ZXC_LEVEL_FASTEST; }
int zxc_max_level(void) { return ZXC_LEVEL_ULTRA; }
int zxc_default_level(void) { return ZXC_LEVEL_DEFAULT; }
const char* zxc_version_string(void) { return ZXC_LIB_VERSION_STR; }
size_t zxc_compress_opts_size(void) { return sizeof(zxc_compress_opts_t); }
size_t zxc_decompress_opts_size(void) { return sizeof(zxc_decompress_opts_t); }

const char* zxc_error_name(const int code) {
    switch (code) {
        case ZXC_OK: return "ZXC_OK";
        case ZXC_ERROR_MEMORY: return "ZXC_ERROR_MEMORY";
        case ZXC_ERROR_DST_TOO_SMALL: return "ZXC_ERROR_DST_TOO_SMALL";
        case ZXC_ERROR_SRC_TOO_SMALL: return "ZXC_ERROR_SRC_TOO_SMALL";
        case ZXC_ERROR_BAD_MAGIC: return "ZXC_ERROR_BAD_MAGIC";
        case ZXC_ERROR_BAD_VERSION: return "ZXC_ERROR_BAD_VERSION";
        case ZXC_ERROR_BAD_HEADER: return "ZXC_ERROR_BAD_HEADER";
        case ZXC_ERROR_BAD_CHECKSUM: return "ZXC_ERROR_BAD_CHECKSUM";
        case ZXC_ERROR_CORRUPT_DATA: return "ZXC_ERROR_CORRUPT_DATA";
        case ZXC_ERROR_BAD_OFFSET: return "ZXC_ERROR_BAD_OFFSET";
        case ZXC_ERROR_OVERFLOW: return "ZXC_ERROR_OVERFLOW";
        case ZXC_ERROR_IO: return "ZXC_ERROR_IO";
        case ZXC_ERROR_NULL_INPUT: return "ZXC_ERROR_NULL_INPUT";
        case ZXC_ERROR_BAD_BLOCK_TYPE: return "ZXC_ERROR_BAD_BLOCK_TYPE";
        case ZXC_ERROR_BAD_BLOCK_SIZE: return "ZXC_ERROR_BAD_BLOCK_SIZE";
        case ZXC_ERROR_DICT_REQUIRED: return "ZXC_ERROR_DICT_REQUIRED";
        case ZXC_ERROR_DICT_MISMATCH: return "ZXC_ERROR_DICT_MISMATCH";
        case ZXC_ERROR_DICT_TOO_LARGE: return "ZXC_ERROR_DICT_TOO_LARGE";
        case ZXC_ERROR_BAD_LEVEL: return "ZXC_ERROR_BAD_LEVEL";
        case ZXC_B200_ERROR_NO_DEVICE: return "ZXC_B200_ERROR_NO_DEVICE";
        case ZXC_B200_ERROR_CUDA: return "ZXC_B200_ERROR_CUDA";
        case ZXC_B200_ERROR_UNSUPPORTED: return "ZXC_B200_ERROR_UNSUPPORTED";
        default: return "ZXC_UNKNOWN_ERROR";
    }
}

uint64_t zxc_compress_bound(const size_t input_size) {
    if (input_size > (SIZE_MAX - (SIZE_MAX >> 8))) return 0;
    uint64_t n = ((uint64_t)input_size + ZXC_BLOCK_SIZE_MIN - 1) / ZXC_BLOCK_SIZE_MIN;
    if (n == 0) n = 1;
    return (uint64_t)ZXC_FILE_HEADER_SIZE + n * (ZXF_BLOCK_HDR + ZXF_BLOCK_CKS + ZXF_BLOCK_OVERHEAD) +
           (uint64_t)input_size + ZXF_BLOCK_HDR /* EOF */ + ZXF_BLOCK_HDR + n * ZXF_SEEK_ENTRY /* SEK */ +
           ZXC_FILE_FOOTER_SIZE;
}

uint64_t zxc_compress_block_bound(size_t input_size) {
    if (input_size == 0 || input_size > ZXC_BLOCK_SIZE_MAX) return 0;
    return (uint64_t)ZXF_BLOCK_HDR + input_size + ZXF_BLOCK_OVERHEAD + ZXF_BLOCK_CKS;
}

uint64_t zxc_decompress_block_bound(const size_t uncompressed_size) {
    if (uncompressed_size > ZXC_BLOCK_SIZE_MAX) return 0;
    return (uint64_t)uncompressed_size + ZXF_TAIL_PAD;
}

/* Device-side footprint of one in-flight encode block: input + hash/chain tables + streams. */
uint64_t zxc_estimate_cctx_size(size_t src_size, int level) {
    if (src_size == 0) return 0;
    const size_t bs = zxf_block_size_ceil(src_size);
    const uint64_t tables = (128u + 32u + 128u) * 1024u;
    return tables + (uint64_t)bs * (level >= ZXC_LEVEL_DENSITY ? 12u : 4u) + 4096;
}

uint64_t zxc_get_decompressed_size(const void* src, const size_t src_size) {
    if (!src || src_size < ZXC_FILE_HEADER_SIZE + ZXC_FILE_FOOTER_SIZE) return 0;
    const uint8_t* p = (const uint8_t*)src;
    if (zxf_le32(p) != ZXF_MAGIC) return 0;
    zxf_file_header_t fh;
    if (zxf_read_file_header(p, src_size, &fh, 1) != ZXC_OK) return 0;
    const uint64_t d = zxf_le64(p + src_size - ZXC_FILE_FOOTER_SIZE);
    return zxf_dsize_plausible(d, fh.block_size, src_size) ? d : 0;
}

uint32_t zxc_get_dict_id(const void* src, size_t src_size) {
    if (!src || src_size < ZXC_FILE_HEADER_SIZE) return 0;
    const uint8_t* p = (const uint8_t*)src;
    if (zxf_le32(p) != ZXF_MAGIC) return 0;
    return (p[6] & ZXF_FLAG_DICT) ? zxf_le32(p + 7) : 0;
}

/* ------------------------------------------------------------------------- */
/* dictionaries (.zxd)                                                       */
/* ------------------------------------------------------------------------- */
uint32_t zxc_dict_id(const void* dict, size_t dict_size, const void* huf_lengths) {
    if (!dict || dict_size == 0) return 0;
    const uint32_t base = zxf_checksum(dict, dict_size);
    return huf_lengths ? zxf_checksum_seed(huf_lengths, ZXC_HUF_TABLE_SIZE, base) : base;
}

uint32_t zxc_dict_get_id(const void* buf, size_t buf_size) {
    if (!buf || buf_size < ZXC_DICT_HEADER_SIZE) return 0;
    const uint8_t* p = (const uint8_t*)buf;
    return zxf_le32(p) == ZXF_DICT_MAGIC ? zxf_le32(p + 8) : 0;
}

size_t zxc_dict_save_bound(size_t content_size) {
    return (size_t)ZXC_DICT_HEADER_SIZE + content_size + ZXC_HUF_TABLE_SIZE;
}

int64_t zxc_dict_save(const void* content, size_t content_size, const void* huf_lengths, void* buf,
                      size_t buf_capacity) {
    if (!content || content_size == 0 || !huf_lengths) return ZXC_ERROR_NULL_INPUT;
    if (content_size > ZXC_DICT_SIZE_MAX) return ZXC_ERROR_DICT_TOO_LARGE;
    const size_t total = zxc_dict_save_bound(content_size);
    if (buf_capacity < total) return ZXC_ERROR_DST_TOO_SMALL;
    uint8_t* d = (uint8_t*)buf;
    zxf_st32(d, ZXF_DICT_MAGIC);
    d[4] = ZXF_DICT_VERSION;
    d[5] = 0;
    zxf_st16(d + 6, (uint32_t)content_size);
    zxf_st32(d + 8, zxc_dict_id(content, content_size, huf_lengths));
    zxf_st32(d + 12, 0);
    zxf_st16(d + 14, zxf_hash16(d));
    memcpy(d + ZXC_DICT_HEADER_SIZE, content, content_size);
    memcpy(d + ZXC_DICT_HEADER_SIZE + content_size, huf_lengths, ZXC_HUF_TABLE_SIZE);
    return (int64_t)total;
}

int zxc_dict_load(const void* buf, size_t buf_size, const void** content_out, size_t* content_size_out,
                  const void** huf_out, uint32_t* dict_id_out) {
    if (!buf || !content_out || !content_size_out) return ZXC_ERROR_NULL_INPUT;
    if (buf_size < ZXC_DICT_HEADER_SIZE) return ZXC_ERROR_SRC_TOO_SMALL;
    const uint8_t* s = (const uint8_t*)buf;
    if (zxf_le32(s) != ZXF_DICT_MAGIC) return ZXC_ERROR_BAD_MAGIC;
    if (s[4] != ZXF_DICT_VERSION) return ZXC_ERROR_BAD_VERSION;
    const size_t csz = zxf_le16(s + 6);
    if (csz == 0) return ZXC_ERROR_CORRUPT_DATA;
    if (buf_size < ZXC_DICT_HEADER_SIZE + csz + ZXC_HUF_TABLE_SIZE) return ZXC_ERROR_SRC_TOO_SMALL;
    uint8_t tmp[ZXC_DICT_HEADER_SIZE];
    memcpy(tmp, s, sizeof tmp);
    zxf_st32(tmp + 12, 0);
    if (zxf_le16(s + 14) != zxf_hash16(tmp)) return ZXC_ERROR_BAD_HEADER;
    const uint8_t* content = s + ZXC_DICT_HEADER_SIZE;
    const uint8_t* huf = content + csz;
    const uint32_t id = zxc_dict_id(content, csz, huf);
    if (zxf_le32(s + 8) != id) return ZXC_ERROR_BAD_CHECKSUM;
    *content_out = content;
    *content_size_out = csz;
    if (huf_out) *huf_out = huf;
    if (dict_id_out) *dict_id_out = id;
    return ZXC_OK;
}

const void* zxc_dict_huf(const void* buf, size_t buf_size) {
    if (!buf || buf_size < ZXC_DICT_HEADER_SIZE) return NULL;
    const uint8_t* s = (const uint8_t*)buf;
    if (zxf_le32(s) != ZXF_DICT_MAGIC || s[4] != ZXF_DICT_VERSION) return NULL;
    const size_t csz = zxf_le16(s + 6);
    if (csz == 0 || buf_size < ZXC_DICT_HEADER_SIZE + csz + ZXC_HUF_TABLE_SIZE) return NULL;
    return s + ZXC_DICT_HEADER_SIZE + csz;
}

/* the trainers (zxc_train_dict, zxc_train_dict_huf, zxc_dict_train) are in zxc_train.c */

/* ------------------------------------------------------------------------- */
/* frame planning (additive public entry)                                    */
/* ------------------------------------------------------------------------- */
static uint32_t expected_block_bytes(uint64_t total, uint32_t bs, uint64_t idx) {
    const uint64_t start = idx * bs;
    if (total <= start) return 0;
    const uint64_t rem = total - start;
    return rem >= bs ? bs : (uint32_t)rem;
}

typedef struct { const uint8_t* p; uint64_t n; } mem_span_t;

static int mem_fetch(void* ctx, void* dst, size_t len, uint64_t off) {
    const mem_span_t* m = (const mem_span_t*)ctx;
    if (off > m->n || len > m->n - off) return ZXC_ERROR_SRC_TOO_SMALL;
    memcpy(dst, m->p + off, len);
    return ZXC_OK;
}

int64_t zxc_b200_plan_frame(const void* frame, size_t frame_size, zxc_b200_job_t* jobs, size_t max_jobs,
                            zxc_b200_frame_info_t* info) {
    if (!frame) return ZXC_ERROR_NULL_INPUT;
    if (frame_size < ZXC_FILE_HEADER_SIZE + ZXC_FILE_FOOTER_SIZE) return ZXC_ERROR_SRC_TOO_SMALL;
    zxw_walk_t w;
    const int rc = zxw_walk((const uint8_t*)frame, frame_size, &w);
    if (rc != ZXC_OK) return rc;
    int64_t ret;
    if (w.end != ZXW_END_EOF) {
        ret = ZXC_ERROR_BAD_HEADER;
    } else {
        ret = (int64_t)w.n_jobs;
        if (info) {
            mem_span_t m = {(const uint8_t*)frame, frame_size};
            zxw_seek_t sk;
            info->decoded_size = w.footer_size;
            info->block_size = w.block_size;
            info->n_blocks = (uint32_t)w.n_jobs;
            info->dict_id = w.dict_id;
            info->has_checksum = w.has_checksum;
            info->global_hash = w.footer_hash;
            info->seekable = 0;
            if (zxw_seek_parse(mem_fetch, &m, frame_size, &sk) == ZXC_OK) {
                info->seekable = sk.num_blocks == w.n_jobs;
                zxw_seek_free(&sk);
            }
        }
        if (jobs) {
            if (max_jobs < w.n_jobs) {
                ret = ZXC_ERROR_DST_TOO_SMALL;
            } else {
                for (size_t i = 0; i < w.n_jobs; i++) {
                    jobs[i] = w.jobs[i];
                    jobs[i].dst_cap = expected_block_bytes(w.footer_size, w.block_size, i);
                }
            }
        }
    }
    zxw_free(&w);
    return ret;
}

/* ------------------------------------------------------------------------- */
/* contexts                                                                  */
/* ------------------------------------------------------------------------- */
struct zxc_dctx_s {
    zxg_ctx* gpu; /* owned device context (stream + buffers), created lazily */
    int is_static;
};

struct zxc_cctx_s {
    zxg_ctx* gpu;
    int is_static;
    int level;
    int checksum;
    size_t block_size;
};

zxc_dctx* zxc_create_dctx(void) { return (zxc_dctx*)calloc(1, sizeof(zxc_dctx)); }

void zxc_free_dctx(zxc_dctx* d) {
    if (!d) return;
    if (d->gpu) zxg_destroy(d->gpu);
    d->gpu = NULL;
    if (!d->is_static) free(d);
}

static int level_clamp(int level) { return level <= 0 ? ZXC_LEVEL_DEFAULT : (level > ZXC_LEVEL_ULTRA ? ZXC_LEVEL_ULTRA : level); }

zxc_cctx* zxc_create_cctx(const zxc_compress_opts_t* opts) {
    zxc_cctx* c = (zxc_cctx*)calloc(1, sizeof(zxc_cctx));
    if (!c) return NULL;
    c->level = level_clamp(opts ? opts->level : 0);
    c->block_size = (opts && opts->block_size) ? opts->block_size : ZXC_BLOCK_SIZE_DEFAULT;
    c->checksum = opts ? opts->checksum_enabled : 0;
    if (opts && !zxf_valid_block_size(c->block_size)) {
        free(c);
        return NULL;
    }
    return c;
}

void zxc_free_cctx(zxc_cctx* c) {
    if (!c) return;
    if (c->gpu) zxg_destroy(c->gpu);
    c->gpu = NULL;
    if (!c->is_static) free(c);
}

/* Static-workspace variants: the handle lives in the caller's memory; device
 * scratch is still owned by the library (host workspaces cannot hold HBM). */
size_t zxc_static_dctx_workspace_size(const size_t block_size) {
    return zxf_valid_block_size(block_size) ? ((sizeof(zxc_dctx) + 63) & ~(size_t)63) : 0;
}
zxc_dctx* zxc_init_static_dctx(void* workspace, const size_t workspace_size, const size_t block_size) {
    const size_t need = zxc_static_dctx_workspace_size(block_size);
    if (!workspace || need == 0 || workspace_size < need || ((uintptr_t)workspace & 7)) return NULL;
    zxc_dctx* d = (zxc_dctx*)workspace;
    memset(d, 0, sizeof *d);
    d->is_static = 1;
    return d;
}
size_t zxc_static_cctx_workspace_size(const size_t block_size, const int level) {
    (void)level;
    return zxf_valid_block_size(block_size) ? ((sizeof(zxc_cctx) + 63) & ~(size_t)63) : 0;
}
zxc_cctx* zxc_init_static_cctx(void* workspace, const size_t workspace_size, const zxc_compress_opts_t* opts) {
    const size_t bs = (opts && opts->block_size) ? opts->block_size : ZXC_BLOCK_SIZE_DEFAULT;
    const size_t need = zxc_static_cctx_workspace_size(bs, opts ? opts->level : 0);
    if (!workspace || need == 0 || workspace_size < need || ((uintptr_t)workspace & 7)) return NULL;
    zxc_cctx* c = (zxc_cctx*)workspace;
    memset(c, 0, sizeof *c);
    c->is_static = 1;
    c->level = level_clamp(opts ? opts->level : 0);
    c->block_size = bs;
    c->checksum = opts ? opts->checksum_enabled : 0;
    return c;
}

/* ------------------------------------------------------------------------- */
/* frame decode                                                              */
/* ------------------------------------------------------------------------- */
/* First job in stream order that did not produce exactly its planned size.  *size_mismatch = 1 when the plan, not
 * the block, may be at fault: a block decoded to another size, or -- block_size != 0 -- a block that was given less
 * room than block_size (the frame's tail) ran out of it.  The reference decodes every block into block_size bytes
 * and only then asks whether the result still fits (DST_TOO_SMALL, zxc_dispatch.c:912-1001); the caller re-plans. */
/* ---- several GPUs behind one call -------------------------------------------------------------------------
 * The reference's data-parallel entry is a fork-join over host threads (zxc_seekable.c:999-1108: contiguous block
 * stripes, one worker each).  The same split works over devices: with ZXC_B200_DEVICES=<n> | all in the environment
 * (opt-in; default 1) a large frame or range is cut into contiguous block stripes, one host thread per device runs
 * the usual overlapped H2D / decode / D2H pipeline on its stripe through a context of that device (its own PCIe
 * link, copy pool and NUMA-local bounce buffers), and the statuses land in one table so the verdict logic is the
 * single-device one.  Never on by default: a process launched once per GPU (torchrun) must not fan out again. */
#define ZX_MAX_DEV 16
typedef struct {
    int device, own_thread;
    const uint8_t* src;
    zxg_fetch_fn fetch;
    void* fetch_ctx;
    uint8_t* dst;              /* where decoded byte clip_lo lands */
    uint64_t clip_lo, clip_hi; /* decoded range wanted, job coordinates */
    const zxc_b200_job_t* jobs;
    uint32_t n;
    int32_t* st;
    const void* dict;
    uint32_t dict_size;
    const void* dict_huf;
    uint32_t bs;
    int verify, pinned, rc; /* pinned: src and dst are both page-locked */
} zx_part;

/* One stripe through an overlapped pipeline: zxg_decode_pipelined straight from / into the caller's memory when the
 * source is memory-backed, both buffers are page-locked and the stripe's blocks are wanted whole; zxg_decode_staged
 * through the pinned bounce buffers otherwise. */
static void part_run(zx_part* p, zxg_ctx* g) {
    const uint32_t n = p->n;
    const uint64_t d0 = p->jobs[0].dst_off, d1 = p->jobs[n - 1].dst_off + p->jobs[n - 1].dst_cap;
    const zxc_b200_job_t* jb = p->jobs;
    zxc_b200_job_t* local = NULL;
    if (d0 != 0) { /* a later stripe: stripe-local decoded coordinates; source offsets stay absolute */
        local = (zxc_b200_job_t*)malloc((size_t)n * sizeof *local);
        if (!local) { p->rc = ZXC_ERROR_MEMORY; return; }
        for (uint32_t i = 0; i < n; i++) {
            local[i] = p->jobs[i];
            local[i].dst_off -= d0;
        }
        jb = local;
    }
    const uint64_t src_lo = p->jobs[0].src_off, src_hi = p->jobs[n - 1].src_off + p->jobs[n - 1].src_len;
    const uint64_t lo = p->clip_lo > d0 ? p->clip_lo : d0, hi = p->clip_hi < d1 ? p->clip_hi : d1;
    uint8_t* out = p->dst + (lo - p->clip_lo);
    if (p->pinned && !p->fetch && lo == d0 && hi == d1)
        p->rc = zxg_decode_pipelined(g, p->src, src_lo, src_hi, out, d1 - d0, jb, n, p->st, p->dict, p->dict_size,
                                     p->dict_huf, p->bs, p->verify);
    else
        p->rc = zxg_decode_staged(g, p->src, p->fetch, p->fetch_ctx, src_lo, src_hi, out, lo - d0, hi - d0, jb, n, p->st,
                                  p->dict, p->dict_size, p->dict_huf, p->bs, p->verify);
    free(local);
}

static void* part_main(void* arg) {
    zx_part* p = (zx_part*)arg;
    p->rc = zxg_set_device(p->device);
    if (p->rc != ZXC_OK) return NULL;
    zxg_ctx* g = zxg_acquire();
    if (!g) { p->rc = ZXC_ERROR_MEMORY; return NULL; }
    part_run(p, g);
    zxg_release(g);
    return NULL;
}

/* how many devices a call decoding `decoded_bytes` may use: the environment's wish, the devices there are, and at
 * least 64 MiB of output per stripe */
static int multi_devices(uint64_t decoded_bytes) {
    const char* e = getenv("ZXC_B200_DEVICES");
    if (!e || !*e) return 1;
    int want = strcmp(e, "all") == 0 ? ZX_MAX_DEV : atoi(e);
    if (want <= 1) return 1;
    const int nd = zxg_device_count();
    if (want > nd) want = nd;
    if (want > ZX_MAX_DEV) want = ZX_MAX_DEV;
    const uint64_t by_size = decoded_bytes >> 26;
    if ((uint64_t)want > by_size) want = (int)by_size;
    return want < 1 ? 1 : want;
}

/* the whole call's jobs (contiguous, dst_off ascending) over D devices; g0 = the caller's context (stripe 0, calling
 * thread) */
static int decode_multi(int D, zxg_ctx* g0, const zx_part* whole) {
    zx_part parts[ZX_MAX_DEV];
    pthread_t th[ZX_MAX_DEV];
    const int cur = zxg_current_device(), nd = zxg_device_count();
    const uint32_t n = whole->n, per = (n + (uint32_t)D - 1) / (uint32_t)D;
    int np = 0;
    for (uint32_t start = 0; start < n && np < ZX_MAX_DEV; start += per, np++) {
        zx_part* p = &parts[np];
        *p = *whole;
        p->device = (cur + np) % (nd > 0 ? nd : 1);
        p->jobs = whole->jobs + start;
        p->n = n - start < per ? n - start : per;
        p->st = whole->st + start;
    }
    for (int k = 1; k < np; k++) parts[k].own_thread = pthread_create(&th[k], NULL, part_main, &parts[k]) == 0;
    part_run(&parts[0], g0);
    for (int k = 1; k < np; k++) {
        if (parts[k].own_thread) pthread_join(th[k], NULL);
        else { /* no thread to be had: this stripe on the caller's device after all */
            part_run(&parts[k], g0);
        }
    }
    zxg_set_device(cur);
    for (int k = 0; k < np; k++)
        if (parts[k].rc != ZXC_OK) return parts[k].rc;
    return ZXC_OK;
}

/* decoded bytes from which a call overlaps H2D, decode and D2H chunk by chunk; below it, one round trip */
#define STREAM_MIN_BYTES ((uint64_t)32 << 20)

/* The decode of a planned frame or range between host buffers, by one of three routes:
 *   - may_stream and >= STREAM_MIN_BYTES decoded: decode_multi over several devices when the environment asks for
 *     it (multi_devices), else one stripe on the caller's context (part_run: pipelined or staged);
 *   - otherwise in HBM: one H2D of the source span (through a bounce when the source is `fetch`), zxg_decode_jobs, and
 *     one D2H of [clip_lo, clip_hi) -- only when every job produced its planned size, so a failed small decode leaves
 *     dst untouched.
 * Jobs: source offsets absolute (src / fetch coordinates), decoded offsets from 0; decoded bytes [clip_lo, clip_hi)
 * land at dst.  The per-job statuses in st are the caller's to judge; the return value is ZXC_OK or a failure of the
 * call itself (memory, CUDA, fetch). */
static int decode_to_host(zxg_ctx* g, const uint8_t* src, zxg_fetch_fn fetch, void* fetch_ctx, uint8_t* dst,
                          uint64_t clip_lo, uint64_t clip_hi, const zxc_b200_job_t* jobs, uint32_t n, int32_t* st,
                          const void* dict, uint32_t dict_size, const void* dict_huf, uint32_t bs, int verify,
                          int may_stream) {
    const uint64_t produced = jobs[n - 1].dst_off + jobs[n - 1].dst_cap;
    if (may_stream && produced >= STREAM_MIN_BYTES) {
        zx_part whole = {.src = src, .fetch = fetch, .fetch_ctx = fetch_ctx, .dst = dst, .clip_lo = clip_lo,
                         .clip_hi = clip_hi, .jobs = jobs, .n = n, .st = st, .dict = dict, .dict_size = dict_size,
                         .dict_huf = dict_huf, .bs = bs, .verify = verify,
                         .pinned = src && zxg_host_pinned(src) && zxg_host_pinned(dst)};
        const int D = multi_devices(produced);
        if (D > 1) return decode_multi(D, g, &whole);
        part_run(&whole, g);
        return whole.rc;
    }
    const uint64_t src_lo = jobs[0].src_off, src_hi = jobs[n - 1].src_off + jobs[n - 1].src_len;
    uint8_t* d_in = (uint8_t*)zxg_buffer(g, ZXG_BUF_IN, (size_t)(src_hi - src_lo) + 16);
    uint8_t* d_out = (uint8_t*)zxg_buffer(g, ZXG_BUF_OUT, (size_t)produced + 16);
    if (!d_in || !d_out) return ZXC_ERROR_MEMORY;
    int rc;
    if (!fetch) {
        rc = zxg_h2d(g, d_in, src + src_lo, (size_t)(src_hi - src_lo));
    } else { /* a reader-backed source: pull the compressed span through a host bounce */
        const size_t chunk = (size_t)16 << 20;
        uint8_t* bounce = (uint8_t*)malloc(src_hi - src_lo < chunk ? (size_t)(src_hi - src_lo) : chunk);
        rc = bounce ? ZXC_OK : ZXC_ERROR_MEMORY;
        for (uint64_t p = src_lo; rc == ZXC_OK && p < src_hi;) {
            const size_t len = src_hi - p < chunk ? (size_t)(src_hi - p) : chunk;
            rc = fetch(fetch_ctx, bounce, len, p);
            if (rc == ZXC_OK) rc = zxg_h2d(g, d_in + (p - src_lo), bounce, len);
            if (rc == ZXC_OK) rc = zxg_sync(g);
            p += len;
        }
        free(bounce);
    }
    if (rc != ZXC_OK) return rc;
    rc = zxg_decode_jobs(g, d_in - src_lo, d_out, jobs, n, st, dict, dict_size, dict_huf, bs, verify);
    if (rc != ZXC_OK) return rc;
    for (uint32_t i = 0; i < n; i++)
        if (st[i] < 0 || (uint32_t)st[i] != jobs[i].dst_cap) return ZXC_OK;
    return zxg_d2h(g, dst, d_out + clip_lo, (size_t)(clip_hi - clip_lo));
}

/* The reference hands every block block_size + ZXC_DECOMPRESS_TAIL_PAD bytes of room (zxc_dispatch.c:902,
 * :961-976) and only afterwards asks whether the result fits the caller's buffer, so a damaged block may
 * legally decode to a little more than block_size.  The regular plan gives block i exactly its expected
 * size; a block that ran out of room there (OVERFLOW, or DST_TOO_SMALL from the literal count) is therefore
 * not a verdict yet but a plan mismatch, settled by the general split below. */
static int64_t first_failure(const int32_t* st, const zxc_b200_job_t* jobs, size_t n, int* size_mismatch) {
    *size_mismatch = 0;
    for (size_t i = 0; i < n; i++) {
        if (st[i] == ZXC_ERROR_OVERFLOW || st[i] == ZXC_ERROR_DST_TOO_SMALL) {
            *size_mismatch = 1;
            return st[i];
        }
        if (st[i] < 0) return st[i];
        if ((uint32_t)st[i] != jobs[i].dst_cap) {
            *size_mismatch = 1;
            return ZXC_ERROR_CORRUPT_DATA;
        }
    }
    return 0;
}

/* Frames whose non-final blocks decode to less than block_size.  The reference's encoder never emits one, but
 * its decoder accepts any split (zxc_dispatch.c:912-1001: every block is decoded on its own and appended), so
 * this build does too: one pass over all blocks to learn their sizes (each into its own block_size slot), the
 * reference's verdict order over those sizes (first failing block, then capacity), then a second pass that
 * decodes every block at its true offset.  Only reached after the regular plan saw a size mismatch. */
static int64_t decompress_frame_any_split(zxg_ctx* g, const uint8_t* src, const zxw_walk_t* w, uint8_t* dst,
                                          size_t dst_capacity, const uint8_t* dict, size_t dict_size,
                                          const uint8_t* dict_huf, int verify, uint64_t* produced_out) {
    const size_t n = w->n_jobs;
    const uint32_t bs = w->block_size;
    zxc_b200_job_t* jobs = (zxc_b200_job_t*)malloc(n * sizeof *jobs);
    int32_t* st = (int32_t*)malloc(n * sizeof *st);
    int64_t ret = ZXC_OK;
    if (!jobs || !st) { ret = ZXC_ERROR_MEMORY; goto out; }
    const uint64_t src_lo = w->jobs[0].src_off, src_hi = w->jobs[n - 1].src_off + w->jobs[n - 1].src_len;
    uint8_t* d_in = (uint8_t*)zxg_buffer(g, ZXG_BUF_IN, (size_t)(src_hi - src_lo) + 16);
    if (!d_in) { ret = ZXC_ERROR_MEMORY; goto out; }
    int rc = zxg_h2d(g, d_in, src + src_lo, (size_t)(src_hi - src_lo));
    if (rc != ZXC_OK) { ret = rc; goto out; }
    /* pass 1: sizes, a window of blocks at a time (the bytes are thrown away) */
    const size_t room = (size_t)bs + ZXF_TAIL_PAD; /* what the reference gives one block (:902) */
    const size_t win = ((size_t)256 << 20) / room ? ((size_t)256 << 20) / room : 1;
    for (size_t i0 = 0; i0 < n; i0 += win) {
        const size_t cnt = n - i0 < win ? n - i0 : win;
        uint8_t* d_tmp = (uint8_t*)zxg_buffer(g, ZXG_BUF_OUT, cnt * room + 16);
        if (!d_tmp) { ret = ZXC_ERROR_MEMORY; goto out; }
        for (size_t k = 0; k < cnt; k++) {
            jobs[i0 + k] = w->jobs[i0 + k];
            jobs[i0 + k].dst_off = (uint64_t)k * room;
            jobs[i0 + k].dst_cap = (uint32_t)room;
        }
        rc = zxg_decode_jobs(g, d_in - src_lo, d_tmp, jobs + i0, (uint32_t)cnt, st + i0, dict, (uint32_t)dict_size, dict_huf, bs,
                             verify);
        if (rc != ZXC_OK) { ret = rc; goto out; }
    }
    /* the reference's order: a block's own error first, then whether it still fits */
    uint64_t op = 0;
    for (size_t i = 0; i < n; i++) {
        if (st[i] < 0) { ret = st[i]; goto out; }
        if ((uint64_t)st[i] > dst_capacity - op) { ret = ZXC_ERROR_DST_TOO_SMALL; goto out; }
        jobs[i].dst_off = op;
        jobs[i].dst_cap = (uint32_t)st[i];
        op += (uint64_t)st[i];
    }
    /* pass 2: every block at its true offset */
    if (op > 0) {
        uint8_t* d_out = (uint8_t*)zxg_buffer(g, ZXG_BUF_OUT, (size_t)op + 16);
        if (!d_out) { ret = ZXC_ERROR_MEMORY; goto out; }
        rc = zxg_decode_jobs(g, d_in - src_lo, d_out, jobs, (uint32_t)n, st, dict, (uint32_t)dict_size, dict_huf, bs, verify);
        if (rc != ZXC_OK) { ret = rc; goto out; }
        for (size_t i = 0; i < n; i++)
            if (st[i] < 0 || (uint32_t)st[i] != jobs[i].dst_cap) { ret = st[i] < 0 ? st[i] : ZXC_ERROR_CORRUPT_DATA; goto out; }
        rc = zxg_d2h(g, dst, d_out, (size_t)op);
        if (rc != ZXC_OK) { ret = rc; goto out; }
    }
    *produced_out = op;
out:
    free(jobs);
    free(st);
    return ret;
}

/* The reference attaches the dictionary's literal table once per frame (zxc_cctx_attach_dict_huf, zxc_common.c:490):
 * an all-zero table counts as no table, so enc_lit = 3 blocks then need one (DICT_REQUIRED); a table with a length
 * above 11, or whose lengths are not a complete code (one symbol of length 1 excepted), fails the whole frame.
 * Returns 1 for a usable table, 0 for none, ZXC_ERROR_CORRUPT_DATA for a bad one. */
static int dict_huf_attach(const uint8_t* h) {
    if (!h) return 0;
    uint32_t kraft = 0, present = 0, any = 0, len1 = 0;
    for (int i = 0; i < 128; i++) {
        any |= h[i];
        for (int k = 0; k < 2; k++) {
            const uint32_t l = (h[i] >> (4 * k)) & 15u;
            if (l > 11) return ZXC_ERROR_CORRUPT_DATA;
            if (l) {
                kraft += 1u << (11 - l);
                present++;
                len1 += l == 1;
            }
        }
    }
    if (!any) return 0;
    if (kraft != (1u << 11) && !(present == 1 && len1 == 1)) return ZXC_ERROR_CORRUPT_DATA;
    return 1;
}

static int64_t decompress_frame(zxg_ctx* g, const uint8_t* src, size_t src_size, uint8_t* dst,
                                size_t dst_capacity, const zxc_decompress_opts_t* opts) {
    const int checksum_enabled = opts ? opts->checksum_enabled : 0;
    const uint8_t* dict = opts ? (const uint8_t*)opts->dict : NULL;
    const size_t dict_size = (opts && opts->dict) ? opts->dict_size : 0;
    const uint8_t* dict_huf = (opts && opts->dict) ? (const uint8_t*)opts->dict_huf : NULL;

    if (dict_size > ZXC_DICT_SIZE_MAX) return ZXC_ERROR_DICT_TOO_LARGE; /* zxc_dispatch.c:671 */
    zxw_walk_t w;
    const int wrc = zxw_walk(src, src_size, &w);
    if (wrc != ZXC_OK) return wrc;
    int64_t ret;
    int32_t* status = NULL;

    if (w.dict_id != 0) {
        if (!dict || dict_size == 0) { ret = ZXC_ERROR_DICT_REQUIRED; goto out; }
        if (zxc_dict_id(dict, dict_size, dict_huf) != w.dict_id) { ret = ZXC_ERROR_DICT_MISMATCH; goto out; }
    }
    if (dict_size) {
        const int arc = dict_huf_attach(dict_huf);
        if (arc < 0) { ret = arc; goto out; }
        if (arc == 0) dict_huf = NULL;
    }
    const int verify = w.has_checksum && checksum_enabled;

    /* Output placement: block i starts at i*block_size.  That holds for every
     * frame the reference encoder emits; the decode verifies it per block. */
    size_t n_fit = 0;
    uint64_t produced = 0;
    for (size_t i = 0; i < w.n_jobs; i++) {
        uint32_t exp = expected_block_bytes(w.footer_size, w.block_size, i);
        if (i + 1 < w.n_jobs && exp != w.block_size) exp = w.block_size; /* footer smaller than the walk: decided below */
        if (exp == 0) exp = w.block_size;
        if (w.jobs[i].dst_off + exp > dst_capacity) break;
        w.jobs[i].dst_cap = exp;
        produced = w.jobs[i].dst_off + exp;
        n_fit++;
    }

    if (n_fit > 0) {
        status = (int32_t*)malloc(n_fit * sizeof *status);
        if (!status) { ret = ZXC_ERROR_MEMORY; goto out; }
        /* in place (source and destination overlap): the whole frame must be on the device before the first decoded
         * byte comes back, so no streaming */
        const int overlap = (const uint8_t*)src < dst + dst_capacity && dst < (const uint8_t*)src + src_size;
        const int rc = decode_to_host(g, src, NULL, NULL, dst, 0, produced, w.jobs, (uint32_t)n_fit, status, dict,
                                      (uint32_t)dict_size, dict_huf, w.block_size, verify, !overlap);
        if (rc != ZXC_OK) { ret = rc; goto out; }
        /* a short final block is legal when the footer agrees; anything else is decided by the
         * reference's own order: first block error, else capacity, else footer */
        int mismatch = 0;
        const int64_t ff = first_failure(status, w.jobs, n_fit, &mismatch);
        if (ff < 0 && mismatch) goto any_split;
        if (ff < 0) { ret = ff; goto out; }
    }
    if (n_fit < w.n_jobs && w.end == ZXW_END_EOF && w.footer_size <= dst_capacity) goto any_split; /* short blocks may fit */
    if (0) {
    any_split:; /* a block decoded to something other than its planned size: general split (see above) */
        uint64_t p2 = 0;
        const int64_t r2 = decompress_frame_any_split(g, src, &w, dst, dst_capacity, dict, dict_size, dict_huf, verify, &p2);
        if (r2 < 0) { ret = r2; goto out; }
        produced = p2;
        n_fit = w.n_jobs;
    }
    /* decoded: capacity, block-stream end, footer size, global hash */
    if (n_fit < w.n_jobs) { ret = ZXC_ERROR_DST_TOO_SMALL; goto out; }
    if (w.end == ZXW_END_BAD_HEADER) { ret = ZXC_ERROR_BAD_HEADER; goto out; }
    if (w.end == ZXW_END_EOF) {
        if (w.footer_size != produced) { ret = ZXC_ERROR_CORRUPT_DATA; goto out; }
        if (verify && w.footer_hash != w.global_hash) { ret = ZXC_ERROR_BAD_CHECKSUM; goto out; }
    }
    ret = (int64_t)produced;
out:
    free(status);
    zxw_free(&w);
    return ret;
}

static int64_t decompress_entry(zxg_ctx* owned, const void* src, size_t src_size, void* dst, size_t dst_capacity,
                                const zxc_decompress_opts_t* opts) {
    if (!src || (!dst && dst_capacity != 0)) return ZXC_ERROR_NULL_INPUT;
    if (src_size < ZXC_FILE_HEADER_SIZE + ZXC_FILE_FOOTER_SIZE) return ZXC_ERROR_SRC_TOO_SMALL;
    if (!dst || dst_capacity == 0) { /* empty-frame shortcut (zxc_dispatch.c:848-853) */
        if (zxf_le32((const uint8_t*)src) != ZXF_MAGIC) return ZXC_ERROR_BAD_MAGIC;
        return zxf_le64((const uint8_t*)src + src_size - ZXC_FILE_FOOTER_SIZE) == 0 ? 0 : ZXC_ERROR_DST_TOO_SMALL;
    }
    /* header-level rejects need no device: keep them ahead of device bring-up so the
     * reference's reject vectors read the same on any box */
    zxf_file_header_t fh;
    const int hrc = zxf_read_file_header((const uint8_t*)src, src_size, &fh, 1);
    if (hrc != ZXC_OK) return hrc;
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    zxg_ctx* g = owned ? owned : zxg_acquire();
    if (!g) return ZXC_ERROR_MEMORY;
    const int64_t r = decompress_frame(g, (const uint8_t*)src, src_size, (uint8_t*)dst, dst_capacity, opts);
    if (!owned) zxg_release(g);
    return r;
}

int64_t zxc_decompress(const void* src, const size_t src_size, void* dst, const size_t dst_capacity,
                       const zxc_decompress_opts_t* opts) {
    return decompress_entry(NULL, src, src_size, dst, dst_capacity, opts);
}

int64_t zxc_decompress_dctx(zxc_dctx* dctx, const void* src, size_t src_size, void* dst, size_t dst_capacity,
                            const zxc_decompress_opts_t* opts) {
    if (!dctx) return ZXC_ERROR_NULL_INPUT;
    if (!dctx->gpu && zxg_init() == ZXC_OK) dctx->gpu = zxg_create();
    return decompress_entry(dctx->gpu, src, src_size, dst, dst_capacity, opts);
}

/* in-place: the frame is staged to HBM before any output is written back, so
 * the reference's read/write-gap margins are not needed for correctness; the
 * bound keeps the reference's formula so callers size buffers identically. */
static uint64_t inplace_margin(uint64_t dsize, size_t bs, int has_cs) {
    const uint64_t nb = (dsize + bs - 1) / bs;
    return (uint64_t)bs + nb * (ZXF_BLOCK_HDR + (has_cs ? ZXF_BLOCK_CKS : 0)) + ZXF_BLOCK_HDR +
           (ZXF_BLOCK_HDR + nb * ZXF_SEEK_ENTRY) + ZXC_FILE_FOOTER_SIZE + ZXF_TAIL_PAD;
}

/* on the frame's 16 header bytes and its footer's 8-byte size */
static int inplace_probe(const uint8_t* header, uint64_t d, size_t comp_size, uint64_t* dsize, uint64_t* margin) {
    if (zxf_le32(header) != ZXF_MAGIC) return ZXC_ERROR_BAD_MAGIC;
    zxf_file_header_t fh;
    if (zxf_read_file_header(header, ZXC_FILE_HEADER_SIZE, &fh, 1) != ZXC_OK) return ZXC_ERROR_BAD_HEADER;
    if (!zxf_dsize_plausible(d, fh.block_size, comp_size)) return ZXC_ERROR_CORRUPT_DATA;
    *dsize = d;
    *margin = inplace_margin(d, fh.block_size, fh.has_checksum);
    return ZXC_OK;
}

static size_t inplace_bound(const uint8_t* header, uint64_t d, size_t src_size) {
    uint64_t m = 0;
    if (inplace_probe(header, d, src_size, &d, &m) != ZXC_OK) return 0;
    const uint64_t by_payload = d + m;
    const uint64_t by_placement = (uint64_t)src_size + m;
    return (size_t)(by_payload > by_placement ? by_payload : by_placement);
}

size_t zxc_decompress_inplace_bound(const void* src, const size_t src_size) {
    if (!src || src_size < ZXC_FILE_HEADER_SIZE + ZXC_FILE_FOOTER_SIZE) return 0;
    const uint8_t* s = (const uint8_t*)src;
    return inplace_bound(s, zxf_le64(s + src_size - ZXC_FILE_FOOTER_SIZE), src_size);
}

int64_t zxc_decompress_inplace(void* buffer, const size_t buffer_capacity, const size_t comp_size,
                               const zxc_decompress_opts_t* opts) {
    if (!buffer || comp_size < ZXC_FILE_HEADER_SIZE + ZXC_FILE_FOOTER_SIZE || comp_size > buffer_capacity)
        return ZXC_ERROR_NULL_INPUT;
    uint8_t* buf = (uint8_t*)buffer;
    const uint8_t* comp = buf + (buffer_capacity - comp_size);
    uint64_t d = 0, m = 0;
    const int rc = inplace_probe(comp, zxf_le64(comp + comp_size - ZXC_FILE_FOOTER_SIZE), comp_size, &d, &m);
    if (rc != ZXC_OK) return rc;
    if (d > buffer_capacity || buffer_capacity - d < m) return ZXC_ERROR_DST_TOO_SMALL;
    /* source and destination overlap: decompress_frame then takes the in-HBM route, where the whole
     * frame is on the device before the first decoded byte comes back */
    return decompress_entry(NULL, comp, comp_size, buf, buffer_capacity, opts);
}

/* ------------------------------------------------------------------------- */
/* block API (frameless)                                                     */
/* ------------------------------------------------------------------------- */
static int64_t decode_one_block(zxc_dctx* dctx, const void* src, size_t src_size, void* dst, size_t dst_capacity,
                                const zxc_decompress_opts_t* opts) {
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    if (!dctx->gpu) dctx->gpu = zxg_create();
    zxg_ctx* g = dctx->gpu;
    if (!g) return ZXC_ERROR_MEMORY;
    const uint8_t* dict = opts ? (const uint8_t*)opts->dict : NULL;
    const size_t dict_size = (opts && opts->dict) ? opts->dict_size : 0;
    const uint8_t* dict_huf = NULL; /* the reference's block API attaches no literal table: enc_lit = 3 needs one */
    const int verify = opts ? opts->checksum_enabled : 0;
    if (dict_size > ZXC_DICT_SIZE_MAX) return ZXC_ERROR_DICT_TOO_LARGE;
    uint8_t* d_in = (uint8_t*)zxg_buffer(g, ZXG_BUF_IN, src_size + 16);
    uint8_t* d_out = (uint8_t*)zxg_buffer(g, ZXG_BUF_OUT, dst_capacity + 16);
    if (!d_in || !d_out) return ZXC_ERROR_MEMORY;
    int rc = zxg_h2d(g, d_in, src, src_size);
    if (rc != ZXC_OK) return rc;
    zxc_b200_job_t job = {0, 0, (uint32_t)(src_size > 0xFFFFFFFFu ? 0xFFFFFFFFu : src_size), (uint32_t)dst_capacity};
    int32_t st = 0;
    rc = zxg_decode_jobs(g, d_in, d_out, &job, 1, &st, dict, (uint32_t)dict_size, dict_huf,
                         (uint32_t)zxf_block_size_ceil(dst_capacity), verify);
    if (rc != ZXC_OK) return rc;
    if (st < 0) return st;
    rc = zxg_d2h(g, dst, d_out, (size_t)st);
    return rc != ZXC_OK ? rc : (int64_t)st;
}

int64_t zxc_decompress_block(zxc_dctx* dctx, const void* src, size_t src_size, void* dst, size_t dst_capacity,
                             const zxc_decompress_opts_t* opts) {
    if (!dctx || !src || !dst || src_size < ZXF_BLOCK_HDR || dst_capacity == 0) return ZXC_ERROR_NULL_INPUT;
    if (dst_capacity > ZXC_BLOCK_SIZE_MAX + ZXF_TAIL_PAD) return ZXC_ERROR_BAD_BLOCK_SIZE;
    return decode_one_block(dctx, src, src_size, dst, dst_capacity, opts);
}

/* The GPU decoder writes exact bytes, so the "safe" (exact-capacity) variant is the same path. */
int64_t zxc_decompress_block_safe(zxc_dctx* dctx, const void* src, const size_t src_size, void* dst,
                                  const size_t dst_capacity, const zxc_decompress_opts_t* opts) {
    if (!dctx || !src || !dst || src_size < ZXF_BLOCK_HDR || dst_capacity == 0) return ZXC_ERROR_NULL_INPUT;
    if (dst_capacity > ZXC_BLOCK_SIZE_MAX) return ZXC_ERROR_BAD_BLOCK_SIZE;
    return decode_one_block(dctx, src, src_size, dst, dst_capacity, opts);
}

/* ------------------------------------------------------------------------- */
/* encode entry points: frame assembly on the host around zxg_encode_body     */
/* (all levels encode on the GPU; without a device they fail loudly).        */
/* ------------------------------------------------------------------------- */
/* the dictionary's shared literal table (zxc_cctx_attach_dict_huf, zxc_common.c:490-513): an all-zero table means
 * "none" (*have = 0); a malformed one fails the call.  Fills huf_lens with one length per byte. */
static int unpack_dict_huf(const uint8_t* dict_huf, uint8_t huf_lens[256], int* have) {
    int have_huf = 0;
    if (dict_huf) {
        for (int i = 0; i < ZXC_HUF_TABLE_SIZE; i++) {
            huf_lens[2 * i] = dict_huf[i] & 15u;
            huf_lens[2 * i + 1] = dict_huf[i] >> 4;
            have_huf |= dict_huf[i];
        }
        if (have_huf) {
            zxh_geom_t geom;
            if (zxh_geometry(huf_lens, &geom) != 0) return ZXC_ERROR_CORRUPT_DATA;
            have_huf = 1;
        }
    }
    *have = have_huf;
    return ZXC_OK;
}

/* the SEK block's header: its payload is one ZXF_SEEK_ENTRY per block */
static void seek_table_header(uint8_t* dst, uint32_t num_blocks) {
    zxf_write_block_header(dst, ZXF_BLOCK_HDR, ZXF_BT_SEK, num_blocks * ZXF_SEEK_ENTRY);
}

/* bytes of a frame around its body: file header, EOF block, SEK table, footer */
static uint64_t frame_fixed_bytes(uint32_t nb, int seekable) {
    return ZXC_FILE_HEADER_SIZE + ZXF_BLOCK_HDR + ((seekable && nb > 0) ? zxc_seek_table_size(nb) : 0) +
           ZXC_FILE_FOOTER_SIZE;
}

static int64_t compress_frame(zxg_ctx* g, const uint8_t* src, size_t src_size, uint8_t* dst, size_t dst_capacity,
                              int level, size_t block_size, int checksum, int seekable, const uint8_t* dict,
                              size_t dict_size, const uint8_t* dict_huf) {
    const uint64_t nb64 = (src_size + block_size - 1) / block_size;
    if (nb64 > 0xFFFFFFFFull - 2) return ZXC_ERROR_BAD_BLOCK_SIZE;
    const uint32_t nb = (uint32_t)nb64;
    const size_t trailer = frame_fixed_bytes(nb, seekable) - ZXC_FILE_HEADER_SIZE;
    if (dst_capacity < ZXC_FILE_HEADER_SIZE + trailer) return ZXC_ERROR_DST_TOO_SMALL;
    const uint32_t did = (dict && dict_size) ? zxc_dict_id(dict, dict_size, dict_huf) : 0;
    uint8_t huf_lens[256];
    int have_huf = 0;
    int r = unpack_dict_huf(dict_huf, huf_lens, &have_huf);
    if (r != ZXC_OK) return r;
    r = zxf_write_file_header(dst, dst_capacity, block_size, checksum, did);
    if (r < 0) return r;
    uint32_t* sizes = nb ? (uint32_t*)malloc((size_t)nb * sizeof *sizes) : NULL;
    if (nb && !sizes) return ZXC_ERROR_MEMORY;
    uint64_t body = 0;
    const uint64_t body_cap = dst_capacity - ZXC_FILE_HEADER_SIZE - trailer;
    const int rc = zxg_encode_body(g, src, src_size, (uint32_t)block_size, level, checksum, nb,
                                   dst + ZXC_FILE_HEADER_SIZE, body_cap, sizes, &body, dict, (uint32_t)dict_size,
                                   have_huf ? huf_lens : NULL);
    if (rc != ZXC_OK) {
        free(sizes);
        return rc;
    }
    uint8_t* op = dst + ZXC_FILE_HEADER_SIZE + body;
    uint32_t ghash = 0;
    if (checksum) { /* global hash: rotate-xor fold of the per-block checksums, in order (:751-758) */
        const uint8_t* bp = dst + ZXC_FILE_HEADER_SIZE;
        for (uint32_t i = 0; i < nb; i++) {
            bp += sizes[i];
            ghash = zxf_hash_combine(ghash, zxf_le32(bp - ZXF_BLOCK_CKS));
        }
    }
    op += zxf_write_block_header(op, ZXF_BLOCK_HDR, ZXF_BT_EOF, 0);
    if (seekable && nb > 0) op += zxc_write_seek_table(op, zxc_seek_table_size(nb), sizes, nb);
    op += zxf_write_footer(op, ZXC_FILE_FOOTER_SIZE, src_size, ghash, checksum);
    free(sizes);
    return (int64_t)(op - dst);
}

int64_t zxc_compress(const void* src, const size_t src_size, void* dst, const size_t dst_capacity,
                     const zxc_compress_opts_t* opts) {
    if (!dst || dst_capacity == 0 || (src_size > 0 && !src)) return ZXC_ERROR_NULL_INPUT;
    const int checksum = opts ? opts->checksum_enabled : 0;
    const int seekable = opts ? opts->seekable : 0;
    const int level = level_clamp(opts ? opts->level : 0);
    const size_t dict_size = (opts && opts->dict) ? opts->dict_size : 0;
    const size_t block_size = (opts && opts->block_size) ? opts->block_size : ZXC_BLOCK_SIZE_DEFAULT;
    if (dict_size > ZXC_DICT_SIZE_MAX) return ZXC_ERROR_DICT_TOO_LARGE;
    if (!zxf_valid_block_size(block_size)) return ZXC_ERROR_BAD_BLOCK_SIZE;
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    /* every level encodes on the GPU: greedy / lazy parsers (1-5), optimal parser + PivCo stage (6-7) */
    const uint8_t* dict = opts ? (const uint8_t*)opts->dict : NULL;
    const uint8_t* dict_huf = (opts && opts->dict) ? (const uint8_t*)opts->dict_huf : NULL;
    zxg_ctx* g = zxg_acquire();
    if (!g) return ZXC_ERROR_MEMORY;
    const int64_t r = compress_frame(g, (const uint8_t*)src, src_size, (uint8_t*)dst, dst_capacity, level, block_size,
                                     checksum, seekable, dict, dict_size, dict_huf);
    zxg_release(g);
    return r;
}

/* ---- device to device (include/zxc_b200.h) ---- */
/* A prepared dictionary in device memory: the regions the calls would stage from its bytes, and what they would decide
 * about its literal table. */
struct zxc_b200_dict_device_s {
    zxg_ddict_t g;
    void* mem;       /* owned: zxg_ddict_bytes(size) bytes on `device` */
    uint32_t id;     /* zxc_dict_id(dict, size, huf) */
    int device;
    int huf_rc;      /* unpack_dict_huf's verdict: what the frame compress calls return (ZXC_OK or CORRUPT_DATA) */
    int huf_verdict; /* dict_huf_attach's: what the frame decode calls report on the device */
};

zxc_b200_dict_device* zxc_b200_dict_device_create(const void* dict, size_t dict_size, const void* dict_huf, int* err,
                                                  void* stream) {
    int rc_;
    int* rc = err ? err : &rc_;
    *rc = ZXC_ERROR_NULL_INPUT;
    if (!dict || dict_size == 0) return NULL;
    *rc = ZXC_ERROR_DICT_TOO_LARGE;
    if (dict_size > ZXC_DICT_SIZE_MAX) return NULL;
    *rc = zxg_init();
    if (*rc != ZXC_OK) return NULL;
    zxc_b200_dict_device* dd = (zxc_b200_dict_device*)calloc(1, sizeof *dd);
    if (dd) dd->mem = zxg_dev_alloc(zxg_ddict_bytes((uint32_t)dict_size));
    if (!dd || !dd->mem) {
        free(dd);
        *rc = ZXC_ERROR_MEMORY;
        return NULL;
    }
    uint8_t lens[256];
    int have_huf = 0;
    dd->huf_rc = unpack_dict_huf((const uint8_t*)dict_huf, lens, &have_huf);
    dd->huf_verdict = dict_huf_attach((const uint8_t*)dict_huf);
    dd->id = zxc_dict_id(dict, dict_size, dict_huf);
    dd->device = zxg_current_device();
    *rc = zxg_ddict_build(dd->mem, dict, (uint32_t)dict_size, dd->huf_verdict == 1 ? dict_huf : NULL,
                          dd->huf_rc == ZXC_OK && have_huf ? lens : NULL, stream, &dd->g);
    if (*rc != ZXC_OK) {
        zxg_dev_free(dd->mem);
        free(dd);
        return NULL;
    }
    return dd;
}

uint32_t zxc_b200_dict_device_id(const zxc_b200_dict_device* dd) { return dd ? dd->id : 0; }
size_t zxc_b200_dict_device_size(const zxc_b200_dict_device* dd) { return dd ? dd->g.dict_size : 0; }

void zxc_b200_dict_device_free(zxc_b200_dict_device* dd) {
    if (!dd) return;
    const int prev = zxg_current_device();
    const int rc = dd->device == prev ? ZXC_OK : zxg_set_device(dd->device);
    zxg_dev_free(dd->mem); /* waits for the calls that may still read it */
    if (rc == ZXC_OK && dd->device != prev) zxg_set_device(prev);
    free(dd);
}

/* The device check of a device call: a device, and the prepared dictionary's (when given) current */
static int device_ready(const zxc_b200_dict_device* dd) {
    const int rc = zxg_init();
    if (rc != ZXC_OK) return rc;
    return dd && dd->device != zxg_current_device() ? ZXC_B200_ERROR_NO_DEVICE : ZXC_OK;
}

/* Each device call has one body for its two entry points: the base call passes its opts, the _using_dict variant opts
 * without their dictionary fields and the prepared dictionary dd (NULL: none). */
static const zxc_compress_opts_t* copts_no_dict(const zxc_compress_opts_t* opts, zxc_compress_opts_t* tmp) {
    if (!opts) return NULL;
    *tmp = *opts;
    tmp->dict = NULL;
    tmp->dict_size = 0;
    tmp->dict_huf = NULL;
    return tmp;
}
static const zxc_decompress_opts_t* dopts_no_dict(const zxc_decompress_opts_t* opts, zxc_decompress_opts_t* tmp) {
    if (!opts) return NULL;
    *tmp = *opts;
    tmp->dict = NULL;
    tmp->dict_size = 0;
    tmp->dict_huf = NULL;
    return tmp;
}

/* zxc_compress's option checks, in its order; fills the effective level, block size and block count */
static int device_opts(uint64_t src_size, const zxc_compress_opts_t* opts, int* level, size_t* block_size,
                       uint32_t* n_blocks) {
    const size_t dict_size = (opts && opts->dict) ? opts->dict_size : 0;
    *level = level_clamp(opts ? opts->level : 0);
    *block_size = (opts && opts->block_size) ? opts->block_size : ZXC_BLOCK_SIZE_DEFAULT;
    if (dict_size > ZXC_DICT_SIZE_MAX) return ZXC_ERROR_DICT_TOO_LARGE;
    if (!zxf_valid_block_size(*block_size)) return ZXC_ERROR_BAD_BLOCK_SIZE;
    const uint64_t nb64 = (src_size + *block_size - 1) / *block_size;
    if (nb64 > 0xFFFFFFFFull - 2) return ZXC_ERROR_BAD_BLOCK_SIZE;
    *n_blocks = (uint32_t)nb64;
    return ZXC_OK;
}

/* The dictionary of a frame compress: opts' host bytes (staged by the call) or the prepared dd */
typedef struct {
    const uint8_t* dict;
    uint32_t dict_size;
    const zxg_ddict_t* dd;
    uint32_t id;
    const uint8_t* huf_lens; /* the host table's unpacked lengths when it is usable (dd carries its own) */
    uint8_t lens[256];
} cdict_t;
/* unpack_dict_huf's verdict on the table, and the rest of *c */
static int cdict_resolve(const zxc_compress_opts_t* opts, const zxc_b200_dict_device* dd, cdict_t* c) {
    memset(c, 0, sizeof *c);
    if (dd) {
        c->dd = &dd->g;
        c->id = dd->id;
        return dd->huf_rc;
    }
    const uint8_t* dict_huf = (opts && opts->dict) ? (const uint8_t*)opts->dict_huf : NULL;
    c->dict = opts ? (const uint8_t*)opts->dict : NULL;
    c->dict_size = (uint32_t)((opts && opts->dict) ? opts->dict_size : 0);
    int have_huf = 0;
    const int rc = unpack_dict_huf(dict_huf, c->lens, &have_huf);
    if (rc != ZXC_OK) return rc;
    c->huf_lens = have_huf ? c->lens : NULL;
    c->id = (c->dict && c->dict_size) ? zxc_dict_id(c->dict, c->dict_size, dict_huf) : 0;
    return ZXC_OK;
}

size_t zxc_b200_encode_scratch_size(uint64_t src_size, const zxc_compress_opts_t* opts) {
    int level;
    size_t bs;
    uint32_t nb;
    if (device_opts(src_size, opts, &level, &bs, &nb) != ZXC_OK) return 0;
    const size_t dict_size = (opts && opts->dict) ? opts->dict_size : 0;
    return zxg_encode_scratch_bytes(src_size, (uint32_t)bs, level, nb, (uint32_t)dict_size);
}

static int compress_device(const void* d_src, uint64_t src_size, void* d_dst, uint64_t dst_capacity,
                           const zxc_compress_opts_t* opts, const zxc_b200_dict_device* dd, void* d_scratch,
                           size_t scratch_size, int64_t* d_result, zxc_b200_job_t* d_jobs, void* stream) {
    if (!d_dst || dst_capacity == 0 || (src_size > 0 && !d_src) || !d_scratch || !d_result) return ZXC_ERROR_NULL_INPUT;
    int level;
    size_t block_size;
    uint32_t nb;
    int rc = device_opts(src_size, opts, &level, &block_size, &nb);
    if (rc != ZXC_OK) return rc;
    rc = device_ready(dd);
    if (rc != ZXC_OK) return rc;
    const int checksum = opts ? opts->checksum_enabled : 0;
    const int seekable = opts ? opts->seekable : 0;
    zxg_frame_bytes_t fb;
    memset(&fb, 0, sizeof fb);
    fb.fixed = frame_fixed_bytes(nb, seekable);
    fb.dst_capacity = dst_capacity;
    fb.seekable = seekable && nb > 0;
    if (dst_capacity < fb.fixed) return ZXC_ERROR_DST_TOO_SMALL;
    cdict_t c;
    rc = cdict_resolve(opts, dd, &c);
    if (rc != ZXC_OK) return rc;
    zxf_write_file_header(fb.header, sizeof fb.header, block_size, checksum, c.id);
    zxf_write_block_header(fb.eof, sizeof fb.eof, ZXF_BT_EOF, 0);
    if (fb.seekable) seek_table_header(fb.sek, nb);
    zxf_write_footer(fb.footer, sizeof fb.footer, src_size, 0, checksum);
    return zxg_compress_device(d_src, src_size, d_dst, (uint32_t)block_size, level, checksum, nb, c.dict, c.dict_size,
                               c.huf_lens, c.dd, &fb, d_scratch, scratch_size, d_result, d_jobs, stream);
}

int zxc_b200_compress_device(const void* d_src, uint64_t src_size, void* d_dst, uint64_t dst_capacity,
                             const zxc_compress_opts_t* opts, void* d_scratch, size_t scratch_size, int64_t* d_result,
                             zxc_b200_job_t* d_jobs, void* stream) {
    return compress_device(d_src, src_size, d_dst, dst_capacity, opts, NULL, d_scratch, scratch_size, d_result, d_jobs,
                           stream);
}

int zxc_b200_compress_device_using_dict(const void* d_src, uint64_t src_size, void* d_dst, uint64_t dst_capacity,
                                        const zxc_compress_opts_t* opts, const zxc_b200_dict_device* dd,
                                        void* d_scratch, size_t scratch_size, int64_t* d_result,
                                        zxc_b200_job_t* d_jobs, void* stream) {
    zxc_compress_opts_t t;
    return compress_device(d_src, src_size, d_dst, dst_capacity, copts_no_dict(opts, &t), dd, d_scratch, scratch_size,
                           d_result, d_jobs, stream);
}

size_t zxc_b200_compress_device_to_host_scratch_size(uint64_t src_size, uint64_t window,
                                                     const zxc_compress_opts_t* opts) {
    int level;
    size_t bs;
    uint32_t nb;
    if (device_opts(src_size, opts, &level, &bs, &nb) != ZXC_OK) return 0;
    const size_t dict_size = (opts && opts->dict) ? opts->dict_size : 0;
    const int seekable = opts && opts->seekable && nb > 0;
    return zxg_c2h_scratch_bytes(src_size, window, (uint32_t)bs, level, nb, (uint32_t)dict_size, seekable);
}

/* zxc_b200_compress_device's host verdicts, then UNSUPPORTED for a room that is not mapped page-locked memory */
static int compress_device_to_host(const void* d_src, uint64_t src_size, void* h_dst, uint64_t dst_capacity,
                                   const zxc_compress_opts_t* opts, const zxc_b200_dict_device* dd, uint64_t window,
                                   void* d_scratch, size_t scratch_size, int64_t* d_result, void* stream) {
    if (!h_dst || dst_capacity == 0 || (src_size > 0 && !d_src) || !d_scratch || !d_result) return ZXC_ERROR_NULL_INPUT;
    int level;
    size_t block_size;
    uint32_t nb;
    int rc = device_opts(src_size, opts, &level, &block_size, &nb);
    if (rc != ZXC_OK) return rc;
    rc = device_ready(dd);
    if (rc != ZXC_OK) return rc;
    const int checksum = opts ? opts->checksum_enabled : 0;
    const int seekable = opts ? opts->seekable : 0;
    zxg_frame_bytes_t fb;
    memset(&fb, 0, sizeof fb);
    fb.fixed = frame_fixed_bytes(nb, seekable);
    fb.dst_capacity = dst_capacity;
    fb.seekable = seekable && nb > 0;
    if (dst_capacity < fb.fixed) return ZXC_ERROR_DST_TOO_SMALL;
    cdict_t c;
    rc = cdict_resolve(opts, dd, &c);
    if (rc != ZXC_OK) return rc;
    void* mapped = (void*)zxg_host_mapped(h_dst, (size_t)dst_capacity);
    if (!mapped) return ZXC_B200_ERROR_UNSUPPORTED;
    zxf_write_file_header(fb.header, sizeof fb.header, block_size, checksum, c.id);
    zxf_write_block_header(fb.eof, sizeof fb.eof, ZXF_BT_EOF, 0);
    if (fb.seekable) seek_table_header(fb.sek, nb);
    zxf_write_footer(fb.footer, sizeof fb.footer, src_size, 0, checksum);
    return zxg_compress_device_to_host(d_src, src_size, mapped, window, (uint32_t)block_size, level, checksum, nb,
                                       c.dict, c.dict_size, c.huf_lens, c.dd, &fb, d_scratch, scratch_size, d_result,
                                       stream);
}

int zxc_b200_compress_device_to_host(const void* d_src, uint64_t src_size, void* h_dst, uint64_t dst_capacity,
                                     const zxc_compress_opts_t* opts, uint64_t window, void* d_scratch,
                                     size_t scratch_size, int64_t* d_result, void* stream) {
    return compress_device_to_host(d_src, src_size, h_dst, dst_capacity, opts, NULL, window, d_scratch, scratch_size,
                                   d_result, stream);
}

int zxc_b200_compress_device_to_host_using_dict(const void* d_src, uint64_t src_size, void* h_dst,
                                                uint64_t dst_capacity, const zxc_compress_opts_t* opts,
                                                const zxc_b200_dict_device* dd, uint64_t window, void* d_scratch,
                                                size_t scratch_size, int64_t* d_result, void* stream) {
    zxc_compress_opts_t t;
    return compress_device_to_host(d_src, src_size, h_dst, dst_capacity, copts_no_dict(opts, &t), dd, window,
                                   d_scratch, scratch_size, d_result, stream);
}

size_t zxc_b200_compress_device_batch_scratch_size(uint32_t max_frames, uint64_t max_total_src,
                                                   const zxc_compress_opts_t* opts) {
    int level;
    size_t bs;
    uint32_t nb;
    if (device_opts(0, opts, &level, &bs, &nb) != ZXC_OK) return 0;
    const size_t dict_size = (opts && opts->dict) ? opts->dict_size : 0;
    return zxg_compress_batch_scratch_bytes(max_frames, max_total_src, (uint32_t)bs, level, (uint32_t)dict_size);
}

/* The host decides what needs no descriptor, in zxc_b200_compress_device's order; the device makes that call's
 * per-buffer checks and the rest per frame and writes them to d_results (zxc_cbatch.cuh). */
static int compress_device_batch(const zxc_b200_frame_t* d_frames, uint32_t n_frames, const zxc_compress_opts_t* opts,
                                 const zxc_b200_dict_device* dd, void* d_scratch, size_t scratch_size,
                                 int64_t* d_results, void* stream) {
    if (n_frames > 0 && (!d_frames || !d_results || !d_scratch)) return ZXC_ERROR_NULL_INPUT;
    int level;
    size_t block_size;
    uint32_t nb;
    int rc = device_opts(0, opts, &level, &block_size, &nb);
    if (rc != ZXC_OK) return rc;
    rc = device_ready(dd);
    if (rc != ZXC_OK) return rc;
    const int checksum = opts ? opts->checksum_enabled : 0;
    cdict_t c;
    rc = cdict_resolve(opts, dd, &c);
    if (rc != ZXC_OK || n_frames == 0) return rc;
    uint8_t header[16], eof[8];
    zxf_write_file_header(header, sizeof header, block_size, checksum, c.id);
    zxf_write_block_header(eof, sizeof eof, ZXF_BT_EOF, 0);
    return zxg_compress_device_batch(d_frames, n_frames, (uint32_t)block_size, level, checksum,
                                     opts ? opts->seekable : 0, c.dict, c.dict_size, c.huf_lens, c.dd, header, eof,
                                     d_scratch, scratch_size, d_results, stream);
}

int zxc_b200_compress_device_batch(const zxc_b200_frame_t* d_frames, uint32_t n_frames, const zxc_compress_opts_t* opts,
                                   void* d_scratch, size_t scratch_size, int64_t* d_results, void* stream) {
    return compress_device_batch(d_frames, n_frames, opts, NULL, d_scratch, scratch_size, d_results, stream);
}

int zxc_b200_compress_device_batch_using_dict(const zxc_b200_frame_t* d_frames, uint32_t n_frames,
                                              const zxc_compress_opts_t* opts, const zxc_b200_dict_device* dd,
                                              void* d_scratch, size_t scratch_size, int64_t* d_results, void* stream) {
    zxc_compress_opts_t t;
    return compress_device_batch(d_frames, n_frames, copts_no_dict(opts, &t), dd, d_scratch, scratch_size, d_results,
                                 stream);
}

size_t zxc_b200_decompress_device_scratch_size(uint64_t dst_capacity, uint32_t block_size) {
    if (!zxf_valid_block_size(block_size)) return 0;
    return zxg_decompress_scratch_bytes(dst_capacity, block_size);
}

/* The decode options of the device-resident decodes: decompress_frame's dictionary checks that need no frame bytes,
 * for opts' host dictionary or the prepared dd */
static int device_dopts(const zxc_decompress_opts_t* opts, const zxc_b200_dict_device* dd, zxg_dopts_t* o) {
    memset(o, 0, sizeof *o);
    o->checksum_enabled = opts ? opts->checksum_enabled : 0;
    if (dd) {
        o->d_dict = dd->g.dec;
        o->d_dict_huf = dd->g.dec_huf;
        o->dict_size = dd->g.dict_size;
        o->dict_id = dd->id;
        o->huf_verdict = dd->huf_verdict;
        return ZXC_OK;
    }
    const uint8_t* dict = opts ? (const uint8_t*)opts->dict : NULL;
    const size_t dict_size = (opts && opts->dict) ? opts->dict_size : 0;
    const uint8_t* dict_huf = (opts && opts->dict) ? (const uint8_t*)opts->dict_huf : NULL;
    if (dict_size > ZXC_DICT_SIZE_MAX) return ZXC_ERROR_DICT_TOO_LARGE;
    o->dict = dict_size ? dict : NULL;
    o->dict_size = (uint32_t)dict_size;
    o->dict_id = (dict && dict_size) ? zxc_dict_id(dict, dict_size, dict_huf) : 0;
    o->huf_verdict = dict_size ? dict_huf_attach(dict_huf) : 0;
    o->dict_huf = o->huf_verdict == 1 ? dict_huf : NULL;
    return ZXC_OK;
}

/* The host decides what needs no frame bytes, in zxc_decompress's order (decompress_entry, decompress_frame); the
 * device decides the rest and writes it to *d_result (zxc_dplan.cuh). */
static int decompress_device(const void* d_src, uint64_t src_size, void* d_dst, uint64_t dst_capacity,
                             const zxc_decompress_opts_t* opts, const zxc_b200_dict_device* dd, void* d_scratch,
                             size_t scratch_size, int64_t* d_result, void* stream) {
    if (!d_src || (!d_dst && dst_capacity != 0) || !d_scratch || !d_result) return ZXC_ERROR_NULL_INPUT;
    if (src_size < ZXC_FILE_HEADER_SIZE + ZXC_FILE_FOOTER_SIZE) return ZXC_ERROR_SRC_TOO_SMALL;
    zxg_dopts_t o;
    const int orc = device_dopts(opts, dd, &o);
    if (orc != ZXC_OK) return orc;
    const int irc = device_ready(dd);
    if (irc != ZXC_OK) return irc;
    return zxg_decompress_device(d_src, src_size, d_dst, dst_capacity, &o, d_scratch, scratch_size, d_result, stream);
}

int zxc_b200_decompress_device(const void* d_src, uint64_t src_size, void* d_dst, uint64_t dst_capacity,
                               const zxc_decompress_opts_t* opts, void* d_scratch, size_t scratch_size,
                               int64_t* d_result, void* stream) {
    return decompress_device(d_src, src_size, d_dst, dst_capacity, opts, NULL, d_scratch, scratch_size, d_result, stream);
}

int zxc_b200_decompress_device_using_dict(const void* d_src, uint64_t src_size, void* d_dst, uint64_t dst_capacity,
                                          const zxc_decompress_opts_t* opts, const zxc_b200_dict_device* dd,
                                          void* d_scratch, size_t scratch_size, int64_t* d_result, void* stream) {
    zxc_decompress_opts_t t;
    return decompress_device(d_src, src_size, d_dst, dst_capacity, dopts_no_dict(opts, &t), dd, d_scratch,
                             scratch_size, d_result, stream);
}

size_t zxc_b200_decompress_inplace_device_scratch_size(uint64_t buffer_capacity, uint32_t block_size, uint64_t window) {
    if (!zxf_valid_block_size(block_size)) return 0;
    return zxg_decompress_inplace_scratch_bytes(buffer_capacity, block_size, window);
}

size_t zxc_b200_decompress_inplace_device_bound(const void* d_src, uint64_t src_size, void* stream) {
    if (!d_src || src_size < ZXC_FILE_HEADER_SIZE + ZXC_FILE_FOOTER_SIZE || zxg_init() != ZXC_OK) return 0;
    uint8_t header[ZXC_FILE_HEADER_SIZE], footer[8];
    if (zxg_d2h_sync(header, d_src, sizeof header, stream) != ZXC_OK ||
        zxg_d2h_sync(footer, (const uint8_t*)d_src + src_size - ZXC_FILE_FOOTER_SIZE, sizeof footer, stream) != ZXC_OK)
        return 0;
    return inplace_bound(header, zxf_le64(footer), src_size);
}

uint64_t zxc_b200_seek_table_device_bound(const void* d_frame, uint64_t frame_size, void* stream) {
    if (!d_frame || frame_size < ZXC_FILE_HEADER_SIZE + ZXF_BLOCK_HDR + ZXC_FILE_FOOTER_SIZE || zxg_init() != ZXC_OK)
        return 0;
    const uint8_t* f = (const uint8_t*)d_frame;
    uint8_t header[ZXC_FILE_HEADER_SIZE], footer[8], sek[ZXF_BLOCK_HDR];
    zxf_file_header_t fh;
    if (zxg_d2h_sync(header, f, sizeof header, stream) != ZXC_OK ||
        zxf_read_file_header(header, sizeof header, &fh, 1) != ZXC_OK ||
        zxg_d2h_sync(footer, f + frame_size - ZXC_FILE_FOOTER_SIZE, sizeof footer, stream) != ZXC_OK)
        return 0;
    const uint64_t total = zxf_le64(footer);
    if (total == 0) return frame_size;
    const uint64_t nb = total / fh.block_size + (total % fh.block_size != 0);
    if (nb > UINT32_MAX / ZXF_SEEK_ENTRY) return 0;
    const uint64_t table = zxc_seek_table_size((uint32_t)nb);
    /* the table zxw_walk's prefetch hint would find: a SEK header for nb entries where it would start */
    if (table + ZXC_FILE_FOOTER_SIZE + ZXC_FILE_HEADER_SIZE <= frame_size) {
        uint8_t type;
        uint32_t comp;
        if (zxg_d2h_sync(sek, f + frame_size - ZXC_FILE_FOOTER_SIZE - table, sizeof sek, stream) != ZXC_OK) return 0;
        if (zxf_read_block_header(sek, sizeof sek, &type, &comp) == ZXC_OK && type == ZXF_BT_SEK &&
            comp == (uint32_t)(nb * ZXF_SEEK_ENTRY))
            return frame_size;
    }
    return frame_size + table;
}

size_t zxc_b200_seek_table_device_scratch_size(uint64_t frame_size, uint32_t max_blocks) {
    return zxg_seek_table_scratch_bytes(frame_size, max_blocks);
}

/* The host decides what needs no frame bytes; the device decides the rest (zxc_dindex.cuh). */
int zxc_b200_add_seek_table_device(void* d_buffer, uint64_t frame_size, uint64_t buffer_capacity, void* d_scratch,
                                   size_t scratch_size, int64_t* d_result, void* stream) {
    if (!d_buffer || !d_scratch || !d_result || frame_size > buffer_capacity) return ZXC_ERROR_NULL_INPUT;
    if (frame_size < ZXC_FILE_HEADER_SIZE + ZXF_BLOCK_HDR + ZXC_FILE_FOOTER_SIZE) return ZXC_ERROR_SRC_TOO_SMALL;
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    return zxg_add_seek_table_device(d_buffer, frame_size, buffer_capacity, d_scratch, scratch_size, d_result, stream);
}

/* The host decides what zxc_decompress_inplace decides without the frame's bytes, then what
 * zxc_b200_decompress_device decides without them; the device decides the rest (zxc_dinplace.cuh). */
static int decompress_inplace_device(void* d_buffer, uint64_t buffer_capacity, uint64_t comp_size,
                                     const zxc_decompress_opts_t* opts, const zxc_b200_dict_device* dd,
                                     void* d_scratch, size_t scratch_size, int64_t* d_result, void* stream) {
    if (!d_buffer || comp_size < ZXC_FILE_HEADER_SIZE + ZXC_FILE_FOOTER_SIZE || comp_size > buffer_capacity ||
        !d_scratch || !d_result)
        return ZXC_ERROR_NULL_INPUT;
    zxg_dopts_t o;
    const int orc = device_dopts(opts, dd, &o);
    if (orc != ZXC_OK) return orc;
    const int irc = device_ready(dd);
    if (irc != ZXC_OK) return irc;
    return zxg_decompress_inplace_device(d_buffer, buffer_capacity, comp_size, &o, d_scratch, scratch_size, d_result,
                                         stream);
}

int zxc_b200_decompress_inplace_device(void* d_buffer, uint64_t buffer_capacity, uint64_t comp_size,
                                       const zxc_decompress_opts_t* opts, void* d_scratch, size_t scratch_size,
                                       int64_t* d_result, void* stream) {
    return decompress_inplace_device(d_buffer, buffer_capacity, comp_size, opts, NULL, d_scratch, scratch_size,
                                     d_result, stream);
}

int zxc_b200_decompress_inplace_device_using_dict(void* d_buffer, uint64_t buffer_capacity, uint64_t comp_size,
                                                  const zxc_decompress_opts_t* opts, const zxc_b200_dict_device* dd,
                                                  void* d_scratch, size_t scratch_size, int64_t* d_result,
                                                  void* stream) {
    zxc_decompress_opts_t t;
    return decompress_inplace_device(d_buffer, buffer_capacity, comp_size, dopts_no_dict(opts, &t), dd, d_scratch,
                                     scratch_size, d_result, stream);
}

size_t zxc_b200_decompress_device_batch_scratch_size(uint32_t max_frames, uint64_t max_total_capacity,
                                                     uint32_t block_size) {
    if (!zxf_valid_block_size(block_size)) return 0;
    return zxg_decompress_batch_scratch_bytes(max_frames, max_total_capacity, block_size);
}

/* The host decides what needs neither the descriptors nor the frames' bytes; the device decides the rest per frame
 * and writes it to d_results (zxc_dbatch.cuh). */
static int decompress_device_batch(const zxc_b200_frame_t* d_frames, uint32_t n_frames,
                                   const zxc_decompress_opts_t* opts, const zxc_b200_dict_device* dd, void* d_scratch,
                                   size_t scratch_size, int64_t* d_results, void* stream) {
    if (n_frames > 0 && (!d_frames || !d_results || !d_scratch)) return ZXC_ERROR_NULL_INPUT;
    zxg_dopts_t o;
    const int orc = device_dopts(opts, dd, &o);
    if (orc != ZXC_OK) return orc;
    const int irc = device_ready(dd);
    if (irc != ZXC_OK || n_frames == 0) return irc;
    return zxg_decompress_device_batch(d_frames, n_frames, &o, d_scratch, scratch_size, d_results, stream);
}

int zxc_b200_decompress_device_batch(const zxc_b200_frame_t* d_frames, uint32_t n_frames,
                                     const zxc_decompress_opts_t* opts, void* d_scratch, size_t scratch_size,
                                     int64_t* d_results, void* stream) {
    return decompress_device_batch(d_frames, n_frames, opts, NULL, d_scratch, scratch_size, d_results, stream);
}

int zxc_b200_decompress_device_batch_using_dict(const zxc_b200_frame_t* d_frames, uint32_t n_frames,
                                                const zxc_decompress_opts_t* opts, const zxc_b200_dict_device* dd,
                                                void* d_scratch, size_t scratch_size, int64_t* d_results,
                                                void* stream) {
    zxc_decompress_opts_t t;
    return decompress_device_batch(d_frames, n_frames, dopts_no_dict(opts, &t), dd, d_scratch, scratch_size,
                                   d_results, stream);
}

/* ---- the block API in HBM: zxc_compress_block / zxc_decompress_block(_safe) over a batch ---- */
size_t zxc_b200_compress_blocks_device_scratch_size(uint32_t max_blocks, uint64_t max_total_src, uint32_t max_src_size,
                                                    const zxc_compress_opts_t* opts) {
    const size_t dict_size = (opts && opts->dict) ? opts->dict_size : 0;
    if (dict_size > ZXC_DICT_SIZE_MAX) return 0;
    return zxg_compress_blocks_scratch_bytes(max_blocks, max_total_src, max_src_size, level_clamp(opts ? opts->level : 0),
                                             (uint32_t)dict_size);
}

/* The host decides what needs no descriptor; the device makes zxc_compress_block's per-item checks and the rest and
 * writes them to d_results (zxc_blocks.cuh).  The options resolve as on a fresh zxc_create_cctx(NULL) context. */
static int compress_blocks_device(const zxc_b200_frame_t* d_items, uint32_t n_items, const zxc_compress_opts_t* opts,
                                  const zxc_b200_dict_device* dd, void* d_scratch, size_t scratch_size,
                                  int64_t* d_results, void* stream) {
    if (n_items > 0 && (!d_items || !d_results || !d_scratch)) return ZXC_ERROR_NULL_INPUT;
    const uint8_t* dict = opts ? (const uint8_t*)opts->dict : NULL;
    const size_t dict_size = (opts && opts->dict) ? opts->dict_size : 0;
    if (dict_size > ZXC_DICT_SIZE_MAX) return ZXC_ERROR_DICT_TOO_LARGE;
    const int irc = device_ready(dd);
    if (irc != ZXC_OK || n_items == 0) return irc;
    return zxg_compress_blocks_device(d_items, n_items, level_clamp(opts ? opts->level : 0),
                                      opts ? opts->checksum_enabled : 0, dict, (uint32_t)dict_size,
                                      dd ? &dd->g : NULL, d_scratch, scratch_size, d_results, stream);
}

int zxc_b200_compress_blocks_device(const zxc_b200_frame_t* d_items, uint32_t n_items, const zxc_compress_opts_t* opts,
                                    void* d_scratch, size_t scratch_size, int64_t* d_results, void* stream) {
    return compress_blocks_device(d_items, n_items, opts, NULL, d_scratch, scratch_size, d_results, stream);
}

int zxc_b200_compress_blocks_device_using_dict(const zxc_b200_frame_t* d_items, uint32_t n_items,
                                               const zxc_compress_opts_t* opts, const zxc_b200_dict_device* dd,
                                               void* d_scratch, size_t scratch_size, int64_t* d_results, void* stream) {
    zxc_compress_opts_t t;
    return compress_blocks_device(d_items, n_items, copts_no_dict(opts, &t), dd, d_scratch, scratch_size, d_results,
                                  stream);
}

size_t zxc_b200_decompress_blocks_device_scratch_size(uint32_t max_blocks, uint64_t max_dst_capacity) {
    return zxg_decompress_blocks_scratch_bytes(max_blocks, max_dst_capacity);
}

static int decompress_blocks_device(const zxc_b200_frame_t* d_items, uint32_t n_items,
                                    const zxc_decompress_opts_t* opts, const zxc_b200_dict_device* dd, int safe,
                                    void* d_scratch, size_t scratch_size, int64_t* d_results, void* stream) {
    if (n_items > 0 && (!d_items || !d_results || !d_scratch)) return ZXC_ERROR_NULL_INPUT;
    zxg_dopts_t o;
    const int orc = device_dopts(opts, dd, &o);
    if (orc != ZXC_OK) return orc;
    o.dict_huf = NULL; /* the block API attaches no literal table (decode_one_block) */
    o.d_dict_huf = NULL;
    const int irc = device_ready(dd);
    if (irc != ZXC_OK || n_items == 0) return irc;
    return zxg_decompress_blocks_device(d_items, n_items, &o, safe, d_scratch, scratch_size, d_results, stream);
}

int zxc_b200_decompress_blocks_device(const zxc_b200_frame_t* d_items, uint32_t n_items,
                                      const zxc_decompress_opts_t* opts, int safe, void* d_scratch,
                                      size_t scratch_size, int64_t* d_results, void* stream) {
    return decompress_blocks_device(d_items, n_items, opts, NULL, safe, d_scratch, scratch_size, d_results, stream);
}

int zxc_b200_decompress_blocks_device_using_dict(const zxc_b200_frame_t* d_items, uint32_t n_items,
                                                 const zxc_decompress_opts_t* opts, const zxc_b200_dict_device* dd,
                                                 int safe, void* d_scratch, size_t scratch_size, int64_t* d_results,
                                                 void* stream) {
    zxc_decompress_opts_t t;
    return decompress_blocks_device(d_items, n_items, dopts_no_dict(opts, &t), dd, safe, d_scratch, scratch_size,
                                    d_results, stream);
}

int64_t zxc_compress_cctx(zxc_cctx* cctx, const void* src, size_t src_size, void* dst, size_t dst_capacity,
                          const zxc_compress_opts_t* opts) {
    if (!cctx) return ZXC_ERROR_NULL_INPUT;
    zxc_compress_opts_t o;
    memset(&o, 0, sizeof o);
    if (opts) o = *opts;
    if (o.level <= 0) o.level = cctx->level;
    if (o.block_size == 0) o.block_size = cctx->block_size;
    if (!opts) o.checksum_enabled = cctx->checksum;
    return zxc_compress(src, src_size, dst, dst_capacity, &o);
}

int64_t zxc_compress_block(zxc_cctx* cctx, const void* src, size_t src_size, void* dst, size_t dst_capacity,
                           const zxc_compress_opts_t* opts) {
    if (!cctx || !src || !dst || src_size == 0 || dst_capacity == 0) return ZXC_ERROR_NULL_INPUT;
    if (src_size > ZXC_BLOCK_SIZE_MAX) return ZXC_ERROR_BAD_BLOCK_SIZE;
    const int checksum = opts ? opts->checksum_enabled : cctx->checksum;
    const int level = level_clamp((opts && opts->level > 0) ? opts->level : cctx->level);
    const uint8_t* dict = opts ? (const uint8_t*)opts->dict : NULL;
    const size_t dict_size = (opts && opts->dict) ? opts->dict_size : 0;
    if (dict_size > ZXC_DICT_SIZE_MAX) return ZXC_ERROR_DICT_TOO_LARGE;
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    cctx->level = level; /* sticky, like the reference (zxc_dispatch.c:1667-1669) */
    cctx->checksum = checksum;
    if (!cctx->gpu) cctx->gpu = zxg_create();
    if (!cctx->gpu) return ZXC_ERROR_MEMORY;
    uint32_t size = 0;
    uint64_t body = 0;
    /* one frameless block: the same kernel with a single job */
    const int rc = zxg_encode_body(cctx->gpu, (const uint8_t*)src, src_size, (uint32_t)zxf_block_size_ceil(src_size),
                                   level, checksum, 1, (uint8_t*)dst, dst_capacity, &size, &body, dict,
                                   (uint32_t)dict_size, NULL /* the block API attaches no shared table */);
    return rc != ZXC_OK ? rc : (int64_t)body;
}

/* ------------------------------------------------------------------------- */
/* seekable                                                                  */
/* ------------------------------------------------------------------------- */
struct zxc_seekable_s {
    const uint8_t* src; /* borrowed, or NULL in reader mode */
    uint64_t src_size;
    zxc_reader_t reader;
    void* owned_reader_ctx;
    zxw_seek_t tab;
    uint8_t* dict; /* owned copy */
    size_t dict_size;
    uint8_t dict_huf[ZXC_HUF_TABLE_SIZE];
    int has_dict_huf;
    zxg_ctx* gpu;
    zxc_b200_job_t* jobs_buf; /* job and status tables of the last range call, kept: a million-block range would */
    int32_t* st_buf;          /* otherwise fault in 28 MB of fresh pages on every call */
    size_t tab_cap;
};

static int seekable_fetch(void* ctx, void* dst, size_t len, uint64_t off) {
    zxc_seekable* s = (zxc_seekable*)ctx;
    if (off > s->src_size || len > s->src_size - off) return ZXC_ERROR_SRC_TOO_SMALL;
    if (s->src) {
        memcpy(dst, s->src + off, len);
        return ZXC_OK;
    }
    const int64_t r = s->reader.read_at(s->reader.ctx, dst, len, off);
    if (r != (int64_t)len) return r < 0 ? (int)r : ZXC_ERROR_IO;
    return ZXC_OK;
}

static zxc_seekable* seekable_new(const uint8_t* src, uint64_t size, const zxc_reader_t* r) {
    zxc_seekable* s = (zxc_seekable*)calloc(1, sizeof *s);
    if (!s) return NULL;
    s->src = src;
    s->src_size = size;
    if (r) s->reader = *r;
    if (zxw_seek_parse(seekable_fetch, s, size, &s->tab) != ZXC_OK) {
        free(s);
        return NULL;
    }
    return s;
}

zxc_seekable* zxc_seekable_open(const void* src, const size_t src_size) {
    if (!src || src_size == 0) return NULL;
    return seekable_new((const uint8_t*)src, src_size, NULL);
}

zxc_seekable* zxc_seekable_open_reader(const zxc_reader_t* r) {
    if (!r || !r->read_at || r->size == 0) return NULL;
    return seekable_new(NULL, r->size, r);
}

void zxc_seekable_free(zxc_seekable* s) {
    if (!s) return;
    if (s->gpu) zxg_destroy(s->gpu);
    zxw_seek_free(&s->tab);
    free(s->jobs_buf);
    free(s->st_buf);
    free(s->dict);
    free(s->owned_reader_ctx);
    free(s);
}

uint32_t zxc_seekable_get_num_blocks(const zxc_seekable* s) { return s ? s->tab.num_blocks : 0; }
uint64_t zxc_seekable_get_decompressed_size(const zxc_seekable* s) { return s ? s->tab.total : 0; }
uint32_t zxc_seekable_get_block_comp_size(const zxc_seekable* s, const uint32_t i) {
    return (s && i < s->tab.num_blocks) ? s->tab.comp_sizes[i] : 0;
}
uint32_t zxc_seekable_get_block_decomp_size(const zxc_seekable* s, const uint32_t i) {
    return (s && i < s->tab.num_blocks) ? expected_block_bytes(s->tab.total, s->tab.block_size, i) : 0;
}

/* zxc_seekable.c:1144-1174: arguments are validated before the installed dictionary is touched, so a
 * rejected call (NULL / empty, too large, id mismatch) leaves the handle as it was. */
int zxc_seekable_set_dict(zxc_seekable* s, const void* dict, size_t dict_size, const void* dict_huf) {
    if (!s || !dict || dict_size == 0) return ZXC_ERROR_NULL_INPUT;
    if (dict_size > ZXC_DICT_SIZE_MAX) return ZXC_ERROR_DICT_TOO_LARGE;
    if (s->tab.dict_id != 0 && zxc_dict_id(dict, dict_size, dict_huf) != s->tab.dict_id)
        return ZXC_ERROR_DICT_MISMATCH;
    uint8_t* copy = (uint8_t*)malloc(dict_size);
    if (!copy) {
        free(s->dict); /* the reference drops the old dictionary before it allocates (:1152-1158) */
        s->dict = NULL;
        s->dict_size = 0;
        s->has_dict_huf = 0;
        return ZXC_ERROR_MEMORY;
    }
    memcpy(copy, dict, dict_size);
    free(s->dict);
    s->dict = copy;
    s->dict_size = dict_size;
    s->has_dict_huf = 0;
    if (dict_huf) {
        memcpy(s->dict_huf, dict_huf, ZXC_HUF_TABLE_SIZE);
        s->has_dict_huf = 1;
    }
    return ZXC_OK;
}

static int64_t seekable_range(zxc_seekable* s, void* dst, size_t dst_capacity, uint64_t offset, size_t len) {
    if (len == 0) return 0;
    if (!s || !dst) return ZXC_ERROR_NULL_INPUT;
    if (dst_capacity < len) return ZXC_ERROR_DST_TOO_SMALL;
    if (offset + len > s->tab.total || offset + len < offset) return ZXC_ERROR_SRC_TOO_SMALL;
    if (s->tab.dict_id != 0 && (!s->dict || s->dict_size == 0)) return ZXC_ERROR_DICT_REQUIRED;
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    if (!s->gpu) s->gpu = zxg_create();
    zxg_ctx* g = s->gpu;
    if (!g) return ZXC_ERROR_MEMORY;

    const uint32_t bs = s->tab.block_size;
    const uint32_t b0 = (uint32_t)(offset / bs), b1 = (uint32_t)((offset + len - 1) / bs);
    const uint32_t nb = b1 - b0 + 1;
    const uint64_t c_hi = s->tab.comp_offsets[b1 + 1];
    const uint64_t out_lo = (uint64_t)b0 * bs;

    if (nb > s->tab_cap) {
        free(s->jobs_buf);
        free(s->st_buf);
        s->jobs_buf = (zxc_b200_job_t*)malloc((size_t)nb * sizeof *s->jobs_buf);
        s->st_buf = (int32_t*)malloc((size_t)nb * sizeof *s->st_buf);
        s->tab_cap = (s->jobs_buf && s->st_buf) ? nb : 0;
        if (!s->tab_cap) {
            free(s->jobs_buf);
            free(s->st_buf);
            s->jobs_buf = NULL;
            s->st_buf = NULL;
            return ZXC_ERROR_MEMORY;
        }
    }
    zxc_b200_job_t* jobs = s->jobs_buf;
    int32_t* st = s->st_buf;
    for (uint32_t i = 0; i < nb; i++) { /* source offsets in the frame; decoded ones from the first covered block */
        jobs[i].src_off = s->tab.comp_offsets[b0 + i];
        jobs[i].src_len = s->tab.comp_sizes[b0 + i];
        jobs[i].dst_off = (uint64_t)i * bs;
        jobs[i].dst_cap = expected_block_bytes(s->tab.total, bs, b0 + i);
    }
    if (s->src && c_hi > s->src_size) return ZXC_ERROR_SRC_TOO_SMALL;
    const uint64_t clip_lo = offset - out_lo;
    /* checksums are never verified on the seekable path (zxc_seekable.c:707, :909) */
    const int rc = decode_to_host(g, s->src, s->src ? NULL : seekable_fetch, s, (uint8_t*)dst, clip_lo, clip_lo + len,
                                  jobs, nb, st, s->dict, (uint32_t)s->dict_size, s->has_dict_huf ? s->dict_huf : NULL,
                                  bs, 0, 1);
    if (rc != ZXC_OK) return rc;
    int mismatch = 0;
    const int64_t ff = first_failure(st, jobs, nb, &mismatch);
    return ff < 0 ? ff : (int64_t)len;
}

int64_t zxc_seekable_decompress_range(zxc_seekable* s, void* dst, const size_t dst_capacity, const uint64_t offset,
                                      const size_t len) {
    return seekable_range(s, dst, dst_capacity, offset, len);
}

int64_t zxc_seekable_decompress_range_mt(zxc_seekable* s, void* dst, const size_t dst_capacity,
                                         const uint64_t offset, const size_t len, int n_threads) {
    (void)n_threads; /* the fan-out is the GPU launch: one warp per covered block */
    return seekable_range(s, dst, dst_capacity, offset, len);
}

size_t zxc_seek_table_size(const uint32_t num_blocks) {
    return (size_t)ZXF_BLOCK_HDR + (size_t)num_blocks * ZXF_SEEK_ENTRY;
}

int64_t zxc_write_seek_table(uint8_t* dst, const size_t dst_capacity, const uint32_t* comp_sizes,
                             const uint32_t num_blocks) {
    if (num_blocks > UINT32_MAX / ZXF_SEEK_ENTRY) return ZXC_ERROR_OVERFLOW;
    const size_t total = zxc_seek_table_size(num_blocks);
    if (dst_capacity < total) return ZXC_ERROR_DST_TOO_SMALL;
    if (!dst || !comp_sizes) return ZXC_ERROR_NULL_INPUT;
    seek_table_header(dst, num_blocks);
    for (uint32_t i = 0; i < num_blocks; i++) zxf_st32(dst + ZXF_BLOCK_HDR + 4 * (size_t)i, comp_sizes[i]);
    return (int64_t)total;
}

/* ------------------------------------------------------------------------- */
/* FILE* helpers: thin host readers around the buffer API.                  */
/* (push streaming, zxc_cstream_* / zxc_dstream_*, is in zxc_pstream.c)     */
/* ------------------------------------------------------------------------- */
static uint8_t* slurp(FILE* f, size_t* n_out) {
    size_t cap = 1 << 20, n = 0;
    uint8_t* b = (uint8_t*)malloc(cap);
    if (!b) return NULL;
    for (;;) {
        if (n == cap) {
            cap *= 2;
            uint8_t* nb = (uint8_t*)realloc(b, cap);
            if (!nb) { free(b); return NULL; }
            b = nb;
        }
        const size_t r = fread(b + n, 1, cap - n, f);
        n += r;
        if (r == 0) break;
    }
    *n_out = n;
    return b;
}

int64_t zxc_stream_decompress(FILE* f_in, FILE* f_out, const zxc_decompress_opts_t* opts) {
    if (!f_in) return ZXC_ERROR_NULL_INPUT;
    size_t n = 0;
    uint8_t* in = slurp(f_in, &n);
    if (!in) return ZXC_ERROR_MEMORY;
    if (ferror(f_in)) { free(in); return ZXC_ERROR_IO; }
    int64_t r;
    if (n < ZXC_FILE_HEADER_SIZE + ZXC_FILE_FOOTER_SIZE) { free(in); return ZXC_ERROR_SRC_TOO_SMALL; }
    zxf_file_header_t fh;
    r = zxf_read_file_header(in, n, &fh, 1);
    if (r != ZXC_OK) { free(in); return r; }
    const uint64_t d = zxf_le64(in + n - ZXC_FILE_FOOTER_SIZE);
    if (!zxf_dsize_plausible(d, fh.block_size, n)) { free(in); return ZXC_ERROR_CORRUPT_DATA; }
    uint8_t* out = (uint8_t*)malloc(d ? (size_t)d : 1);
    if (!out) { free(in); return ZXC_ERROR_MEMORY; }
    r = zxc_decompress(in, n, d ? out : NULL, (size_t)d, opts);
    if (r > 0 && f_out && fwrite(out, 1, (size_t)r, f_out) != (size_t)r) r = ZXC_ERROR_IO;
    free(out);
    free(in);
    return r;
}

int64_t zxc_stream_get_decompressed_size(FILE* f_in) {
    if (!f_in) return ZXC_ERROR_NULL_INPUT;
    const long pos = ftell(f_in);
    uint8_t hdr[ZXC_FILE_HEADER_SIZE], ftr[ZXC_FILE_FOOTER_SIZE];
    if (fseek(f_in, 0, SEEK_END) != 0) return ZXC_ERROR_IO;
    const long size = ftell(f_in);
    int64_t r = ZXC_ERROR_IO;
    if (size >= (long)(ZXC_FILE_HEADER_SIZE + ZXC_FILE_FOOTER_SIZE) && fseek(f_in, 0, SEEK_SET) == 0 &&
        fread(hdr, 1, sizeof hdr, f_in) == sizeof hdr && fseek(f_in, size - ZXC_FILE_FOOTER_SIZE, SEEK_SET) == 0 &&
        fread(ftr, 1, sizeof ftr, f_in) == sizeof ftr) {
        zxf_file_header_t fh;
        const int hrc = zxf_read_file_header(hdr, sizeof hdr, &fh, 1);
        r = hrc != ZXC_OK ? hrc : (int64_t)zxf_le64(ftr);
    } else if (size >= 0 && size < (long)(ZXC_FILE_HEADER_SIZE + ZXC_FILE_FOOTER_SIZE)) {
        r = ZXC_ERROR_SRC_TOO_SMALL;
    }
    if (pos >= 0) fseek(f_in, pos, SEEK_SET);
    return r;
}

/* positioned reads like the reference's FILE* reader (zxc_seekable.c:414-421: pread, safe from several threads); a
 * stream without a descriptor (fmemopen) falls back to fseek + fread under a lock */
static pthread_mutex_t g_file_mu = PTHREAD_MUTEX_INITIALIZER;
static int64_t file_read_at(void* ctx, void* dst, size_t len, uint64_t offset) {
    FILE* f = (FILE*)((void**)ctx)[0];
    const int fd = fileno(f);
    if (fd >= 0) {
        size_t got = 0;
        while (got < len) {
            const ssize_t r = pread(fd, (uint8_t*)dst + got, len - got, (off_t)(offset + got));
            if (r < 0) return ZXC_ERROR_IO;
            if (r == 0) break;
            got += (size_t)r;
        }
        return (int64_t)got;
    }
    pthread_mutex_lock(&g_file_mu);
    int64_t r = ZXC_ERROR_IO;
    if (fseek(f, (long)offset, SEEK_SET) == 0) r = (int64_t)fread(dst, 1, len, f);
    pthread_mutex_unlock(&g_file_mu);
    return r;
}

zxc_seekable* zxc_seekable_open_file(FILE* f) {
    if (!f) return NULL;
    if (fseek(f, 0, SEEK_END) != 0) return NULL;
    const long size = ftell(f);
    if (size <= 0) return NULL;
    void** rc = (void**)malloc(sizeof(void*));
    if (!rc) return NULL;
    rc[0] = f;
    zxc_reader_t r = {file_read_at, rc, (uint64_t)size};
    zxc_seekable* s = seekable_new(NULL, (uint64_t)size, &r);
    if (!s) { free(rc); return NULL; }
    s->owned_reader_ctx = rc;
    return s;
}

/* FILE* -> FILE* compression (reference src/lib/zxc_driver.c:1035-1056).  The reference's streaming
 * engine emits exactly the frame zxc_compress emits for the same options (checked in
 * tests/test_encode_gpu.py), so the host side reads the input, runs the GPU frame encoder once and
 * writes the result; f_out == NULL is the reference's dry run (size only). */
int64_t zxc_stream_compress(FILE* f_in, FILE* f_out, const zxc_compress_opts_t* opts) {
    if (!f_in) return ZXC_ERROR_NULL_INPUT;
    const size_t block_size = (opts && opts->block_size) ? opts->block_size : ZXC_BLOCK_SIZE_DEFAULT;
    if (!zxf_valid_block_size(block_size)) return ZXC_ERROR_BAD_BLOCK_SIZE;
    if (opts && opts->dict && opts->dict_size > ZXC_DICT_SIZE_MAX) return ZXC_ERROR_DICT_TOO_LARGE;
    size_t n = 0;
    uint8_t* in = slurp(f_in, &n);
    if (!in) return ZXC_ERROR_MEMORY;
    if (ferror(f_in)) { free(in); return ZXC_ERROR_IO; }
    /* blocks are block_size long, so the frame bound follows the caller's block size, not the default */
    const uint64_t nb = (n + block_size - 1) / block_size;
    const size_t cap = (size_t)(n + nb * (ZXF_BLOCK_HDR + ZXF_BLOCK_CKS + 64) + zxc_seek_table_size((uint32_t)(nb ? nb : 1)) + 256);
    uint8_t* out = (uint8_t*)malloc(cap);
    if (!out) { free(in); return ZXC_ERROR_MEMORY; }
    int64_t r = zxc_compress(in, n, out, cap, opts);
    if (r > 0 && f_out && fwrite(out, 1, (size_t)r, f_out) != (size_t)r) r = ZXC_ERROR_IO;
    free(out);
    free(in);
    return r;
}
