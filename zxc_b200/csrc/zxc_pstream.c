/*
 * zxc_pstream.c -- push streaming (include/zxc_pstream.h) over the GPU block codec.
 *
 * Both directions run the reference's state machine (src/lib/zxc_pstream.c) on the host for everything that is not
 * a block payload: file header, block headers, EOF, SEK skip, footer, and the partial accumulators carried between
 * calls.  Only the per-block work differs.  The reference encodes or decodes one block per state-machine step; here
 * a step that needs a block first looks ahead for every whole block the call can reach, runs them through one
 * zxg_encode_body / zxg_decode_jobs call (one launch), and the state machine then takes the results one block at a
 * time in stream order, exactly as the reference would have produced them.  Where the reference stops (out full,
 * a block's error), the remaining results of the batch are dropped and their input is not consumed: a later call
 * sees the same bytes again.  DESIGN.md section 7f has the batch-size rule and the waste bound.
 *
 * Each stream owns one zxg_ctx, created on the first call that has to encode or decode a block, on the device that
 * is current then; later calls switch to that device around their GPU work and back.
 */
#include <stdlib.h>
#include <string.h>

#include "zxc.h"
#include "zxc_format.h"
#include "zxc_gpu.h"

/* a batch never covers more than this many uncompressed bytes */
#define PS_BATCH_BYTES ((size_t)64 << 20)

/* ------------------------------------------------------------------------- */
/* the stream's device context                                               */
/* ------------------------------------------------------------------------- */
typedef struct {
    zxg_ctx* g;
    int device;
} ps_gpu;

/* Makes the stream's context usable: created on first use on the current device, else its device made current.
 * *prev receives the device to restore with ps_gpu_leave. */
static int ps_gpu_enter(ps_gpu* s, int* prev) {
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    *prev = zxg_current_device();
    if (!s->g) {
        s->g = zxg_create();
        if (!s->g) return ZXC_ERROR_MEMORY;
        s->device = *prev;
        return ZXC_OK;
    }
    return s->device == *prev ? ZXC_OK : zxg_set_device(s->device);
}

static void ps_gpu_leave(const ps_gpu* s, int prev) {
    if (s->device != prev) zxg_set_device(prev);
}

/* grows a host buffer to at least `need` bytes (contents kept) */
static int ps_grow(void** p, size_t* cap, size_t need) {
    if (*cap >= need) return ZXC_OK;
    const size_t want = need + (need >> 3);
    void* n = realloc(*p, want);
    if (!n) return ZXC_ERROR_MEMORY;
    *p = n;
    *cap = want;
    return ZXC_OK;
}

static size_t ps_min(size_t a, size_t b) { return a < b ? a : b; }

/* ========================================================================= */
/* compression                                                               */
/* ========================================================================= */
typedef enum {
    CS_INIT = 0,
    CS_DRAIN_HEADER,
    CS_ACCUMULATE,
    CS_DRAIN_BLOCK,
    CS_DRAIN_LAST,
    CS_DRAIN_EOF,
    CS_DRAIN_FOOTER,
    CS_DONE,
    CS_ERRORED
} cs_state_t;

struct zxc_cstream_s {
    int level, checksum;
    size_t block_size;
    ps_gpu gpu;
    uint8_t* acc; /* a partial block carried between calls */
    size_t acc_used;
    uint8_t fixed[ZXC_FILE_HEADER_SIZE]; /* file header, EOF block or footer being drained */
    const uint8_t* pending;              /* `fixed`, or one encoded block inside `body` */
    size_t pending_len, pending_pos;
    uint64_t total_in;
    uint32_t global_hash;
    cs_state_t state;
    int error_code;
    /* the current batch: blocks encoded by one launch, taken one at a time */
    uint8_t* stage; /* gathered input when the accumulator heads a batch */
    size_t stage_cap;
    uint8_t* body; /* encoded blocks back to back */
    size_t body_cap;
    uint32_t* sizes;
    size_t sizes_cap;
    uint64_t batch_src; /* input bytes of the batch */
    uint32_t batch_n, batch_i;
    uint64_t batch_off; /* offset of block batch_i in body */
    size_t want;        /* blocks the next batch of this call may cover (0: none run yet in this call) */
};

static int cs_set_error(zxc_cstream* cs, int code) {
    cs->error_code = code;
    cs->state = CS_ERRORED;
    return code;
}

static int level_of(int level) {
    return level <= 0 ? ZXC_LEVEL_DEFAULT : (level > ZXC_LEVEL_ULTRA ? ZXC_LEVEL_ULTRA : level);
}

zxc_cstream* zxc_cstream_create(const zxc_compress_opts_t* opts) {
    /* the reference's checks: no dictionary (the stream's header carries no dictionary id), then the block size its
     * zxc_create_cctx accepts; seekable, n_threads and the progress callback are ignored */
    if (opts && (opts->dict || opts->dict_size || opts->dict_huf)) return NULL;
    const size_t bs = (opts && opts->block_size) ? opts->block_size : ZXC_BLOCK_SIZE_DEFAULT;
    if (!zxf_valid_block_size(bs)) return NULL;
    zxc_cstream* cs = (zxc_cstream*)calloc(1, sizeof *cs);
    if (!cs) return NULL;
    cs->level = level_of(opts ? opts->level : 0);
    cs->checksum = opts ? opts->checksum_enabled : 0;
    cs->block_size = bs;
    cs->acc = (uint8_t*)malloc(bs);
    if (!cs->acc) {
        free(cs);
        return NULL;
    }
    cs->state = CS_INIT;
    return cs;
}

void zxc_cstream_free(zxc_cstream* cs) {
    if (!cs) return;
    if (cs->gpu.g) zxg_destroy(cs->gpu.g);
    free(cs->acc);
    free(cs->stage);
    free(cs->body);
    free(cs->sizes);
    free(cs);
}

size_t zxc_cstream_in_size(const zxc_cstream* cs) { return cs ? cs->block_size : 0; }

size_t zxc_cstream_out_size(const zxc_cstream* cs) {
    if (!cs) return 0;
    const uint64_t b = zxc_compress_block_bound(cs->block_size);
    return (b == 0 || b > SIZE_MAX) ? cs->block_size : (size_t)b;
}

static void cs_stage_fixed(zxc_cstream* cs, size_t len) {
    cs->pending = cs->fixed;
    cs->pending_len = len;
    cs->pending_pos = 0;
}

static int cs_drain(zxc_cstream* cs, zxc_outbuf_t* out) {
    const size_t n = ps_min(out->size - out->pos, cs->pending_len - cs->pending_pos);
    if (n) {
        memcpy((uint8_t*)out->dst + out->pos, cs->pending + cs->pending_pos, n);
        out->pos += n;
        cs->pending_pos += n;
    }
    return cs->pending_pos == cs->pending_len;
}

/* Encodes n_blocks blocks of src (src_size bytes, every block block_size long but the last) in one launch; the
 * results are taken with cs_take. */
static int cs_encode(zxc_cstream* cs, const uint8_t* src, uint64_t src_size, uint32_t n_blocks) {
    int prev = 0;
    int rc = ps_gpu_enter(&cs->gpu, &prev);
    if (rc != ZXC_OK) return rc;
    const uint64_t cap = (uint64_t)n_blocks * zxc_compress_block_bound(cs->block_size);
    rc = ps_grow((void**)&cs->body, &cs->body_cap, (size_t)cap);
    if (rc == ZXC_OK) rc = ps_grow((void**)&cs->sizes, &cs->sizes_cap, (size_t)n_blocks * sizeof *cs->sizes);
    uint64_t body = 0;
    if (rc == ZXC_OK)
        rc = zxg_encode_body(cs->gpu.g, src, src_size, (uint32_t)cs->block_size, cs->level, cs->checksum, n_blocks,
                             cs->body, cap, cs->sizes, &body, NULL, 0, NULL);
    ps_gpu_leave(&cs->gpu, prev);
    if (rc != ZXC_OK) return rc;
    cs->batch_src = src_size;
    cs->batch_n = n_blocks;
    cs->batch_i = 0;
    cs->batch_off = 0;
    return ZXC_OK;
}

/* The next block of the batch becomes the pending output, with the reference's bookkeeping (cs_compress_block_from):
 * input total, and the block's checksum trailer folded into the global hash. */
static void cs_take(zxc_cstream* cs) {
    const uint32_t i = cs->batch_i;
    const uint64_t lo = (uint64_t)i * cs->block_size;
    const uint64_t len = cs->batch_src - lo < cs->block_size ? cs->batch_src - lo : cs->block_size;
    const size_t csize = cs->sizes[i];
    cs->pending = cs->body + cs->batch_off;
    cs->pending_len = csize;
    cs->pending_pos = 0;
    cs->total_in += len;
    if (cs->checksum && csize >= ZXF_BLOCK_CKS)
        cs->global_hash = zxf_hash_combine(cs->global_hash, zxf_le32(cs->pending + csize - ZXF_BLOCK_CKS));
    cs->batch_off += csize;
    cs->batch_i++;
}

/* Blocks the next batch may cover: enough to fill the caller's room if every block reached its bound, doubled for
 * every further batch in the same call, never more than PS_BATCH_BYTES of input. */
static size_t cs_batch_blocks(zxc_cstream* cs, const zxc_outbuf_t* out) {
    if (cs->want == 0)
        cs->want = (out->size - out->pos) / zxc_compress_block_bound(cs->block_size) + 1;
    else
        cs->want *= 2;
    const size_t cap = PS_BATCH_BYTES / cs->block_size ? PS_BATCH_BYTES / cs->block_size : 1;
    if (cs->want > cap) cs->want = cap;
    return cs->want;
}

/* A full accumulator, then every whole block waiting in `in`, as one batch (the accumulator is copied ahead of
 * them so that the batch is one contiguous input). */
static int cs_encode_from_acc(zxc_cstream* cs, const zxc_outbuf_t* out, const zxc_inbuf_t* in) {
    const size_t bs = cs->block_size;
    const size_t k = ps_min(1 + (in->size - in->pos) / bs, cs_batch_blocks(cs, out));
    if (k == 1) return cs_encode(cs, cs->acc, bs, 1);
    const int rc = ps_grow((void**)&cs->stage, &cs->stage_cap, k * bs);
    if (rc != ZXC_OK) return rc;
    memcpy(cs->stage, cs->acc, bs);
    memcpy(cs->stage + bs, (const uint8_t*)in->src + in->pos, (k - 1) * bs);
    return cs_encode(cs, cs->stage, (uint64_t)k * bs, (uint32_t)k);
}

int64_t zxc_cstream_compress(zxc_cstream* cs, zxc_outbuf_t* out, zxc_inbuf_t* in) {
    if (!cs || !out || !in || in->pos > in->size || out->pos > out->size || (in->size > in->pos && !in->src) ||
        (out->size > out->pos && !out->dst) || cs->state == CS_DONE)
        return ZXC_ERROR_NULL_INPUT;
    if (cs->state == CS_ERRORED) return cs->error_code;
    /* a batch lives within one call: the caller's buffers may change between calls */
    cs->batch_n = cs->batch_i = 0;
    cs->want = 0;
    const size_t bs = cs->block_size;
    for (;;) {
        switch (cs->state) {
            case CS_INIT:
                cs_stage_fixed(cs, (size_t)zxf_write_file_header(cs->fixed, sizeof cs->fixed, bs, cs->checksum, 0));
                cs->state = CS_DRAIN_HEADER;
                break;
            case CS_DRAIN_HEADER:
            case CS_DRAIN_BLOCK:
                if (!cs_drain(cs, out)) return (int64_t)(cs->pending_len - cs->pending_pos);
                cs->state = CS_ACCUMULATE;
                break;
            case CS_ACCUMULATE: {
                const size_t avail = in->size - in->pos;
                if (cs->acc_used == 0 && avail >= bs) {
                    /* a whole block straight from `in`: the next one of the batch, or the head of a new one */
                    if (cs->batch_i == cs->batch_n) {
                        const size_t k = ps_min(avail / bs, cs_batch_blocks(cs, out));
                        const int rc = cs_encode(cs, (const uint8_t*)in->src + in->pos, (uint64_t)k * bs, (uint32_t)k);
                        if (rc != ZXC_OK) return cs_set_error(cs, rc);
                    }
                    cs_take(cs);
                    in->pos += bs;
                    cs->state = CS_DRAIN_BLOCK;
                    break;
                }
                const size_t n = ps_min(avail, bs - cs->acc_used);
                if (n) {
                    memcpy(cs->acc + cs->acc_used, (const uint8_t*)in->src + in->pos, n);
                    in->pos += n;
                    cs->acc_used += n;
                }
                if (cs->acc_used == bs) {
                    const int rc = cs_encode_from_acc(cs, out, in);
                    if (rc != ZXC_OK) return cs_set_error(cs, rc);
                    cs_take(cs);
                    cs->acc_used = 0;
                    cs->state = CS_DRAIN_BLOCK;
                    break;
                }
                return 0;
            }
            case CS_DRAIN_LAST:
            case CS_DRAIN_EOF:
            case CS_DRAIN_FOOTER:
            case CS_DONE:
            case CS_ERRORED:
                return ZXC_ERROR_NULL_INPUT; /* states of zxc_cstream_end */
        }
    }
}

int64_t zxc_cstream_end(zxc_cstream* cs, zxc_outbuf_t* out) {
    if (!cs || !out || cs->state == CS_DONE) return ZXC_ERROR_NULL_INPUT;
    if (cs->state == CS_ERRORED) return cs->error_code;
    cs->batch_n = cs->batch_i = 0;
    for (;;) {
        switch (cs->state) {
            case CS_INIT:
                cs_stage_fixed(cs, (size_t)zxf_write_file_header(cs->fixed, sizeof cs->fixed, cs->block_size,
                                                                 cs->checksum, 0));
                cs->state = CS_DRAIN_HEADER;
                break;
            case CS_DRAIN_HEADER:
            case CS_DRAIN_BLOCK:
                if (!cs_drain(cs, out)) return (int64_t)(cs->pending_len - cs->pending_pos);
                cs->state = CS_ACCUMULATE;
                break;
            case CS_ACCUMULATE:
                if (cs->acc_used > 0) { /* the short last block, encoded at the stream's block size */
                    const int rc = cs_encode(cs, cs->acc, cs->acc_used, 1);
                    if (rc != ZXC_OK) return cs_set_error(cs, rc);
                    cs_take(cs);
                    cs->acc_used = 0;
                    cs->state = CS_DRAIN_LAST;
                    break;
                }
                cs_stage_fixed(cs, (size_t)zxf_write_block_header(cs->fixed, sizeof cs->fixed, ZXF_BT_EOF, 0));
                cs->state = CS_DRAIN_EOF;
                break;
            case CS_DRAIN_LAST:
                if (!cs_drain(cs, out)) return (int64_t)(cs->pending_len - cs->pending_pos);
                cs_stage_fixed(cs, (size_t)zxf_write_block_header(cs->fixed, sizeof cs->fixed, ZXF_BT_EOF, 0));
                cs->state = CS_DRAIN_EOF;
                break;
            case CS_DRAIN_EOF:
                if (!cs_drain(cs, out)) return (int64_t)(cs->pending_len - cs->pending_pos);
                cs_stage_fixed(cs, (size_t)zxf_write_footer(cs->fixed, sizeof cs->fixed, cs->total_in, cs->global_hash,
                                                            cs->checksum));
                cs->state = CS_DRAIN_FOOTER;
                break;
            case CS_DRAIN_FOOTER:
                if (!cs_drain(cs, out)) return (int64_t)(cs->pending_len - cs->pending_pos);
                cs->state = CS_DONE;
                return 0;
            case CS_DONE:
            case CS_ERRORED:
                return cs->state == CS_ERRORED ? cs->error_code : 0;
        }
    }
}

/* ========================================================================= */
/* decompression                                                             */
/* ========================================================================= */
typedef enum {
    DS_NEED_FILE_HEADER = 0,
    DS_NEED_BLOCK_HEADER,
    DS_NEED_BLOCK_PAYLOAD,
    DS_DECODE_BLOCK,
    DS_EMIT_DECODED,
    DS_PEEK_TAIL,
    DS_DRAIN_SEK_PAYLOAD,
    DS_NEED_FOOTER_FULL,
    DS_NEED_FOOTER_REST,
    DS_VALIDATE_FOOTER,
    DS_DONE,
    DS_ERRORED
} ds_state_t;

struct zxc_dstream_s {
    int checksum_enabled;
    ps_gpu gpu;
    size_t block_size; /* 0 until the file header is parsed */
    int file_has_checksum;
    uint8_t scratch[32]; /* file header, block header, tail peek, footer */
    size_t scratch_used, scratch_need;
    uint8_t* payload; /* the current block: header + payload (+ checksum trailer) */
    size_t payload_cap, payload_used, payload_need;
    size_t decoded_cap;     /* room the decoder gives one block: block_size + tail pad */
    const uint8_t* decoded; /* a decoded block being drained (inside `host_out`) */
    size_t decoded_size, decoded_pos;
    size_t sek_remaining;
    uint64_t total_out;
    uint32_t global_hash;
    ds_state_t state;
    int error_code;
    /* the current batch: decoded by one launch into one slot of decoded_cap bytes each, taken one at a time */
    zxc_b200_job_t* jobs;
    int32_t* st;
    size_t jobs_cap;
    uint8_t* host_out; /* the slots copied back, up to the last one the call takes */
    size_t host_out_cap;
    uint32_t batch_n, batch_i;
};

static int ds_set_error(zxc_dstream* ds, int code) {
    ds->error_code = code;
    ds->state = DS_ERRORED;
    return code;
}

zxc_dstream* zxc_dstream_create(const zxc_decompress_opts_t* opts) {
    if (opts && (opts->dict || opts->dict_size || opts->dict_huf)) return NULL;
    zxc_dstream* ds = (zxc_dstream*)calloc(1, sizeof *ds);
    if (!ds) return NULL;
    ds->checksum_enabled = opts ? opts->checksum_enabled : 0;
    ds->state = DS_NEED_FILE_HEADER;
    ds->scratch_need = ZXC_FILE_HEADER_SIZE;
    return ds;
}

void zxc_dstream_free(zxc_dstream* ds) {
    if (!ds) return;
    if (ds->gpu.g) zxg_destroy(ds->gpu.g);
    free(ds->payload);
    free(ds->jobs);
    free(ds->st);
    free(ds->host_out);
    free(ds);
}

int zxc_dstream_finished(const zxc_dstream* ds) { return (ds && ds->state == DS_DONE) ? 1 : 0; }

size_t zxc_dstream_in_size(const zxc_dstream* ds) {
    if (!ds) return 0;
    if (ds->block_size == 0) return ZXC_BLOCK_SIZE_DEFAULT;
    const uint64_t b = zxc_compress_block_bound(ds->block_size);
    return (b == 0 || b > SIZE_MAX) ? ds->block_size : (size_t)b;
}

size_t zxc_dstream_out_size(const zxc_dstream* ds) {
    if (!ds) return 0;
    return ds->block_size == 0 ? ZXC_BLOCK_SIZE_DEFAULT : ds->block_size;
}

static int ds_pull_scratch(zxc_dstream* ds, zxc_inbuf_t* in) {
    const size_t n = ps_min(ds->scratch_need - ds->scratch_used, in->size - in->pos);
    if (n) {
        memcpy(ds->scratch + ds->scratch_used, (const uint8_t*)in->src + in->pos, n);
        in->pos += n;
        ds->scratch_used += n;
    }
    return ds->scratch_used == ds->scratch_need;
}

static int ds_pull_payload(zxc_dstream* ds, zxc_inbuf_t* in) {
    const size_t n = ps_min(ds->payload_need - ds->payload_used, in->size - in->pos);
    if (n) {
        memcpy(ds->payload + ds->payload_used, (const uint8_t*)in->src + in->pos, n);
        in->pos += n;
        ds->payload_used += n;
    }
    return ds->payload_used == ds->payload_need;
}

static void ds_want_block_header(zxc_dstream* ds) {
    ds->state = DS_NEED_BLOCK_HEADER;
    ds->scratch_used = 0;
    ds->scratch_need = ZXF_BLOCK_HDR;
}

/* The reference's verdict on a block header (ds_handle_need_block_header): ZXC_OK with *need = payload + trailer
 * bytes of a data block, 1 for the EOF block, or the error. */
static int ds_block_header(const zxc_dstream* ds, const uint8_t* hdr, size_t* need) {
    uint8_t type;
    uint32_t comp;
    const int rc = zxf_read_block_header(hdr, ZXF_BLOCK_HDR, &type, &comp);
    if (rc != ZXC_OK) return rc;
    if (type == ZXF_BT_EOF) return comp != 0 ? ZXC_ERROR_BAD_BLOCK_SIZE : 1;
    const uint64_t n = (uint64_t)comp + (ds->file_has_checksum ? ZXF_BLOCK_CKS : 0);
    if (n > zxc_compress_block_bound(ds->block_size)) return ZXC_ERROR_BAD_BLOCK_SIZE;
    *need = (size_t)n;
    return ZXC_OK;
}

/* Decodes the block held in `payload` and the whole data blocks that follow it in `in`, up to the batch size, in one
 * launch.  The decoded slots are copied back up to the last block the caller's room lets this call take. */
static int ds_decode_batch(zxc_dstream* ds, const zxc_outbuf_t* out, const zxc_inbuf_t* in) {
    const size_t bs = ds->block_size, slot = ds->decoded_cap, room = out->size - out->pos;
    /* the reference takes blocks until one no longer fits the room, and that one too; a block yields at most
     * decoded_cap bytes and, unless damaged or hand-made, exactly bs (the last one less) */
    size_t kmax = room / bs + 1;
    const size_t cap = PS_BATCH_BYTES / bs ? PS_BATCH_BYTES / bs : 1;
    if (kmax > cap) kmax = cap;
    const uint8_t* src = (const uint8_t*)in->src;
    size_t p = in->pos, k = 1;
    while (k < kmax && in->size - p >= ZXF_BLOCK_HDR) {
        size_t need = 0;
        if (ds_block_header(ds, src + p, &need) != ZXC_OK) break; /* EOF, or a header the state machine rejects */
        if (in->size - p - ZXF_BLOCK_HDR < need) break;
        p += ZXF_BLOCK_HDR + need;
        k++;
    }
    int rc = ps_grow((void**)&ds->jobs, &ds->jobs_cap, k * sizeof *ds->jobs);
    if (rc != ZXC_OK) return rc;
    void* st = realloc(ds->st, ds->jobs_cap / sizeof *ds->jobs * sizeof *ds->st);
    if (!st) return ZXC_ERROR_MEMORY;
    ds->st = (int32_t*)st;
    /* job table: the held block at 0, then the blocks of `in` in order; output slot i at i * slot */
    uint64_t off = 0;
    size_t q = in->pos;
    for (size_t i = 0; i < k; i++) {
        size_t len = ds->payload_used;
        if (i > 0) {
            size_t need = 0;
            ds_block_header(ds, src + q, &need);
            len = ZXF_BLOCK_HDR + need;
            q += len;
        }
        ds->jobs[i].src_off = off;
        ds->jobs[i].src_len = (uint32_t)len;
        ds->jobs[i].dst_off = (uint64_t)i * slot;
        ds->jobs[i].dst_cap = (uint32_t)slot;
        off += len;
    }
    int prev = 0;
    rc = ps_gpu_enter(&ds->gpu, &prev);
    if (rc != ZXC_OK) return rc;
    zxg_ctx* g = ds->gpu.g;
    uint8_t* d_in = (uint8_t*)zxg_buffer(g, ZXG_BUF_IN, (size_t)off + 16);
    uint8_t* d_out = (uint8_t*)zxg_buffer(g, ZXG_BUF_OUT, k * slot + 16);
    rc = d_in && d_out ? ZXC_OK : ZXC_ERROR_MEMORY;
    if (rc == ZXC_OK) rc = zxg_h2d(g, d_in, ds->payload, ds->payload_used);
    if (rc == ZXC_OK) rc = zxg_h2d(g, d_in + ds->payload_used, src + in->pos, (size_t)off - ds->payload_used);
    if (rc == ZXC_OK)
        rc = zxg_decode_jobs(g, d_in, d_out, ds->jobs, (uint32_t)k, ds->st, NULL, 0, NULL, (uint32_t)bs,
                             ds->file_has_checksum && ds->checksum_enabled);
    if (rc == ZXC_OK) {
        /* the blocks this call will take (see DS_DECODE_BLOCK): up to the first error, or the first block that does
         * not fit what is left of the room */
        size_t m = 0, r = room;
        while (m < k) {
            const int32_t s = ds->st[m++];
            if (s < 0) break;
            if (r < slot && (size_t)s > r) break;
            r -= (size_t)s;
        }
        const int32_t last = ds->st[m - 1];
        const size_t bytes = (m - 1) * slot + (last > 0 ? (size_t)last : 0);
        rc = ps_grow((void**)&ds->host_out, &ds->host_out_cap, bytes ? bytes : 1);
        if (rc == ZXC_OK) rc = zxg_d2h(g, ds->host_out, d_out, bytes);
        if (rc == ZXC_OK) rc = zxg_sync(g);
    }
    ps_gpu_leave(&ds->gpu, prev);
    if (rc != ZXC_OK) return rc;
    ds->batch_n = (uint32_t)k;
    ds->batch_i = 0;
    return ZXC_OK;
}

static int ds_drain(zxc_dstream* ds, zxc_outbuf_t* out, size_t* produced) {
    const size_t n = ps_min(out->size - out->pos, ds->decoded_size - ds->decoded_pos);
    if (n) {
        memcpy((uint8_t*)out->dst + out->pos, ds->decoded + ds->decoded_pos, n);
        out->pos += n;
        ds->decoded_pos += n;
        ds->total_out += n;
        *produced += n;
    }
    return ds->decoded_pos == ds->decoded_size;
}

int64_t zxc_dstream_decompress(zxc_dstream* ds, zxc_outbuf_t* out, zxc_inbuf_t* in) {
    if (!ds || !out || !in || in->pos > in->size || out->pos > out->size || (in->size > in->pos && !in->src) ||
        (out->size > out->pos && !out->dst))
        return ZXC_ERROR_NULL_INPUT;
    if (ds->state == DS_ERRORED) return ds->error_code;
    if (ds->state == DS_DONE) return 0;
    /* a batch lives within one call; a block held for draining (`decoded`) stays valid across calls, since no new
     * batch is decoded before it is drained */
    ds->batch_n = ds->batch_i = 0;
    size_t produced = 0;
    for (;;) {
        switch (ds->state) {
            case DS_NEED_FILE_HEADER: {
                if (!ds_pull_scratch(ds, in)) return (int64_t)produced;
                zxf_file_header_t fh;
                const int rc = zxf_read_file_header(ds->scratch, ds->scratch_used, &fh, 1);
                if (rc != ZXC_OK) return ds_set_error(ds, rc);
                ds->block_size = fh.block_size;
                ds->file_has_checksum = fh.has_checksum;
                /* a block of the largest announced size plus its header (ds_handle_need_block_header grows to this) */
                ds->payload_cap = (size_t)zxc_compress_block_bound(ds->block_size) + ZXF_BLOCK_HDR;
                ds->payload = (uint8_t*)malloc(ds->payload_cap);
                if (!ds->payload) return ds_set_error(ds, ZXC_ERROR_MEMORY);
                ds->decoded_cap = ds->block_size + ZXF_TAIL_PAD;
                ds_want_block_header(ds);
                break;
            }
            case DS_NEED_BLOCK_HEADER: {
                if (!ds_pull_scratch(ds, in)) return (int64_t)produced;
                size_t need = 0;
                const int rc = ds_block_header(ds, ds->scratch, &need);
                if (rc < 0) return ds_set_error(ds, rc);
                if (rc == 1) { /* EOF: a SEK block or the footer follows */
                    ds->state = DS_PEEK_TAIL;
                    ds->scratch_used = 0;
                    ds->scratch_need = ZXF_BLOCK_HDR;
                    break;
                }
                memcpy(ds->payload, ds->scratch, ZXF_BLOCK_HDR);
                ds->payload_used = ZXF_BLOCK_HDR;
                ds->payload_need = need + ZXF_BLOCK_HDR;
                ds->state = DS_NEED_BLOCK_PAYLOAD;
                break;
            }
            case DS_NEED_BLOCK_PAYLOAD:
                if (!ds_pull_payload(ds, in)) return (int64_t)produced;
                ds->state = DS_DECODE_BLOCK;
                break;
            case DS_DECODE_BLOCK: {
                /* the block is the next one of this call's batch (its bytes were pulled from `in` just now), or the
                 * head of a new batch */
                if (ds->batch_i == ds->batch_n) {
                    const int rc = ds_decode_batch(ds, out, in);
                    if (rc != ZXC_OK) return ds_set_error(ds, rc);
                }
                const uint32_t i = ds->batch_i++;
                const int32_t dsz = ds->st[i];
                if (dsz < 0) return ds_set_error(ds, dsz);
                if (ds->checksum_enabled && ds->file_has_checksum && ds->payload_used >= ZXF_BLOCK_CKS)
                    ds->global_hash = zxf_hash_combine(ds->global_hash,
                                                       zxf_le32(ds->payload + ds->payload_used - ZXF_BLOCK_CKS));
                const uint8_t* dec = ds->host_out + (size_t)i * ds->decoded_cap;
                if (out->size - out->pos >= ds->decoded_cap) { /* the reference decodes straight into `out` */
                    memcpy((uint8_t*)out->dst + out->pos, dec, (size_t)dsz);
                    out->pos += (size_t)dsz;
                    produced += (size_t)dsz;
                    ds->total_out += (size_t)dsz;
                    ds->decoded_size = ds->decoded_pos = 0;
                    ds_want_block_header(ds);
                    break;
                }
                ds->decoded = dec;
                ds->decoded_size = (size_t)dsz;
                ds->decoded_pos = 0;
                ds->state = DS_EMIT_DECODED;
                break;
            }
            case DS_EMIT_DECODED:
                if (!ds_drain(ds, out, &produced)) return (int64_t)produced;
                ds_want_block_header(ds);
                break;
            case DS_PEEK_TAIL: {
                if (!ds_pull_scratch(ds, in)) return (int64_t)produced;
                uint8_t type;
                uint32_t comp;
                if (zxf_read_block_header(ds->scratch, ds->scratch_used, &type, &comp) == ZXC_OK && type == ZXF_BT_SEK) {
                    ds->sek_remaining = comp;
                    ds->state = DS_DRAIN_SEK_PAYLOAD;
                    break;
                }
                ds->state = DS_NEED_FOOTER_REST; /* the 8 bytes were the footer's first 8 */
                ds->scratch_need = ZXC_FILE_FOOTER_SIZE;
                break;
            }
            case DS_DRAIN_SEK_PAYLOAD: {
                const size_t n = ps_min(in->size - in->pos, ds->sek_remaining);
                in->pos += n;
                ds->sek_remaining -= n;
                if (ds->sek_remaining > 0) return (int64_t)produced;
                ds->state = DS_NEED_FOOTER_FULL;
                ds->scratch_used = 0;
                ds->scratch_need = ZXC_FILE_FOOTER_SIZE;
                break;
            }
            case DS_NEED_FOOTER_REST:
            case DS_NEED_FOOTER_FULL:
                if (!ds_pull_scratch(ds, in)) return (int64_t)produced;
                ds->state = DS_VALIDATE_FOOTER;
                break;
            case DS_VALIDATE_FOOTER:
                if (zxf_le64(ds->scratch) != ds->total_out) return ds_set_error(ds, ZXC_ERROR_CORRUPT_DATA);
                if (ds->checksum_enabled && ds->file_has_checksum && zxf_le32(ds->scratch + 8) != ds->global_hash)
                    return ds_set_error(ds, ZXC_ERROR_BAD_CHECKSUM);
                ds->state = DS_DONE;
                return (int64_t)produced;
            case DS_DONE:
            case DS_ERRORED:
                return ds->state == DS_ERRORED ? ds->error_code : (int64_t)produced;
        }
    }
}
