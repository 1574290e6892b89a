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
 *
 * The device streams (zxc_b200_cstream_device / _dstream_device, include/zxc_b200.h) are the same two state machines
 * over device-resident chunks: a stream with a `dev` record keeps its blocks in device memory, and the few helpers
 * below that move bytes (ps_out, cs_fill_acc, cs_encode, cs_stage_fixed, ds_pull_scratch, ds_pull_payload,
 * ds_decode_batch, ds_trailer) take the device branch for it.  Copies into `out` are queued as pieces and run as one
 * gather launch before the next batch reuses its slots and at the end of the call (ps_flush).  DESIGN.md section 7l.
 */
#include <stdlib.h>
#include <string.h>

#include "zxc.h"
#include "zxc_format.h"
#include "zxc_gpu.h"

/* a batch never covers more than this many uncompressed bytes */
#define PS_BATCH_BYTES ((size_t)64 << 20)
/* how far past a literal run the decode kernels' loads may reach */
#define PS_READ_PAST 8

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

/* ------------------------------------------------------------------------- */
/* a device stream's record                                                  */
/* ------------------------------------------------------------------------- */
typedef struct {
    void* p;
    size_t cap;
} ps_dbuf;

/* grows a device buffer to at least `need` bytes (contents dropped); the device is idle between calls, and within one
 * a buffer grows only before the work that fills it */
static int ps_dgrow(ps_dbuf* b, size_t need) {
    if (b->cap >= need) return ZXC_OK;
    zxg_dev_free(b->p);
    const size_t want = need + (need >> 3) + 256;
    b->p = zxg_dev_alloc(want);
    b->cap = b->p ? want : 0;
    return b->p ? ZXC_OK : ZXC_ERROR_MEMORY;
}

typedef struct {
    int device;   /* bound at creation */
    void* stream; /* the current call's */
    zxg_psseg_t* segs; /* copies into `out` queued since the last gather */
    size_t segs_cap, n_segs;
    ps_dbuf d_segs, d_counter, d_scratch, d_jobs, d_st, d_in, d_stage, d_walk;
    ps_dbuf d_hold;  /* cstream: the accumulator; dstream: a block pulled across calls (`payload`) */
    ps_dbuf d_fixed; /* cstream: file header, EOF block and footer, one 16-byte slot each */
    /* dstream: the current batch walk's host mirror, valid within one call */
    zxg_psblk_t* mir;
    size_t mir_cap;
    uint32_t mir_n, mir_i;
    size_t mir_base;        /* in->pos the walk started at */
    int hdr_direct;         /* the current block's header was read whole from this call's `in` */
    const uint8_t* blk;     /* device address of the current block's bytes: in `in`, or d_hold */
    uint32_t blk_trailer;   /* its checksum trailer, when `blk_trailer_ok` */
    int blk_trailer_ok;
    uint32_t* trail;        /* the batch's trailers */
    size_t trail_cap;
} ps_dev;

static ps_dev* ps_dev_new(void) {
    if (zxg_init() != ZXC_OK) return NULL;
    ps_dev* d = (ps_dev*)calloc(1, sizeof *d);
    if (d) d->device = zxg_current_device();
    return d;
}

static void ps_dev_free(ps_dev* d) {
    if (!d) return;
    int prev = zxg_current_device();
    if (prev != d->device) zxg_set_device(d->device);
    ps_dbuf* all[] = {&d->d_segs, &d->d_counter, &d->d_scratch, &d->d_jobs, &d->d_st, &d->d_in, &d->d_stage,
                      &d->d_walk, &d->d_hold, &d->d_fixed};
    for (size_t i = 0; i < sizeof all / sizeof *all; i++) zxg_dev_free(all[i]->p);
    if (prev != d->device) zxg_set_device(prev);
    free(d->segs);
    zxg_host_free(d->mir);
    free(d->trail);
    free(d);
}

/* n bytes from src (device, or host when `host`) to out->dst + out->pos: a memcpy for a host stream; a queued copy
 * for a device stream */
static int ps_out(ps_dev* d, const zxc_outbuf_t* out, const uint8_t* src, size_t n) {
    uint8_t* dst = (uint8_t*)out->dst + out->pos;
    if (!d) {
        memcpy(dst, src, n);
        return ZXC_OK;
    }
    const size_t pieces = (n + ZXG_PS_PIECE - 1) / ZXG_PS_PIECE;
    int rc = ps_grow((void**)&d->segs, &d->segs_cap, (d->n_segs + pieces) * sizeof *d->segs);
    if (rc != ZXC_OK) return rc;
    for (size_t o = 0; o < n; o += ZXG_PS_PIECE) {
        zxg_psseg_t* g = &d->segs[d->n_segs++];
        g->src = (uint64_t)(uintptr_t)(src + o);
        g->dst = (uint64_t)(uintptr_t)(dst + o);
        g->len = ps_min(n - o, ZXG_PS_PIECE);
    }
    return ZXC_OK;
}

/* runs the queued copies: one gather launch */
static int ps_flush(ps_dev* d) {
    if (!d || d->n_segs == 0) return ZXC_OK;
    int rc = ps_dgrow(&d->d_segs, d->n_segs * sizeof *d->segs);
    if (rc == ZXC_OK) rc = zxg_ps_gather(d->segs, (uint32_t)d->n_segs, (zxg_psseg_t*)d->d_segs.p, d->stream);
    d->n_segs = 0;
    return rc;
}

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
    ps_dev* dev;        /* a device stream: acc, body and pending are device memory */
};

static int cs_set_error(zxc_cstream* cs, int code) {
    cs->error_code = code;
    cs->state = CS_ERRORED;
    return code;
}

static int level_of(int level) {
    return level <= 0 ? ZXC_LEVEL_DEFAULT : (level > ZXC_LEVEL_ULTRA ? ZXC_LEVEL_ULTRA : level);
}

static zxc_cstream* cs_create(const zxc_compress_opts_t* opts, int device) {
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
    if (device) {
        cs->dev = ps_dev_new();
        if (!cs->dev || ps_dgrow(&cs->dev->d_hold, bs) != ZXC_OK || ps_dgrow(&cs->dev->d_fixed, 64) != ZXC_OK) {
            ps_dev_free(cs->dev);
            free(cs);
            return NULL;
        }
        cs->acc = (uint8_t*)cs->dev->d_hold.p;
    } else {
        cs->acc = (uint8_t*)malloc(bs);
        if (!cs->acc) {
            free(cs);
            return NULL;
        }
    }
    cs->state = CS_INIT;
    return cs;
}

zxc_cstream* zxc_cstream_create(const zxc_compress_opts_t* opts) { return cs_create(opts, 0); }

void zxc_cstream_free(zxc_cstream* cs) {
    if (!cs) return;
    if (cs->gpu.g) zxg_destroy(cs->gpu.g);
    if (cs->dev) { /* acc and body are its device buffers */
        ps_dev_free(cs->dev);
    } else {
        free(cs->acc);
        free(cs->body);
    }
    free(cs->stage);
    free(cs->sizes);
    free(cs);
}

size_t zxc_cstream_in_size(const zxc_cstream* cs) { return cs ? cs->block_size : 0; }

size_t zxc_cstream_out_size(const zxc_cstream* cs) {
    if (!cs) return 0;
    const uint64_t b = zxc_compress_block_bound(cs->block_size);
    return (b == 0 || b > SIZE_MAX) ? cs->block_size : (size_t)b;
}

/* `fixed` (len bytes) becomes the pending output.  A device stream copies it to its own slot of d_fixed (0: file
 * header, 1: EOF block, 2: footer), so that each stays intact until the gather that drains it has run. */
static int cs_stage_fixed(zxc_cstream* cs, size_t len, int slot) {
    cs->pending = cs->fixed;
    if (cs->dev) {
        uint8_t* d = (uint8_t*)cs->dev->d_fixed.p + 16 * slot;
        const int rc = zxg_h2d_async(d, cs->fixed, len, cs->dev->stream);
        if (rc != ZXC_OK) return rc;
        cs->pending = d;
    }
    cs->pending_len = len;
    cs->pending_pos = 0;
    return ZXC_OK;
}

/* 1 when the pending output is drained, 0 when out is full, or the error */
static int cs_drain(zxc_cstream* cs, zxc_outbuf_t* out) {
    const size_t n = ps_min(out->size - out->pos, cs->pending_len - cs->pending_pos);
    if (n) {
        const int rc = ps_out(cs->dev, out, cs->pending + cs->pending_pos, n);
        if (rc != ZXC_OK) return rc;
        out->pos += n;
        cs->pending_pos += n;
    }
    return cs->pending_pos == cs->pending_len;
}

/* n bytes of `in` onto the accumulator */
static int cs_fill_acc(zxc_cstream* cs, zxc_inbuf_t* in, size_t n) {
    const uint8_t* src = (const uint8_t*)in->src + in->pos;
    if (cs->dev) {
        const int rc = zxg_d2d_async(cs->acc + cs->acc_used, src, n, cs->dev->stream);
        if (rc != ZXC_OK) return rc;
    } else {
        memcpy(cs->acc + cs->acc_used, src, n);
    }
    in->pos += n;
    cs->acc_used += n;
    return ZXC_OK;
}

/* The device branch of cs_encode: the batch's bytes (a, then b) copied into a padded buffer, the encode kernels, and
 * the block sizes and trailers back in one copy.  The blocks stay in their staging slots (`body`). */
static int cs_encode_dev(zxc_cstream* cs, const uint8_t* a, size_t alen, const uint8_t* b, size_t blen,
                         uint32_t n_blocks) {
    ps_dev* d = cs->dev;
    const uint32_t bs = (uint32_t)cs->block_size, sstride = zxg_ps_stage_stride(bs);
    /* the queued copies may read the slots this batch overwrites */
    int rc = ps_flush(d);
    if (rc == ZXC_OK) rc = ps_dgrow(&d->d_in, alen + blen + 64);
    if (rc == ZXC_OK) rc = ps_dgrow(&d->d_stage, (size_t)n_blocks * sstride);
    if (rc == ZXC_OK) rc = ps_dgrow(&d->d_st, (size_t)n_blocks * 8);
    if (rc == ZXC_OK) rc = ps_dgrow(&d->d_scratch, zxg_ps_encode_scratch_bytes(n_blocks, bs, cs->level));
    if (rc == ZXC_OK) rc = ps_dgrow(&d->d_counter, 32);
    if (rc == ZXC_OK) rc = ps_grow((void**)&cs->sizes, &cs->sizes_cap, (size_t)n_blocks * 8);
    if (rc != ZXC_OK) return rc;
    uint8_t* in = (uint8_t*)d->d_in.p;
    rc = zxg_d2d_async(in, a, alen, d->stream);
    if (rc == ZXC_OK) rc = zxg_d2d_async(in + alen, b, blen, d->stream);
    if (rc == ZXC_OK) rc = zxg_memset_async(in + alen + blen, 0, 64, d->stream);
    if (rc == ZXC_OK)
        rc = zxg_ps_encode(in, alen + blen, bs, cs->level, cs->checksum, n_blocks, d->d_stage.p, (uint32_t*)d->d_st.p,
                           d->d_scratch.p, (unsigned long long*)d->d_counter.p, cs->sizes, d->stream);
    if (rc != ZXC_OK) return rc;
    cs->body = (uint8_t*)d->d_stage.p;
    return ZXC_OK;
}


/* The host branch of cs_encode: the accumulator is copied ahead of the blocks of `in` so that the batch is one
 * contiguous input, and the encoded body comes back to `body`. */
static int cs_encode_host(zxc_cstream* cs, const uint8_t* a, size_t alen, const uint8_t* b, size_t blen,
                          uint32_t n_blocks) {
    const uint8_t* src = alen ? a : b;
    if (alen && blen) {
        const int rc = ps_grow((void**)&cs->stage, &cs->stage_cap, alen + blen);
        if (rc != ZXC_OK) return rc;
        memcpy(cs->stage, a, alen);
        memcpy(cs->stage + alen, b, blen);
        src = cs->stage;
    }
    int prev = 0;
    int rc = ps_gpu_enter(&cs->gpu, &prev);
    if (rc != ZXC_OK) return rc;
    const uint64_t cap = (uint64_t)n_blocks * zxc_compress_block_bound(cs->block_size);
    rc = ps_grow((void**)&cs->body, &cs->body_cap, (size_t)cap);
    if (rc == ZXC_OK) rc = ps_grow((void**)&cs->sizes, &cs->sizes_cap, (size_t)n_blocks * sizeof *cs->sizes);
    uint64_t body = 0;
    if (rc == ZXC_OK)
        rc = zxg_encode_body(cs->gpu.g, src, alen + blen, (uint32_t)cs->block_size, cs->level, cs->checksum, n_blocks,
                             cs->body, cap, cs->sizes, &body, NULL, 0, NULL);
    ps_gpu_leave(&cs->gpu, prev);
    return rc;
}

/* Encodes n_blocks blocks of a followed by b (alen + blen bytes, every block block_size long but the last) in one
 * launch; the results are taken with cs_take. */
static int cs_encode(zxc_cstream* cs, const uint8_t* a, size_t alen, const uint8_t* b, size_t blen,
                     uint32_t n_blocks) {
    const int rc = cs->dev ? cs_encode_dev(cs, a, alen, b, blen, n_blocks) : cs_encode_host(cs, a, alen, b, blen, n_blocks);
    if (rc != ZXC_OK) return rc;
    cs->batch_src = alen + blen;
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
    /* a device stream's blocks stay in their staging slots, its trailers came back behind the sizes */
    cs->pending = cs->dev ? cs->body + (size_t)i * zxg_ps_stage_stride((uint32_t)cs->block_size)
                          : cs->body + cs->batch_off;
    cs->pending_len = csize;
    cs->pending_pos = 0;
    cs->total_in += len;
    if (cs->checksum && csize >= ZXF_BLOCK_CKS)
        cs->global_hash = zxf_hash_combine(cs->global_hash, cs->dev ? cs->sizes[cs->batch_n + i]
                                                                    : zxf_le32(cs->pending + csize - ZXF_BLOCK_CKS));
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

/* A full accumulator, then every whole block waiting in `in`, as one batch. */
static int cs_encode_from_acc(zxc_cstream* cs, const zxc_outbuf_t* out, const zxc_inbuf_t* in) {
    const size_t bs = cs->block_size;
    const size_t k = ps_min(1 + (in->size - in->pos) / bs, cs_batch_blocks(cs, out));
    return cs_encode(cs, cs->acc, bs, (const uint8_t*)in->src + in->pos, (k - 1) * bs, (uint32_t)k);
}

static int64_t cs_compress(zxc_cstream* cs, zxc_outbuf_t* out, zxc_inbuf_t* in) {
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
            case CS_INIT: {
                const int rc = cs_stage_fixed(
                    cs, (size_t)zxf_write_file_header(cs->fixed, sizeof cs->fixed, bs, cs->checksum, 0), 0);
                if (rc != ZXC_OK) return cs_set_error(cs, rc);
                cs->state = CS_DRAIN_HEADER;
                break;
            }
            case CS_DRAIN_HEADER:
            case CS_DRAIN_BLOCK: {
                const int dr = cs_drain(cs, out);
                if (dr < 0) return cs_set_error(cs, dr);
                if (!dr) return (int64_t)(cs->pending_len - cs->pending_pos);
                cs->state = CS_ACCUMULATE;
                break;
            }
            case CS_ACCUMULATE: {
                const size_t avail = in->size - in->pos;
                if (cs->acc_used == 0 && avail >= bs) {
                    /* a whole block straight from `in`: the next one of the batch, or the head of a new one */
                    if (cs->batch_i == cs->batch_n) {
                        const size_t k = ps_min(avail / bs, cs_batch_blocks(cs, out));
                        const int rc = cs_encode(cs, NULL, 0, (const uint8_t*)in->src + in->pos, k * bs, (uint32_t)k);
                        if (rc != ZXC_OK) return cs_set_error(cs, rc);
                    }
                    cs_take(cs);
                    in->pos += bs;
                    cs->state = CS_DRAIN_BLOCK;
                    break;
                }
                const size_t n = ps_min(avail, bs - cs->acc_used);
                if (n) {
                    const int rc = cs_fill_acc(cs, in, n);
                    if (rc != ZXC_OK) return cs_set_error(cs, rc);
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

int64_t zxc_cstream_compress(zxc_cstream* cs, zxc_outbuf_t* out, zxc_inbuf_t* in) { return cs_compress(cs, out, in); }

static int64_t cs_end(zxc_cstream* cs, zxc_outbuf_t* out) {
    if (!cs || !out || cs->state == CS_DONE) return ZXC_ERROR_NULL_INPUT;
    if (cs->state == CS_ERRORED) return cs->error_code;
    cs->batch_n = cs->batch_i = 0;
    for (;;) {
        int rc = ZXC_OK, dr = 1;
        switch (cs->state) {
            case CS_INIT:
                rc = cs_stage_fixed(cs, (size_t)zxf_write_file_header(cs->fixed, sizeof cs->fixed, cs->block_size,
                                                                      cs->checksum, 0), 0);
                cs->state = CS_DRAIN_HEADER;
                break;
            case CS_DRAIN_HEADER:
            case CS_DRAIN_BLOCK:
                if ((dr = cs_drain(cs, out)) != 1) break;
                cs->state = CS_ACCUMULATE;
                break;
            case CS_ACCUMULATE:
                if (cs->acc_used > 0) { /* the short last block, encoded at the stream's block size */
                    rc = cs_encode(cs, cs->acc, cs->acc_used, NULL, 0, 1);
                    if (rc != ZXC_OK) break;
                    cs_take(cs);
                    cs->acc_used = 0;
                    cs->state = CS_DRAIN_LAST;
                    break;
                }
                rc = cs_stage_fixed(cs, (size_t)zxf_write_block_header(cs->fixed, sizeof cs->fixed, ZXF_BT_EOF, 0), 1);
                cs->state = CS_DRAIN_EOF;
                break;
            case CS_DRAIN_LAST:
                if ((dr = cs_drain(cs, out)) != 1) break;
                rc = cs_stage_fixed(cs, (size_t)zxf_write_block_header(cs->fixed, sizeof cs->fixed, ZXF_BT_EOF, 0), 1);
                cs->state = CS_DRAIN_EOF;
                break;
            case CS_DRAIN_EOF:
                if ((dr = cs_drain(cs, out)) != 1) break;
                rc = cs_stage_fixed(cs, (size_t)zxf_write_footer(cs->fixed, sizeof cs->fixed, cs->total_in,
                                                                 cs->global_hash, cs->checksum), 2);
                cs->state = CS_DRAIN_FOOTER;
                break;
            case CS_DRAIN_FOOTER:
                if ((dr = cs_drain(cs, out)) != 1) break;
                cs->state = CS_DONE;
                return 0;
            case CS_DONE:
            case CS_ERRORED:
                return cs->state == CS_ERRORED ? cs->error_code : 0;
        }
        if (rc != ZXC_OK) return cs_set_error(cs, rc);
        if (dr < 0) return cs_set_error(cs, dr);
        if (dr == 0) return (int64_t)(cs->pending_len - cs->pending_pos);
    }
}

int64_t zxc_cstream_end(zxc_cstream* cs, zxc_outbuf_t* out) { return cs_end(cs, out); }

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
    uint8_t* payload; /* the current block: header + payload (+ checksum trailer); device memory for a device stream */
    size_t payload_cap, payload_used, payload_need;
    size_t decoded_cap;     /* room the decoder gives one block: block_size + tail pad */
    const uint8_t* decoded; /* a decoded block being drained (inside `host_out`, or the device stream's slots) */
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
    ps_dev* dev; /* a device stream */
};

static int ds_set_error(zxc_dstream* ds, int code) {
    ds->error_code = code;
    ds->state = DS_ERRORED;
    return code;
}

static zxc_dstream* ds_create(const zxc_decompress_opts_t* opts, int device) {
    if (opts && (opts->dict || opts->dict_size || opts->dict_huf)) return NULL;
    zxc_dstream* ds = (zxc_dstream*)calloc(1, sizeof *ds);
    if (!ds) return NULL;
    if (device && !(ds->dev = ps_dev_new())) {
        free(ds);
        return NULL;
    }
    ds->checksum_enabled = opts ? opts->checksum_enabled : 0;
    ds->state = DS_NEED_FILE_HEADER;
    ds->scratch_need = ZXC_FILE_HEADER_SIZE;
    return ds;
}

zxc_dstream* zxc_dstream_create(const zxc_decompress_opts_t* opts) { return ds_create(opts, 0); }

void zxc_dstream_free(zxc_dstream* ds) {
    if (!ds) return;
    if (ds->gpu.g) zxg_destroy(ds->gpu.g);
    if (ds->dev) /* payload is its d_hold */
        ps_dev_free(ds->dev);
    else
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

/* Blocks one batch may take: the reference takes blocks until one no longer fits the room, and that one too; a block
 * yields at most decoded_cap bytes and, unless damaged or hand-made, exactly bs (the last one less). */
static size_t ds_batch_blocks(const zxc_dstream* ds, const zxc_outbuf_t* out) {
    const size_t bs = ds->block_size;
    const size_t kmax = (out->size - out->pos) / bs + 1, cap = PS_BATCH_BYTES / bs ? PS_BATCH_BYTES / bs : 1;
    return kmax > cap ? cap : kmax;
}

/* ---- the device stream's batch walk: block headers and trailers of `in`, mirrored on the host ---- */
/* Walks from in->pos for at most max_blocks whole blocks (zxc_ps_walk); the mirror then answers header reads. */
static int ds_walk(zxc_dstream* ds, const zxc_inbuf_t* in, size_t max_blocks) {
    ps_dev* d = ds->dev;
    const size_t bytes = (max_blocks + 1) * sizeof(zxg_psblk_t) + sizeof(uint32_t);
    int rc = ps_dgrow(&d->d_walk, bytes);
    if (rc != ZXC_OK) return rc;
    if (d->mir_cap < bytes) { /* page-locked: the walk's result comes back in one DMA copy */
        zxg_host_free(d->mir);
        d->mir_cap = bytes + (bytes >> 3);
        d->mir = (zxg_psblk_t*)zxg_host_alloc(d->mir_cap);
        if (!d->mir) {
            d->mir_cap = 0;
            return ZXC_ERROR_MEMORY;
        }
    }
    uint32_t n = 0;
    rc = zxg_ps_walk((const uint8_t*)in->src + in->pos, in->size - in->pos, (uint32_t)max_blocks,
                     zxc_compress_block_bound(ds->block_size), ds->file_has_checksum, (zxg_psblk_t*)d->d_walk.p,
                     d->mir, &n, d->stream);
    if (rc != ZXC_OK) return rc;
    d->mir_n = n;
    d->mir_i = 0;
    d->mir_base = in->pos;
    return ZXC_OK;
}

/* the mirror's entry for a header at `pos` of `in`, or NULL */
static const zxg_psblk_t* ds_mirror(ps_dev* d, size_t pos) {
    while (d->mir_i < d->mir_n && d->mir_base + d->mir[d->mir_i].off < pos) d->mir_i++;
    return d->mir_i < d->mir_n && d->mir_base + d->mir[d->mir_i].off == pos ? &d->mir[d->mir_i] : NULL;
}

static int ds_pull_scratch(zxc_dstream* ds, const zxc_outbuf_t* out, zxc_inbuf_t* in) {
    const size_t n = ps_min(ds->scratch_need - ds->scratch_used, in->size - in->pos);
    if (n) {
        const uint8_t* src = (const uint8_t*)in->src + in->pos;
        ps_dev* d = ds->dev;
        if (!d) {
            memcpy(ds->scratch + ds->scratch_used, src, n);
        } else {
            /* a whole block header comes from the batch walk's mirror, run here when it has none for this one (a new
             * batch, or the block after one); anything else -- the file header, pieces cut by a chunk's end, the
             * footer -- is a small copy */
            const int block_hdr = ds->state == DS_NEED_BLOCK_HEADER && ds->scratch_used == 0 && n == ZXF_BLOCK_HDR;
            const zxg_psblk_t* e = block_hdr ? ds_mirror(d, in->pos) : NULL;
            if (block_hdr && (!e || e->len == 0)) {
                const int rc = ds_walk(ds, in, ds_batch_blocks(ds, out));
                if (rc != ZXC_OK) return rc;
                e = ds_mirror(d, in->pos);
            }
            if (e) {
                for (int k = 0; k < ZXF_BLOCK_HDR; k++) ds->scratch[k] = (uint8_t)(e->hdr >> (8 * k));
            } else {
                const int rc = zxg_d2h_sync(ds->scratch + ds->scratch_used, src, n, d->stream);
                if (rc != ZXC_OK) return rc;
            }
            d->hdr_direct = block_hdr;
        }
        in->pos += n;
        ds->scratch_used += n;
    }
    return ds->scratch_used == ds->scratch_need;
}

/* The block's header goes ahead of its payload: copied for a host stream; for a device stream it is needed in device
 * memory only when the block has to be held across calls (ds_pull_payload). */
static void ds_start_block(zxc_dstream* ds, size_t need) {
    if (!ds->dev) memcpy(ds->payload, ds->scratch, ZXF_BLOCK_HDR);
    ds->payload_used = ZXF_BLOCK_HDR;
    ds->payload_need = need + ZXF_BLOCK_HDR;
}

static int ds_pull_payload(zxc_dstream* ds, zxc_inbuf_t* in) {
    const size_t n = ps_min(ds->payload_need - ds->payload_used, in->size - in->pos);
    ps_dev* d = ds->dev;
    if (d && ds->payload_used == ZXF_BLOCK_HDR) {
        d->blk_trailer_ok = 0;
        if (d->hdr_direct && n == ds->payload_need - ZXF_BLOCK_HDR) {
            /* the whole block is in this call's `in`: it is decoded where it lies, and pulling it only consumes it */
            d->blk = (const uint8_t*)in->src + in->pos - ZXF_BLOCK_HDR;
            const zxg_psblk_t* e = ds_mirror(d, in->pos - ZXF_BLOCK_HDR);
            if (e && e->len) {
                d->blk_trailer = e->trailer;
                d->blk_trailer_ok = 1;
            }
            in->pos += n;
            ds->payload_used += n;
            return 1;
        }
        /* held across calls: its header, then its payload as it arrives, into the device's payload buffer */
        d->blk = ds->payload;
        const int rc = zxg_h2d_async(ds->payload, ds->scratch, ZXF_BLOCK_HDR, d->stream);
        if (rc != ZXC_OK) return rc;
    }
    if (n) {
        const uint8_t* src = (const uint8_t*)in->src + in->pos;
        if (d) {
            const int rc = zxg_d2d_async(ds->payload + ds->payload_used, src, n, d->stream);
            if (rc != ZXC_OK) return rc;
        } else {
            memcpy(ds->payload + ds->payload_used, src, n);
        }
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

/* the number of blocks of a batch this call takes (see DS_DECODE_BLOCK): up to the first error, or the first block
 * that does not fit what is left of the room */
static size_t ds_taken(const zxc_dstream* ds, size_t k, size_t room) {
    size_t m = 0, r = room;
    while (m < k) {
        const int32_t s = ds->st[m++];
        if (s < 0) break;
        if (r < ds->decoded_cap && (size_t)s > r) break;
        r -= (size_t)s;
    }
    return m;
}

static int ds_grow_jobs(zxc_dstream* ds, size_t k) {
    const int rc = ps_grow((void**)&ds->jobs, &ds->jobs_cap, k * sizeof *ds->jobs);
    if (rc != ZXC_OK) return rc;
    void* st = realloc(ds->st, ds->jobs_cap / sizeof *ds->jobs * sizeof *ds->st);
    if (!st) return ZXC_ERROR_MEMORY;
    ds->st = (int32_t*)st;
    return ZXC_OK;
}

/* The device branch of ds_decode_batch.  Block 0 is the current block (where it lies in `in`, or held); the whole
 * blocks behind it come from the walk's mirror and are decoded in `in` where they lie, except those that end less
 * than 8 bytes before in->size: the decode kernels' literal loads reach up to 8 bytes past a run, so those are
 * decoded from a copy (with room behind it) in the handle's memory.  The decoded blocks stay in their slots. */
static int ds_decode_batch_dev(zxc_dstream* ds, const zxc_outbuf_t* out, const zxc_inbuf_t* in) {
    ps_dev* d = ds->dev;
    const size_t slot = ds->decoded_cap, kmax = ds_batch_blocks(ds, out);
    /* the copies queued so far may read the slots this batch overwrites */
    int rc = ps_flush(d);
    if (rc != ZXC_OK) return rc;
    if (kmax > 1 && in->size - in->pos >= ZXF_BLOCK_HDR && !ds_mirror(d, in->pos)) {
        rc = ds_walk(ds, in, kmax - 1);
        if (rc != ZXC_OK) return rc;
    }
    /* blocks 1 .. k - 1: the mirror's entries from in->pos on, as far as the host walk would go */
    const zxg_psblk_t* e1 = in->size - in->pos >= ZXF_BLOCK_HDR ? ds_mirror(d, in->pos) : NULL;
    size_t k = 1;
    while (k < kmax && e1 && e1 + (k - 1) < d->mir + d->mir_n) {
        const zxg_psblk_t* e = e1 + (k - 1);
        size_t need = 0;
        if (e->len == 0 || ds_block_header(ds, (const uint8_t*)&e->hdr, &need) != ZXC_OK) break;
        k++;
    }
    rc = ds_grow_jobs(ds, k);
    if (rc == ZXC_OK) rc = ps_grow((void**)&d->trail, &d->trail_cap, k * sizeof *d->trail);
    if (rc != ZXC_OK) return rc;
    const uint8_t* src = (const uint8_t*)in->src;
    size_t lo = SIZE_MAX; /* blocks of `in` from offset lo on are decoded from the copy */
    for (size_t i = 0; i < k; i++) {
        const uint8_t* b = d->blk;
        size_t len = ds->payload_used;
        d->trail[i] = d->blk_trailer;
        if (i > 0) {
            const zxg_psblk_t* e = e1 + (i - 1);
            b = src + d->mir_base + e->off;
            len = e->len;
            d->trail[i] = e->trailer;
        }
        if (b != ds->payload && (size_t)(b - src) + len + PS_READ_PAST > in->size && lo == SIZE_MAX)
            lo = (size_t)(b - src);
        ds->jobs[i].src_off = (uint64_t)(uintptr_t)b;
        ds->jobs[i].src_len = (uint32_t)len;
        ds->jobs[i].dst_off = (uint64_t)i * slot;
        ds->jobs[i].dst_cap = (uint32_t)slot;
    }
    if (lo != SIZE_MAX) { /* the tail of `in` from the first such block, copied with room behind it */
        rc = ps_dgrow(&d->d_in, in->size - lo + 2 * PS_READ_PAST);
        if (rc == ZXC_OK) rc = zxg_d2d_async(d->d_in.p, src + lo, in->size - lo, d->stream);
        if (rc != ZXC_OK) return rc;
        for (size_t i = 0; i < k; i++) {
            const uintptr_t a = (uintptr_t)ds->jobs[i].src_off;
            if (a >= (uintptr_t)(src + lo) && a < (uintptr_t)(src + in->size))
                ds->jobs[i].src_off = (uint64_t)((uintptr_t)d->d_in.p + (a - (uintptr_t)(src + lo)));
        }
    }
    rc = ps_dgrow(&d->d_stage, k * slot + 16);
    if (rc == ZXC_OK) rc = ps_dgrow(&d->d_jobs, k * sizeof *ds->jobs);
    if (rc == ZXC_OK) rc = ps_dgrow(&d->d_st, k * sizeof *ds->st);
    if (rc == ZXC_OK) rc = ps_dgrow(&d->d_scratch, zxg_ps_decode_scratch_bytes((uint32_t)k, (uint32_t)ds->block_size));
    if (rc == ZXC_OK) rc = ps_dgrow(&d->d_counter, 32);
    if (rc != ZXC_OK) return rc;
    rc = zxg_ps_decode(ds->jobs, (uint32_t)k, (zxc_b200_job_t*)d->d_jobs.p, (int32_t*)d->d_st.p, d->d_stage.p,
                       d->d_scratch.p, d->d_scratch.cap, (unsigned long long*)d->d_counter.p,
                       (uint32_t)ds->block_size, ds->file_has_checksum && ds->checksum_enabled, ds->st, d->stream);
    if (rc != ZXC_OK) return rc;
    /* a held block's trailer, when the global hash needs it and the block is taken */
    if (!d->blk_trailer_ok && ds->checksum_enabled && ds->file_has_checksum && ds->payload_used >= ZXF_BLOCK_CKS &&
        ds->st[0] >= 0) {
        uint8_t t[4];
        rc = zxg_d2h_sync(t, d->blk + ds->payload_used - ZXF_BLOCK_CKS, 4, d->stream);
        if (rc != ZXC_OK) return rc;
        d->trail[0] = zxf_le32(t);
    }
    ds->host_out = NULL;
    ds->batch_n = (uint32_t)k;
    ds->batch_i = 0;
    return ZXC_OK;
}

/* Decodes the block held in `payload` and the whole data blocks that follow it in `in`, up to the batch size, in one
 * launch.  The decoded slots are copied back up to the last block the caller's room lets this call take. */
static int ds_decode_batch(zxc_dstream* ds, const zxc_outbuf_t* out, const zxc_inbuf_t* in) {
    if (ds->dev) return ds_decode_batch_dev(ds, out, in);
    const size_t bs = ds->block_size, slot = ds->decoded_cap, room = out->size - out->pos;
    const size_t kmax = ds_batch_blocks(ds, out);
    const uint8_t* src = (const uint8_t*)in->src;
    size_t p = in->pos, k = 1;
    while (k < kmax && in->size - p >= ZXF_BLOCK_HDR) {
        size_t need = 0;
        if (ds_block_header(ds, src + p, &need) != ZXC_OK) break; /* EOF, or a header the state machine rejects */
        if (in->size - p - ZXF_BLOCK_HDR < need) break;
        p += ZXF_BLOCK_HDR + need;
        k++;
    }
    int rc = ds_grow_jobs(ds, k);
    if (rc != ZXC_OK) return rc;
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
        const size_t m = ds_taken(ds, k, room);
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

/* the checksum trailer of block i of the batch (the current block) */
static uint32_t ds_trailer(const zxc_dstream* ds, uint32_t i) {
    return ds->dev ? ds->dev->trail[i] : zxf_le32(ds->payload + ds->payload_used - ZXF_BLOCK_CKS);
}

/* decoded block i of the batch */
static const uint8_t* ds_slot(const zxc_dstream* ds, uint32_t i) {
    return (ds->dev ? (const uint8_t*)ds->dev->d_stage.p : ds->host_out) + (size_t)i * ds->decoded_cap;
}

static int ds_drain(zxc_dstream* ds, zxc_outbuf_t* out, size_t* produced) {
    const size_t n = ps_min(out->size - out->pos, ds->decoded_size - ds->decoded_pos);
    if (n) {
        const int rc = ps_out(ds->dev, out, ds->decoded + ds->decoded_pos, n);
        if (rc != ZXC_OK) return rc;
        out->pos += n;
        ds->decoded_pos += n;
        ds->total_out += n;
        *produced += n;
    }
    return ds->decoded_pos == ds->decoded_size;
}

static int64_t ds_decompress(zxc_dstream* ds, zxc_outbuf_t* out, zxc_inbuf_t* in) {
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
                const int pr = ds_pull_scratch(ds, out, in);
                if (pr < 0) return ds_set_error(ds, pr);
                if (!pr) return (int64_t)produced;
                zxf_file_header_t fh;
                const int rc = zxf_read_file_header(ds->scratch, ds->scratch_used, &fh, 1);
                if (rc != ZXC_OK) return ds_set_error(ds, rc);
                ds->block_size = fh.block_size;
                ds->file_has_checksum = fh.has_checksum;
                /* a block of the largest announced size plus its header (ds_handle_need_block_header grows to this) */
                ds->payload_cap = (size_t)zxc_compress_block_bound(ds->block_size) + ZXF_BLOCK_HDR;
                if (ds->dev) { /* with room behind it for the decode kernels' read-past */
                    ds->payload = ps_dgrow(&ds->dev->d_hold, ds->payload_cap + 16) == ZXC_OK
                                      ? (uint8_t*)ds->dev->d_hold.p : NULL;
                } else {
                    ds->payload = (uint8_t*)malloc(ds->payload_cap);
                }
                if (!ds->payload) return ds_set_error(ds, ZXC_ERROR_MEMORY);
                ds->decoded_cap = ds->block_size + ZXF_TAIL_PAD;
                ds_want_block_header(ds);
                break;
            }
            case DS_NEED_BLOCK_HEADER: {
                const int pr = ds_pull_scratch(ds, out, in);
                if (pr < 0) return ds_set_error(ds, pr);
                if (!pr) return (int64_t)produced;
                size_t need = 0;
                const int rc = ds_block_header(ds, ds->scratch, &need);
                if (rc < 0) return ds_set_error(ds, rc);
                if (rc == 1) { /* EOF: a SEK block or the footer follows */
                    ds->state = DS_PEEK_TAIL;
                    ds->scratch_used = 0;
                    ds->scratch_need = ZXF_BLOCK_HDR;
                    break;
                }
                ds_start_block(ds, need);
                ds->state = DS_NEED_BLOCK_PAYLOAD;
                break;
            }
            case DS_NEED_BLOCK_PAYLOAD: {
                const int pr = ds_pull_payload(ds, in);
                if (pr < 0) return ds_set_error(ds, pr);
                if (!pr) return (int64_t)produced;
                ds->state = DS_DECODE_BLOCK;
                break;
            }
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
                    ds->global_hash = zxf_hash_combine(ds->global_hash, ds_trailer(ds, i));
                const uint8_t* dec = ds_slot(ds, i);
                if (out->size - out->pos >= ds->decoded_cap) { /* the reference decodes straight into `out` */
                    const int rc = ps_out(ds->dev, out, dec, (size_t)dsz);
                    if (rc != ZXC_OK) return ds_set_error(ds, rc);
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
            case DS_EMIT_DECODED: {
                const int dr = ds_drain(ds, out, &produced);
                if (dr < 0) return ds_set_error(ds, dr);
                if (!dr) return (int64_t)produced;
                ds_want_block_header(ds);
                break;
            }
            case DS_PEEK_TAIL: {
                const int pr = ds_pull_scratch(ds, out, in);
                if (pr < 0) return ds_set_error(ds, pr);
                if (!pr) return (int64_t)produced;
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
            case DS_NEED_FOOTER_FULL: {
                const int pr = ds_pull_scratch(ds, out, in);
                if (pr < 0) return ds_set_error(ds, pr);
                if (!pr) return (int64_t)produced;
                ds->state = DS_VALIDATE_FOOTER;
                break;
            }
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

int64_t zxc_dstream_decompress(zxc_dstream* ds, zxc_outbuf_t* out, zxc_inbuf_t* in) {
    return ds_decompress(ds, out, in);
}

/* ========================================================================= */
/* the device streams (include/zxc_b200.h)                                   */
/* ========================================================================= */
/* A device call: the stream's device made current, the state machine run on `stream`, the queued copies gathered,
 * and the stream waited for, so that the caller may reuse `in` and read `out` on return.  A failure of that last
 * step is the stream's error from then on. */
static int ps_dev_enter(ps_dev* d, void* stream, int* prev) {
    *prev = zxg_current_device();
    d->stream = stream;
    d->n_segs = 0;
    d->mir_n = d->mir_i = 0; /* the mirror describes one call's `in` */
    d->hdr_direct = 0;
    return *prev == d->device ? ZXC_OK : zxg_set_device(d->device);
}

static int ps_dev_leave(ps_dev* d, int prev) {
    int rc = ps_flush(d);
    const int src = zxg_stream_sync(d->stream);
    if (rc == ZXC_OK) rc = src;
    if (prev != d->device) zxg_set_device(prev);
    return rc;
}

zxc_b200_cstream_device* zxc_b200_cstream_device_create(const zxc_compress_opts_t* opts) {
    return (zxc_b200_cstream_device*)cs_create(opts, 1);
}

void zxc_b200_cstream_device_free(zxc_b200_cstream_device* h) { zxc_cstream_free((zxc_cstream*)h); }

size_t zxc_b200_cstream_device_in_size(const zxc_b200_cstream_device* h) {
    return zxc_cstream_in_size((const zxc_cstream*)h);
}

size_t zxc_b200_cstream_device_out_size(const zxc_b200_cstream_device* h) {
    return zxc_cstream_out_size((const zxc_cstream*)h);
}

static int64_t cs_dev_call(zxc_cstream* cs, zxc_outbuf_t* out, zxc_inbuf_t* in, int end, void* stream) {
    if (!cs) return ZXC_ERROR_NULL_INPUT;
    int prev = 0;
    if (ps_dev_enter(cs->dev, stream, &prev) != ZXC_OK) return ZXC_B200_ERROR_CUDA;
    int64_t r = end ? cs_end(cs, out) : cs_compress(cs, out, in);
    const int rc = ps_dev_leave(cs->dev, prev);
    if (rc != ZXC_OK && r >= 0) r = cs_set_error(cs, rc);
    return r;
}

int64_t zxc_b200_cstream_device_compress(zxc_b200_cstream_device* h, zxc_outbuf_t* out, zxc_inbuf_t* in,
                                         void* stream) {
    return cs_dev_call((zxc_cstream*)h, out, in, 0, stream);
}

int64_t zxc_b200_cstream_device_end(zxc_b200_cstream_device* h, zxc_outbuf_t* out, void* stream) {
    return cs_dev_call((zxc_cstream*)h, out, NULL, 1, stream);
}

zxc_b200_dstream_device* zxc_b200_dstream_device_create(const zxc_decompress_opts_t* opts) {
    return (zxc_b200_dstream_device*)ds_create(opts, 1);
}

void zxc_b200_dstream_device_free(zxc_b200_dstream_device* h) { zxc_dstream_free((zxc_dstream*)h); }

int zxc_b200_dstream_device_finished(const zxc_b200_dstream_device* h) {
    return zxc_dstream_finished((const zxc_dstream*)h);
}

size_t zxc_b200_dstream_device_in_size(const zxc_b200_dstream_device* h) {
    return zxc_dstream_in_size((const zxc_dstream*)h);
}

size_t zxc_b200_dstream_device_out_size(const zxc_b200_dstream_device* h) {
    return zxc_dstream_out_size((const zxc_dstream*)h);
}

int64_t zxc_b200_dstream_device_decompress(zxc_b200_dstream_device* h, zxc_outbuf_t* out, zxc_inbuf_t* in,
                                           void* stream) {
    zxc_dstream* ds = (zxc_dstream*)h;
    if (!ds) return ZXC_ERROR_NULL_INPUT;
    int prev = 0;
    if (ps_dev_enter(ds->dev, stream, &prev) != ZXC_OK) return ZXC_B200_ERROR_CUDA;
    int64_t r = ds_decompress(ds, out, in);
    const int rc = ps_dev_leave(ds->dev, prev);
    if (rc != ZXC_OK && r >= 0) r = ds_set_error(ds, rc);
    return r;
}
