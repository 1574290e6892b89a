/*
 * zxc_dseek.c -- random access into a seekable frame held in device memory (include/zxc_b200.h,
 * zxc_b200_seekable_device_*): the device twin of zxc_seekable_open + zxc_seekable_decompress_range (zxc_api.c).
 *
 * Open parses the SEK table on the host with the same parser as zxc_seekable_open (zxw_seek_parse), reading the frame
 * through a few device-to-host copies, and keeps the table's block offsets in device memory: the plan that a range
 * call needs, built once per frame.  A range call is then all device work on the caller's stream (zxc_dseek.cuh).
 *
 * zxc_b200_seekable_device_open_host opens a frame in page-locked host memory into the same handle: the table is read
 * where it lies, and the handle also keeps the frame's device address and its largest on-disk block, with which each
 * range call stages the blocks it covers into its scratch before decoding them.
 */
#include <stdlib.h>
#include <string.h>

#include "zxc.h"
#include "zxc_format.h"
#include "zxc_frame.h"
#include "zxc_gpu.h"

struct zxc_b200_seekable_device_s {
    zxg_dseek_t g;
    uint64_t* d_offs; /* owned */
    uint8_t* d_dict;  /* owned: the dictionary, then its 128-byte table when one was given */
    int device;
};

typedef struct {
    const uint8_t* d_src;
    uint64_t size;
    void* stream;
} dseek_fetch_ctx;

/* seekable_fetch over device memory */
static int dseek_fetch(void* ctx, void* dst, size_t len, uint64_t off) {
    const dseek_fetch_ctx* f = (const dseek_fetch_ctx*)ctx;
    if (off > f->size || len > f->size - off) return ZXC_ERROR_SRC_TOO_SMALL;
    return zxg_d2h_sync(dst, f->d_src + off, len, f->stream);
}

/* seekable_fetch over host memory */
static int dseek_fetch_host(void* ctx, void* dst, size_t len, uint64_t off) {
    const dseek_fetch_ctx* f = (const dseek_fetch_ctx*)ctx;
    if (off > f->size || len > f->size - off) return ZXC_ERROR_SRC_TOO_SMALL;
    memcpy(dst, f->d_src + off, len);
    return ZXC_OK;
}

/* makes the handle's device current; *prev gets the device to restore */
static int dseek_enter(const zxc_b200_seekable_device* h, int* prev) {
    *prev = zxg_current_device();
    return h->device == *prev ? ZXC_OK : zxg_set_device(h->device);
}

static void dseek_leave(const zxc_b200_seekable_device* h, int prev) {
    if (h->device != prev) zxg_set_device(prev);
}

/* the handle for a frame that d_src reads on the device, its table parsed through fetch over f */
static zxc_b200_seekable_device* dseek_open(const void* d_src, uint64_t src_size, zxw_fetch_fn fetch,
                                            dseek_fetch_ctx* f, int host, void* stream) {
    zxw_seek_t tab;
    if (zxw_seek_parse(fetch, f, src_size, &tab) != ZXC_OK) return NULL;
    zxc_b200_seekable_device* h = (zxc_b200_seekable_device*)calloc(1, sizeof *h);
    const size_t offs_bytes = ((size_t)tab.num_blocks + 1) * sizeof(uint64_t);
    if (h) h->d_offs = (uint64_t*)zxg_dev_alloc(offs_bytes);
    if (!h || !h->d_offs || zxg_h2d_sync(h->d_offs, tab.comp_offsets, offs_bytes, stream) != ZXC_OK) {
        if (h) zxg_dev_free(h->d_offs);
        free(h);
        zxw_seek_free(&tab);
        return NULL;
    }
    h->device = zxg_current_device();
    h->g.d_src = d_src;
    h->g.d_offs = h->d_offs;
    h->g.total = tab.total;
    h->g.block_size = tab.block_size;
    h->g.num_blocks = tab.num_blocks;
    h->g.dict_id = tab.dict_id;
    h->g.src_size = src_size;
    for (uint32_t b = 0; host && b < tab.num_blocks; b++)
        if (tab.comp_sizes[b] > h->g.max_comp) h->g.max_comp = tab.comp_sizes[b]; /* >= 8: a block header */
    zxw_seek_free(&tab);
    return h;
}

zxc_b200_seekable_device* zxc_b200_seekable_device_open(const void* d_src, uint64_t src_size, void* stream) {
    if (!d_src || src_size == 0 || zxg_init() != ZXC_OK) return NULL;
    dseek_fetch_ctx f = {(const uint8_t*)d_src, src_size, stream};
    return dseek_open(d_src, src_size, dseek_fetch, &f, 0, stream);
}

zxc_b200_seekable_device* zxc_b200_seekable_device_open_host(const void* h_src, uint64_t src_size, void* stream) {
    if (!h_src || src_size == 0 || zxg_init() != ZXC_OK) return NULL;
    const void* mapped = zxg_host_mapped(h_src, (size_t)src_size);
    if (!mapped) return NULL;
    dseek_fetch_ctx f = {(const uint8_t*)h_src, src_size, stream};
    return dseek_open(mapped, src_size, dseek_fetch_host, &f, 1, stream);
}

/* zxc_seekable_set_dict's verdicts and order (zxc_api.c) */
int zxc_b200_seekable_device_set_dict(zxc_b200_seekable_device* h, const void* dict, size_t dict_size,
                                      const void* dict_huf) {
    if (!h || !dict || dict_size == 0) return ZXC_ERROR_NULL_INPUT;
    if (dict_size > ZXC_DICT_SIZE_MAX) return ZXC_ERROR_DICT_TOO_LARGE;
    if (h->g.dict_id != 0 && zxc_dict_id(dict, dict_size, dict_huf) != h->g.dict_id) return ZXC_ERROR_DICT_MISMATCH;
    int prev;
    int rc = dseek_enter(h, &prev);
    if (rc != ZXC_OK) return rc;
    /* one host buffer, one copy: the dictionary and its table behind it */
    const size_t bytes = dict_size + (dict_huf ? ZXC_HUF_TABLE_SIZE : 0);
    uint8_t* host = (uint8_t*)malloc(bytes);
    uint8_t* d = host ? (uint8_t*)zxg_dev_alloc(bytes) : NULL;
    if (d) {
        memcpy(host, dict, dict_size);
        if (dict_huf) memcpy(host + dict_size, dict_huf, ZXC_HUF_TABLE_SIZE);
        rc = zxg_h2d_sync(d, host, bytes, NULL);
    }
    free(host);
    if (!d || rc != ZXC_OK) {
        zxg_dev_free(d);
        d = NULL;
        rc = rc != ZXC_OK ? rc : ZXC_ERROR_MEMORY; /* the previous dictionary is dropped, as zxc_seekable_set_dict does */
    }
    zxg_dev_free(h->d_dict); /* waits for the range calls that may still read it */
    h->d_dict = d;
    h->g.d_dict = d;
    h->g.dict_size = d ? (uint32_t)dict_size : 0;
    h->g.d_dict_huf = (d && dict_huf) ? d + dict_size : NULL;
    dseek_leave(h, prev);
    return rc;
}

uint32_t zxc_b200_seekable_device_num_blocks(const zxc_b200_seekable_device* h) { return h ? h->g.num_blocks : 0; }
uint64_t zxc_b200_seekable_device_decompressed_size(const zxc_b200_seekable_device* h) { return h ? h->g.total : 0; }
uint32_t zxc_b200_seekable_device_block_size(const zxc_b200_seekable_device* h) { return h ? h->g.block_size : 0; }

size_t zxc_b200_seekable_device_scratch_size(const zxc_b200_seekable_device* h, uint32_t max_ranges,
                                             uint64_t max_bytes) {
    if (!h) return 0;
    const uint64_t bs = h->g.block_size;
    uint64_t J = max_bytes / bs + (max_bytes % bs != 0);
    /* a frame in host memory stages per job, so its table leaves no slack: each range may also cover a short last
     * block whole for fewer than block_size bytes */
    if (h->g.max_comp && h->g.total % bs) J += max_ranges;
    return zxg_dseek_scratch_bytes(h->g.block_size, max_ranges, J, h->g.max_comp);
}

int zxc_b200_seekable_device_decompress_ranges(zxc_b200_seekable_device* h, const zxc_b200_range_t* d_ranges,
                                               uint32_t n_ranges, void* d_dst, uint64_t dst_capacity, void* d_scratch,
                                               size_t scratch_size, int64_t* d_results, void* stream) {
    if (!h || (n_ranges > 0 && (!d_ranges || !d_results || !d_scratch))) return ZXC_ERROR_NULL_INPUT;
    int rc = zxg_init();
    if (rc != ZXC_OK || n_ranges == 0) return rc;
    int prev;
    rc = dseek_enter(h, &prev);
    if (rc != ZXC_OK) return rc;
    rc = zxg_dseek_ranges(&h->g, d_ranges, n_ranges, d_dst, dst_capacity, d_scratch, scratch_size, d_results, stream);
    dseek_leave(h, prev);
    return rc;
}

void zxc_b200_seekable_device_free(zxc_b200_seekable_device* h) {
    if (!h) return;
    int prev;
    const int rc = dseek_enter(h, &prev);
    zxg_dev_free(h->d_dict);
    zxg_dev_free(h->d_offs);
    if (rc == ZXC_OK) dseek_leave(h, prev);
    free(h);
}
