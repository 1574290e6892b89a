/*
 * zxc_train.c -- the reference's dictionary trainers (include/zxc_dict.h) with their data-parallel work on the GPU:
 * argument checks in the reference's order, the reference's sampling arithmetic, the heap order of the candidate
 * segments, and the code lengths of the shared literal table.  The kernels are in zxc_train.cuh (DESIGN.md 7d).
 *
 * Same bytes and the same return codes as the reference for every input (file:line in /root/reference/src/lib):
 *   zxc_train_dict       zxc_dict.c:309-461
 *   zxc_train_dict_huf   zxc_dict.c:490-580
 *   zxc_dict_train       zxc_dict.c:600-638
 *   constants            zxc_internal.h:393-408
 */
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "zxc.h"
#include "zxc_b200.h"
#include "zxc_gpu.h"
#include "zxc_hufenc.h"

#define TR_KGRAM 5u                          /* k-gram length: the format's minimum match */
#define TR_SAMPLE_TARGET ((uint64_t)1 << 19) /* k-gram positions counted, about */
#define TR_MAX_SEGS ((uint64_t)1 << 16)      /* candidate segments kept */
#define TR_SLICE 4096u                       /* the table trainer's slice (the small-block regime) */
#define TR_SLICE_BUDGET ((uint64_t)8 << 20)  /* slice bytes the table trainer parses, about */
#define TR_HUF_MAX_LEN 8                     /* code-length cap of level 6 (ZXC_HUF_MAX_CODE_LEN_DENSITY) */

static double now_ms(void) {
    struct timespec t;
    clock_gettime(CLOCK_MONOTONIC, &t);
    return 1e3 * (double)t.tv_sec + 1e-6 * (double)t.tv_nsec;
}

/* ---- segment order --------------------------------------------------------------------------------------------
 * Descending score by an in-place heapsort: bottom-up build of a min-heap on the score, then repeated extraction of
 * the minimum to the tail.  The sort is not stable, and equal scores are common (repeated records give many segments
 * of one score), so the order of ties -- and with it the dictionary -- is defined by exactly this procedure.  That is
 * why it runs here on the host rather than as a GPU radix or merge sort: at most 65 536 records, a few milliseconds. */
static void seg_sift_down(zxg_seg_t* a, size_t root, size_t n) {
    for (;;) {
        size_t child = 2 * root + 1;
        if (child >= n) return;
        if (child + 1 < n && a[child + 1].score < a[child].score) child++;
        if (a[root].score <= a[child].score) return;
        const zxg_seg_t t = a[root];
        a[root] = a[child];
        a[child] = t;
        root = child;
    }
}

static void seg_sort_desc(zxg_seg_t* a, size_t n) {
    if (n < 2) return;
    for (size_t i = n / 2; i-- > 0;) seg_sift_down(a, i, n);
    for (size_t end = n; end > 1;) {
        end--;
        const zxg_seg_t t = a[0];
        a[0] = a[end];
        a[end] = t;
        seg_sift_down(a, 0, end);
    }
}

/* The bodies of the trainers and of their device twins: `src` says where the sample bytes are.  Everything before
 * the gather -- verdicts, sampling arithmetic, which slices are kept -- is the same code for both. */
static int64_t train_dict(const void* const* samples, const size_t* sample_sizes, size_t n_samples, void* dict_buf,
                          size_t dict_capacity, const zxg_train_src_t* src) {
    if (!samples || !sample_sizes || n_samples == 0 || !dict_buf || dict_capacity == 0) return ZXC_ERROR_NULL_INPUT;
    if (dict_capacity > ZXC_DICT_SIZE_MAX) return ZXC_ERROR_DICT_TOO_LARGE;
    uint64_t corpus_size = 0;
    for (size_t i = 0; i < n_samples; i++) corpus_size += sample_sizes[i];
    if (corpus_size < TR_KGRAM) return ZXC_ERROR_SRC_TOO_SMALL;
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;

    /* the k-gram count samples about TR_SAMPLE_TARGET positions: a full count saturates the 16-bit counters */
    const uint64_t kgram_limit = corpus_size - TR_KGRAM + 1;
    uint64_t freq_stride = kgram_limit / TR_SAMPLE_TARGET;
    if (freq_stride < 1) freq_stride = 1;
    /* segment starts are spread over the whole corpus; the first seg_alloc that make a segment are kept */
    const uint64_t max_segs = corpus_size / TR_KGRAM;
    const uint32_t seg_alloc = (uint32_t)(max_segs < TR_MAX_SEGS ? max_segs : TR_MAX_SEGS);
    uint64_t stride = TR_KGRAM;
    if (corpus_size / seg_alloc > stride) stride = corpus_size / seg_alloc;
    const uint32_t n_starts = (uint32_t)((corpus_size - TR_KGRAM) / stride + 1);

    zxg_seg_t* segs = (zxg_seg_t*)malloc((size_t)seg_alloc * sizeof *segs);
    if (!segs) return ZXC_ERROR_MEMORY;
    zxg_ctx* g = zxg_acquire();
    if (!g) {
        free(segs);
        return ZXC_ERROR_MEMORY;
    }
    double* times = zxg_train_times();
    for (int k = ZXG_T_UPLOAD; k <= ZXG_T_PICK; k++) times[k] = 0;
    uint8_t* out = (uint8_t*)dict_buf;
    const uint32_t cap = (uint32_t)dict_capacity;
    uint32_t n_segs = 0, filled = 0;
    int rc = zxg_train_segments(g, samples, sample_sizes, n_samples, corpus_size, freq_stride, stride, n_starts, seg_alloc,
                                segs, &n_segs, src);
    if (rc == ZXC_OK && n_segs > 0) {
        const double t0 = now_ms();
        seg_sort_desc(segs, n_segs);
        times[ZXG_T_SORT] = now_ms() - t0;
        rc = zxg_train_pick(g, corpus_size, segs, n_segs, cap, out, &filled);
    }
    /* no frequent k-gram, or every segment subsumed by an earlier pick: the tail of the corpus */
    if (rc == ZXC_OK && filled == 0) {
        filled = corpus_size < cap ? (uint32_t)corpus_size : cap;
        rc = zxg_train_tail(g, corpus_size, filled, out);
    }
    zxg_release(g);
    free(segs);
    return rc != ZXC_OK ? rc : (int64_t)filled;
}

static int train_dict_huf(const void* const* samples, const size_t* sample_sizes, size_t n_samples, const void* dict,
                          size_t dict_size, uint8_t* huf_lengths_out, const zxg_train_src_t* src) {
    if (!samples || !sample_sizes || n_samples == 0 || !dict || dict_size == 0 || !huf_lengths_out)
        return ZXC_ERROR_NULL_INPUT;
    if (dict_size > ZXC_DICT_SIZE_MAX) return ZXC_ERROR_DICT_TOO_LARGE;
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;

    /* every slice while the samples fit the budget, else one slice in `stride`, counted across all samples; NULL or
     * empty samples hold no slices (but their sizes count toward the total) */
    uint64_t total = 0;
    for (size_t s = 0; s < n_samples; s++) total += sample_sizes[s];
    const uint64_t stride = total > TR_SLICE_BUDGET ? (total + TR_SLICE_BUDGET - 1) / TR_SLICE_BUDGET : 1;
    size_t kept = 0;
    uint64_t idx = 0;
    for (size_t s = 0; s < n_samples; s++) {
        if (!samples[s] || sample_sizes[s] == 0) continue;
        const uint64_t n_sl = (sample_sizes[s] + TR_SLICE - 1) / TR_SLICE;
        /* slices idx .. idx + n_sl - 1: the multiples of stride among them */
        kept += (size_t)((idx + n_sl + stride - 1) / stride - (idx + stride - 1) / stride);
        idx += n_sl;
    }
    const void** ptrs = (const void**)malloc((kept ? kept : 1) * sizeof *ptrs);
    size_t* lens = (size_t*)malloc((kept ? kept : 1) * sizeof *lens);
    zxh_work_t* W = (zxh_work_t*)malloc(sizeof *W);
    if (!ptrs || !lens || !W) {
        free(ptrs);
        free(lens);
        free(W);
        return ZXC_ERROR_MEMORY;
    }
    size_t k = 0;
    idx = 0;
    for (size_t s = 0; s < n_samples; s++) {
        const uint8_t* sample = (const uint8_t*)samples[s];
        const size_t size = sample_sizes[s];
        if (!sample || size == 0) continue;
        for (size_t off = 0; off < size; off += TR_SLICE, idx++) {
            if (idx % stride != 0) continue;
            ptrs[k] = sample + off;
            lens[k] = size - off < TR_SLICE ? size - off : TR_SLICE;
            k++;
        }
    }

    double* times = zxg_train_times();
    for (int t = ZXG_T_SLICES; t <= ZXG_T_CODES; t++) times[t] = 0;
    uint32_t freq[ZXH_NSYM];
    int rc;
    zxg_ctx* g = zxg_acquire();
    if (!g) {
        rc = ZXC_ERROR_MEMORY;
    } else {
        rc = zxg_train_literals(g, ptrs, lens, kept, dict, (uint32_t)dict_size, freq, src);
        zxg_release(g);
    }
    if (rc == ZXC_OK) {
        const double t0 = now_ms();
        uint32_t any = 0;
        for (int i = 0; i < ZXH_NSYM; i++) any |= freq[i];
        if (!any) {
            /* a low-entropy corpus leaves no literals: an all-zero table, which means "no table" */
            memset(huf_lengths_out, 0, ZXC_HUF_TABLE_SIZE);
        } else {
            uint8_t len[ZXH_NSYM];
            (void)zxh_build_code_lengths(freq, len, TR_HUF_MAX_LEN, W); /* cannot fail: some symbol occurs */
            (void)zxh_nudge_code_lengths(freq, len, TR_HUF_MAX_LEN, W);
            for (int i = 0; i < ZXC_HUF_TABLE_SIZE; i++)
                huf_lengths_out[i] = (uint8_t)((len[2 * i] & 15u) | ((len[2 * i + 1] & 15u) << 4));
        }
        times[ZXG_T_CODES] = now_ms() - t0;
    }
    free(ptrs);
    free(lens);
    free(W);
    return rc;
}

static int64_t dict_train(const void* const* samples, const size_t* sample_sizes, size_t n_samples, void* zxd_buf,
                          size_t zxd_capacity, const zxg_train_src_t* src) {
    if (!samples || !sample_sizes || n_samples == 0 || !zxd_buf || zxd_capacity == 0) return ZXC_ERROR_NULL_INPUT;
    uint8_t* content = (uint8_t*)malloc(ZXC_DICT_SIZE_MAX);
    if (!content) return ZXC_ERROR_MEMORY;
    int64_t out;
    const int64_t content_size = train_dict(samples, sample_sizes, n_samples, content, ZXC_DICT_SIZE_MAX, src);
    if (content_size <= 0) {
        out = content_size < 0 ? content_size : ZXC_ERROR_SRC_TOO_SMALL;
    } else {
        uint8_t huf[ZXC_HUF_TABLE_SIZE];
        const int hrc = train_dict_huf(samples, sample_sizes, n_samples, content, (size_t)content_size, huf, src);
        out = hrc != ZXC_OK ? hrc : zxc_dict_save(content, (size_t)content_size, huf, zxd_buf, zxd_capacity);
    }
    free(content);
    return out;
}

int64_t zxc_train_dict(const void* const* samples, const size_t* sample_sizes, size_t n_samples, void* dict_buf,
                       size_t dict_capacity) {
    return train_dict(samples, sample_sizes, n_samples, dict_buf, dict_capacity, NULL);
}

int zxc_train_dict_huf(const void* const* samples, const size_t* sample_sizes, size_t n_samples, const void* dict,
                       size_t dict_size, uint8_t* huf_lengths_out) {
    return train_dict_huf(samples, sample_sizes, n_samples, dict, dict_size, huf_lengths_out, NULL);
}

int64_t zxc_dict_train(const void* const* samples, const size_t* sample_sizes, size_t n_samples, void* zxd_buf,
                       size_t zxd_capacity) {
    return dict_train(samples, sample_sizes, n_samples, zxd_buf, zxd_capacity, NULL);
}

/* the device twins: the same bodies, the sample bytes gathered in HBM after the work enqueued on `stream` */
int64_t zxc_b200_train_dict_device(const void* const* samples, const size_t* sample_sizes, size_t n_samples,
                                   void* dict_buf, size_t dict_capacity, void* stream) {
    const zxg_train_src_t src = {1, stream};
    return train_dict(samples, sample_sizes, n_samples, dict_buf, dict_capacity, &src);
}

int zxc_b200_train_dict_huf_device(const void* const* samples, const size_t* sample_sizes, size_t n_samples,
                                   const void* dict, size_t dict_size, uint8_t* huf_lengths_out, void* stream) {
    const zxg_train_src_t src = {1, stream};
    return train_dict_huf(samples, sample_sizes, n_samples, dict, dict_size, huf_lengths_out, &src);
}

int64_t zxc_b200_dict_train_device(const void* const* samples, const size_t* sample_sizes, size_t n_samples,
                                   void* zxd_buf, size_t zxd_capacity, void* stream) {
    const zxg_train_src_t src = {1, stream};
    return dict_train(samples, sample_sizes, n_samples, zxd_buf, zxd_capacity, &src);
}

int zxc_b200_train_phase_times(double* ms, int n) {
    const double* t = zxg_train_times();
    int k = 0;
    for (; k < n && k < ZXG_T_N; k++) ms[k] = t[k];
    return k;
}
