/*
 * zxc_gpu.h -- internal C interface between the host C code (zxc_api.c,
 * zxc_frame.c) and the CUDA translation unit (zxc_gpu.cu).  Plain C types only.
 */
#ifndef ZXC_B200_GPU_H
#define ZXC_B200_GPU_H

#include <stddef.h>
#include <stdint.h>

#include "zxc_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* A device context: one CUDA stream plus growable device / pinned buffers that
 * survive between calls.  The buffer API is stateless and thread-safe in the
 * reference (docs/API.md:1530-1538), so contexts come from a mutex-guarded
 * free list instead of a global singleton stream. */
typedef struct zxg_ctx zxg_ctx;

/* ZXC_OK, or ZXC_B200_ERROR_NO_DEVICE (message printed once to stderr). */
int zxg_init(void);
zxg_ctx* zxg_acquire(void);
void zxg_release(zxg_ctx* c);
void zxg_destroy(zxg_ctx* c); /* for contexts owned by a zxc_dctx / zxc_seekable */
zxg_ctx* zxg_create(void);

/* Named device buffers of a context, grown on demand (never shrunk). */
enum { ZXG_BUF_IN = 0, ZXG_BUF_OUT, ZXG_BUF_JOBS, ZXG_BUF_STATUS, ZXG_BUF_DICT, ZXG_BUF_SCRATCH,
       ZXG_BUF_AUX, ZXG_BUF_COUNT };
void* zxg_buffer(zxg_ctx* c, int which, size_t bytes); /* NULL on allocation failure */

/* Host <-> device copies on the context's stream.  Pageable host memory is
 * staged through the context's pinned bounce buffers in chunks so the copy and
 * the host memcpy overlap. */
int zxg_h2d(zxg_ctx* c, void* d_dst, const void* h_src, size_t bytes);
int zxg_d2h(zxg_ctx* c, void* h_dst, const void* d_src, size_t bytes);
int zxg_sync(zxg_ctx* c);
void* zxg_stream(zxg_ctx* c);

/* Whole decode step for host-resident input: upload jobs, launch, fetch statuses.
 * h_status receives n_jobs entries. */
int zxg_decode_jobs(zxg_ctx* c, const void* d_src, void* d_dst, const zxc_b200_job_t* h_jobs,
                    uint32_t n_jobs, int32_t* h_status, const void* h_dict, uint32_t dict_size,
                    const void* h_dict_huf, uint32_t block_size, int verify_checksums);

/* Encode src into the frame body (data blocks back to back); see zxc_gpu.cu. */
int zxg_encode_body(zxg_ctx* c, const uint8_t* h_src, uint64_t src_size, uint32_t block_size, int level,
                    int checksum, uint32_t n_blocks, uint8_t* h_body, uint64_t body_cap, uint32_t* h_sizes,
                    uint64_t* body_size, const void* h_dict, uint32_t dict_size, const uint8_t* h_dict_huf_lens);

/* A prepared dictionary in device memory (zxc_b200_dict_device): one allocation of zxg_ddict_bytes(dict_size) bytes
 * with the regions the per-call staging builds, made once by zxg_ddict_build and only read after that.
 *   decode region: the content, then its 128-byte table when one was given (dec_huf != NULL): dec_stage_dict's region
 *   encode region: the content zero-padded, one seeded head / chain pair per hash (levels 1-2, levels 3-7), then the
 *                  256 literal lengths when enc_lens != NULL: enc_stage_dict's region, with two pairs */
typedef struct {
    const void* dec;
    const void* dec_huf;
    const void* enc;
    const void* enc_lens;
    uint32_t dict_size;
} zxg_ddict_t;
size_t zxg_ddict_bytes(uint32_t dict_size);
/* Builds both regions at d_base from host bytes (h_dec_huf: the table the decode region carries, or NULL; h_lens: the
 * 256 unpacked lengths, or NULL) on `stream` and waits for them; fills *dd. */
int zxg_ddict_build(void* d_base, const void* h_dict, uint32_t dict_size, const void* h_dec_huf, const uint8_t* h_lens,
                    void* stream, zxg_ddict_t* dd);

/* Device-to-device compress (zxc_b200_compress_device).  The host writes the frame's fixed bytes with the
 * zxc_format.c helpers; the device places them around the body it assembles.  The compress calls below take their
 * dictionary as host bytes (h_dict, staged per call into the scratch's dictionary region) or as a prepared dictionary
 * dd (then h_dict is NULL, dict_size 0, and the layout has no dictionary region). */
typedef struct {
    uint8_t header[16];    /* file header */
    uint8_t eof[8];        /* EOF block header */
    uint8_t sek[8];        /* SEK block header (when seekable) */
    uint8_t footer[12];    /* footer with a zero hash; the device writes the hash when checksums are on */
    uint64_t fixed;        /* file header + trailer bytes */
    uint64_t dst_capacity;
    int seekable;          /* a SEK table follows the EOF block (seekable and at least one block) */
} zxg_frame_bytes_t;
/* scratch for the full resident encode grid (0 without a device) */
size_t zxg_encode_scratch_bytes(uint64_t src_size, uint32_t block_size, int level, uint32_t n_blocks,
                                uint32_t dict_size);
/* enqueues the copy, encode and assembly on `stream`; ZXC_ERROR_MEMORY when the scratch holds less than one warp */
int zxg_compress_device(const void* d_src, uint64_t src_size, void* d_dst, uint32_t block_size, int level,
                        int checksum, uint32_t n_blocks, const void* h_dict, uint32_t dict_size,
                        const uint8_t* h_dict_huf_lens, const zxg_ddict_t* dd, const zxg_frame_bytes_t* fb,
                        void* d_scratch, size_t scratch_size, int64_t* d_result, zxc_b200_job_t* d_jobs, void* stream);

/* The decode options of a device-resident decode, resolved on the host from zxc_decompress_opts_t: what needs no
 * frame bytes. */
typedef struct {
    const void* dict;     /* NULL without a dictionary; copied into the scratch */
    const void* dict_huf; /* its literal table, NULL unless dict_huf_attach finds it usable */
    const void* d_dict;   /* or a prepared dictionary's decode region (dict is then NULL): used where it lies */
    const void* d_dict_huf;
    uint32_t dict_size;
    uint32_t dict_id;     /* zxc_dict_id of the dictionary */
    int huf_verdict;      /* dict_huf_attach of its table: 1 usable, 0 none, < 0 malformed */
    int checksum_enabled;
} zxg_dopts_t;

/* Device-to-device decompress (zxc_b200_decompress_device).  Scratch for frames of at most block_size-byte blocks
 * decoded into dst_capacity bytes (0 without a device or for a dst_capacity too large to plan); ZXC_ERROR_MEMORY when
 * the scratch holds less than that for 4 KiB blocks. */
size_t zxg_decompress_scratch_bytes(uint64_t dst_capacity, uint32_t block_size);
int zxg_decompress_device(const void* d_src, uint64_t src_size, void* d_dst, uint64_t dst_capacity,
                          const zxg_dopts_t* o, void* d_scratch, size_t scratch_size, int64_t* d_result, void* stream);

/* In-place decode of a device-resident frame (zxc_b200_decompress_inplace_device; kernels in zxc_dinplace.cuh): the
 * frame of comp_size bytes lies flush-right in d_buffer[0 .. buffer_capacity) and decodes into d_buffer[0 ..).
 * ZXC_ERROR_MEMORY when the scratch holds less than the layout for 4 KiB
 * blocks and the smallest window.  The scratch size for a window of `window` compressed bytes per round (0 without a
 * device or when that cannot be planned). */
size_t zxg_decompress_inplace_scratch_bytes(uint64_t buffer_capacity, uint32_t block_size, uint64_t window);
int zxg_decompress_inplace_device(void* d_buffer, uint64_t buffer_capacity, uint64_t comp_size, const zxg_dopts_t* o,
                                  void* d_scratch, size_t scratch_size, int64_t* d_result, void* stream);

/* Many device-resident frames in one call (zxc_b200_decompress_device_batch; kernels in zxc_dbatch.cuh), with the
 * host's share of the verdicts made as for zxg_decompress_device.  Scratch for up to max_frames frames of at most
 * max_total_capacity output bytes in all and block_size-byte blocks (0 without a device or when that cannot be
 * planned); ZXC_ERROR_MEMORY when the scratch holds less than that for no output and 4 KiB blocks. */
size_t zxg_decompress_batch_scratch_bytes(uint32_t max_frames, uint64_t max_total_capacity, uint32_t block_size);
int zxg_decompress_device_batch(const zxc_b200_frame_t* d_frames, uint32_t n_frames, const zxg_dopts_t* o,
                                void* d_scratch, size_t scratch_size, int64_t* d_results, void* stream);

/* Many device-resident buffers compressed in one call (zxc_b200_compress_device_batch; kernels in zxc_cbatch.cuh), with
 * the options checked and the shared frame bytes (file header, EOF block header) written by the host.  Scratch for up
 * to max_frames buffers of at most max_total_src bytes in all (0 without a device or when that cannot be planned);
 * ZXC_ERROR_MEMORY when the scratch holds less than that for empty buffers. */
size_t zxg_compress_batch_scratch_bytes(uint32_t max_frames, uint64_t max_total_src, uint32_t block_size, int level,
                                        uint32_t dict_size);
int zxg_compress_device_batch(const zxc_b200_frame_t* d_frames, uint32_t n_frames, uint32_t block_size, int level,
                              int checksum, int seekable, const void* h_dict, uint32_t dict_size,
                              const uint8_t* h_dict_huf_lens, const zxg_ddict_t* dd, const uint8_t* header,
                              const uint8_t* eof, void* d_scratch, size_t scratch_size, int64_t* d_results,
                              void* stream);

/* The block API in HBM (zxc_b200_compress_blocks_device, zxc_b200_decompress_blocks_device; kernels in
 * zxc_blocks.cuh), with the options checked by the host.  Scratch sizes (0 without a device or when that cannot be
 * planned); ZXC_ERROR_MEMORY when the scratch holds less than the call's minimum. */
size_t zxg_compress_blocks_scratch_bytes(uint32_t max_blocks, uint64_t max_total_src, uint32_t max_src_size, int level,
                                         uint32_t dict_size);
int zxg_compress_blocks_device(const zxc_b200_frame_t* d_items, uint32_t n_items, int level, int checksum,
                               const void* h_dict, uint32_t dict_size, const zxg_ddict_t* dd, void* d_scratch,
                               size_t scratch_size, int64_t* d_results, void* stream);
size_t zxg_decompress_blocks_scratch_bytes(uint32_t max_blocks, uint64_t max_dst_capacity);
int zxg_decompress_blocks_device(const zxc_b200_frame_t* d_items, uint32_t n_items, const zxg_dopts_t* o, int safe,
                                 void* d_scratch, size_t scratch_size, int64_t* d_results, void* stream);

/* Device-resident seekable frames (zxc_dseek.c; kernels in zxc_dseek.cuh).  What a range call needs of its handle. */
typedef struct {
    const void* d_src;
    const uint64_t* d_offs; /* comp_offsets: num_blocks + 1 entries */
    uint64_t total;
    uint32_t block_size, num_blocks, dict_id;
    const void* d_dict; /* NULL without a dictionary; its 128-byte table right behind it when d_dict_huf is set */
    uint32_t dict_size;
    const void* d_dict_huf;
} zxg_dseek_t;
/* synchronous copies on `stream`, and device memory for a handle (zxg_dev_free waits for the current device first) */
int zxg_d2h_sync(void* h_dst, const void* d_src, size_t bytes, void* stream);
int zxg_h2d_sync(void* d_dst, const void* h_src, size_t bytes, void* stream);
void* zxg_dev_alloc(size_t bytes);
void zxg_dev_free(void* d);
/* scratch for n_ranges ranges with a direct job table of J entries (0 when that cannot be planned) */
size_t zxg_dseek_scratch_bytes(uint32_t block_size, uint32_t n_ranges, uint64_t J);
/* enqueues the plan, the two decodes and the finish; ZXC_ERROR_MEMORY for a scratch below one job-table entry */
int zxg_dseek_ranges(const zxg_dseek_t* h, const zxc_b200_range_t* d_ranges, uint32_t n_ranges, void* d_dst,
                     uint64_t dst_capacity, void* d_scratch, size_t scratch_size, int64_t* d_results, void* stream);

/* Push streams in HBM (zxc_b200_cstream_device / _dstream_device: zxc_pstream.c; kernels in zxc_pstream_device.cuh).
 * Every call enqueues on `stream`; the ones that return host values synchronise it. */
typedef struct {
    uint64_t off;     /* the header's offset from the walk's start */
    uint64_t hdr;     /* its 8 bytes, little-endian */
    uint32_t len;     /* on-disk length of a data block whole in the chunk; 0 for the header the walk stopped at */
    uint32_t trailer; /* the block's checksum trailer (0 without checksums) */
} zxg_psblk_t;
typedef struct {
    uint64_t src, dst, len; /* device addresses; len <= ZXG_PS_PIECE */
} zxg_psseg_t;
#define ZXG_PS_PIECE ((uint64_t)64 << 10)
/* Walks block headers from d_src (size bytes) for at most max_blocks whole data blocks, plus the header it stopped at:
 * h_out (max_blocks + 1 entries) and *n_out, through d_out (as large) and d_n in one copy. */
int zxg_ps_walk(const void* d_src, uint64_t size, uint32_t max_blocks, uint64_t bound, int has_checksum,
                zxg_psblk_t* d_out, zxg_psblk_t* h_out, uint32_t* n_out, void* stream);
/* Device bytes of one batch: the decode scratch for n_jobs jobs; the encode's per-warp scratch and its staging stride. */
size_t zxg_ps_decode_scratch_bytes(uint32_t n_jobs, uint32_t block_size);
size_t zxg_ps_encode_scratch_bytes(uint32_t n_blocks, uint32_t block_size, int level);
uint32_t zxg_ps_stage_stride(uint32_t block_size);
/* Decodes n jobs (src_off: device addresses; dst_off: offsets into d_dst) with the jobs and statuses at d_jobs /
 * d_status and the three work counters at d_counter; h_status gets the n statuses. */
int zxg_ps_decode(const zxc_b200_job_t* h_jobs, uint32_t n, zxc_b200_job_t* d_jobs, int32_t* d_status, void* d_dst,
                  void* d_scratch, size_t scratch_size, unsigned long long* d_counter, uint32_t block_size, int verify,
                  int32_t* h_status, void* stream);
/* Encodes n_blocks blocks of d_src (16-byte aligned, 64 zero bytes behind src_size) into staging slots of
 * zxg_ps_stage_stride(block_size) bytes at d_stage; h_st gets the n sizes, then the n trailers (d_st as large). */
int zxg_ps_encode(const void* d_src, uint64_t src_size, uint32_t block_size, int level, int checksum, uint32_t n_blocks,
                  void* d_stage, uint32_t* d_st, void* d_scratch, unsigned long long* d_counter, uint32_t* h_st,
                  void* stream);
/* Copies the n pieces at h_segs to d_segs (n entries) and gathers them in one launch. */
int zxg_ps_gather(const zxg_psseg_t* h_segs, uint32_t n, zxg_psseg_t* d_segs, void* stream);
/* Stream-ordered copies, not waited for (a pageable host source has been read when they return). */
int zxg_d2d_async(void* d_dst, const void* d_src, size_t bytes, void* stream);
int zxg_h2d_async(void* d_dst, const void* h_src, size_t bytes, void* stream);
int zxg_memset_async(void* d_dst, int v, size_t bytes, void* stream);
int zxg_stream_sync(void* stream);
/* page-locked host memory (cudaMallocHost), for copies that run at full speed; NULL on failure */
void* zxg_host_alloc(size_t bytes);
void zxg_host_free(void* h);

/* Device selection for the calling thread (multi-device fork-join in zxc_api.c): current device, device count,
 * cudaSetDevice.  zxg_acquire() hands out a context of the calling thread's current device. */
int zxg_current_device(void);
int zxg_device_count(void);
int zxg_set_device(int dev); /* ZXC_OK or ZXC_B200_ERROR_CUDA */

/* 1 when the pointer is page-locked (cudaHostAlloc / cudaHostRegister / managed) */
int zxg_host_pinned(const void* p);

/* Frame decode with H2D / decode / D2H overlapped over chunks of whole blocks; both host
 * buffers must be page-locked.  Job offsets are relative to h_src / h_dst; h_status gets
 * n_jobs entries.  The output is copied back even for failing jobs (caller decides). */
int zxg_decode_pipelined(zxg_ctx* c, const uint8_t* h_src, uint64_t src_lo, uint64_t src_hi, uint8_t* h_dst,
                         uint64_t produced, const zxc_b200_job_t* h_jobs, uint32_t n_jobs, int32_t* h_status,
                         const void* h_dict, uint32_t dict_size, const void* h_dict_huf, uint32_t block_size,
                         int verify_checksums);

/* Frame decode for ordinary (pageable) host memory, staged through the context's pinned bounce buffers with
 * H2D / decode / D2H and the host copies overlapped.  Source bytes come from h_src (absolute offsets, like the
 * jobs' src_off) or, when `fetch` is given, from fetch(fetch_ctx, dst, len, offset) (ZXC_OK or a negative code):
 * the reader path of zxc_seekable (include/zxc_seekable.h:96-140).  Decoded bytes [clip_lo, clip_hi) (job dst
 * coordinates) land at h_dst. */
typedef int (*zxg_fetch_fn)(void* ctx, void* dst, size_t len, uint64_t off);
int zxg_decode_staged(zxg_ctx* c, const uint8_t* h_src, zxg_fetch_fn fetch, void* fetch_ctx, uint64_t src_lo,
                      uint64_t src_hi, uint8_t* h_dst, uint64_t clip_lo, uint64_t clip_hi, const zxc_b200_job_t* h_jobs,
                      uint32_t n_jobs, int32_t* h_status, const void* h_dict, uint32_t dict_size, const void* h_dict_huf,
                      uint32_t block_size, int verify_checksums);

/* ---- dictionary training (zxc_train.c; kernels in zxc_train.cuh) ----
 * The content trainer runs zxg_train_segments, orders the segments on the host, then zxg_train_pick (or
 * zxg_train_tail) on the same context: the corpus and the k-gram table stay on the device in between. */
typedef struct { uint32_t offset, len, score; } zxg_seg_t; /* len 0: no segment */

/* Uploads the samples as one corpus, counts the k-grams at every freq_stride-th position, builds a segment per
 * start (start s at s * seg_stride, n_starts of them) and keeps the first seg_alloc in position order:
 * h_segs (seg_alloc entries) and *n_segs. */
int zxg_train_segments(zxg_ctx* c, const void* const* samples, const size_t* sizes, size_t n_samples,
                       uint64_t corpus_size, uint64_t freq_stride, uint64_t seg_stride, uint32_t n_starts,
                       uint32_t seg_alloc, zxg_seg_t* h_segs, uint32_t* n_segs);
/* The greedy pick over the segments in the given order and the reversed emission into h_out (capacity bytes);
 * *filled = bytes picked (0: nothing selected). */
int zxg_train_pick(zxg_ctx* c, uint64_t corpus_size, const zxg_seg_t* h_sorted, uint32_t n_segs, uint32_t capacity,
                   uint8_t* h_out, uint32_t* filled);
/* The last `bytes` bytes of the uploaded corpus. */
int zxg_train_tail(zxg_ctx* c, uint64_t corpus_size, uint32_t bytes, uint8_t* h_out);
/* Literal histogram (256 counts) of the level-6 parses of [dict | piece] for every piece (<= 4096 bytes each). */
int zxg_train_literals(zxg_ctx* c, const void* const* pieces, const size_t* sizes, size_t n, const void* h_dict,
                       uint32_t dict_size, uint32_t* h_freq);

/* Phase times (ms) of the calling thread's last training calls: device time from CUDA events, host time from the
 * host clock. */
enum { ZXG_T_UPLOAD = 0, ZXG_T_COUNT, ZXG_T_SEGMENTS, ZXG_T_SORT, ZXG_T_PICK, ZXG_T_SLICES, ZXG_T_HIST, ZXG_T_CODES,
       ZXG_T_N };
double* zxg_train_times(void);

#ifdef __cplusplus
}
#endif
#endif
