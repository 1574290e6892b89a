/*
 * zxc_b200.h -- ADDITIVE device-resident entry points of the CUDA build.
 *
 * The reference C API (zxc_buffer.h, zxc_seekable.h) takes host pointers, so
 * every call pays PCIe both ways.  These entry points expose the same block
 * decode with the compressed frame and the output already in HBM: the host
 * walks the frame once into a job table (one entry per block), the kernel
 * decodes all jobs in one launch.  They are what bench.py times for the
 * HBM-resident `value`, and what a multi-GPU caller shards by block range.
 * zxc_b200_compress_device is the encode counterpart: HBM in, a complete frame (and its job table) in HBM out.
 *
 * Nothing here exists in the reference; adding symbols passes its ABI policy
 * (abidiff --no-added-syms, .github/workflows/abi-check.yml:128).
 *
 * Pointers named d_* are DEVICE pointers on the current CUDA device.
 * `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 */
#ifndef ZXC_B200_H
#define ZXC_B200_H

#include <stddef.h>
#include <stdint.h>

#include "zxc_export.h"
#include "zxc_opts.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One independent block = one unit of work (a warp of the decode kernel).  Replaces the reference's
 * zxc_seek_mt_job_t (src/lib/zxc_seekable.c:802-815). */
typedef struct {
    uint64_t src_off; /* byte offset of the 8-byte block header inside the source buffer */
    uint64_t dst_off; /* byte offset of the block's first decoded byte inside the output */
    uint32_t src_len; /* on-disk size: header + payload (+4 checksum when the frame has them) */
    uint32_t dst_cap; /* bytes the block may produce (block_size, or the tail remainder) */
} zxc_b200_job_t;

/* What the host learnt from walking a frame. */
typedef struct {
    uint64_t decoded_size;  /* footer value */
    uint32_t block_size;    /* from the file header */
    uint32_t n_blocks;      /* data blocks found before EOF */
    uint32_t dict_id;       /* 0 = none */
    int has_checksum;       /* file flag 0x80 */
    int seekable;           /* a valid SEK table was found and used */
    uint32_t global_hash;   /* footer value (0 without checksums) */
} zxc_b200_frame_info_t;

/* Number of usable CUDA devices (0 when there is no driver / no device). */
ZXC_EXPORT int zxc_b200_device_count(void);

/* Walk a frame held in HOST memory and fill jobs[0..n) (dst offsets assume every
 * block but the last decodes to block_size, which the decode then verifies).
 * Always the sequential header walk of zxc_decompress_frame (src/lib/zxc_dispatch.c:912-1001),
 * so damaged block headers are reported exactly as the reference reports them; the SEK
 * table is only probed to fill info->seekable.  jobs may be NULL to query the count.  Returns the number of blocks or a negative zxc_error_t. */
ZXC_EXPORT int64_t zxc_b200_plan_frame(const void* frame, size_t frame_size, zxc_b200_job_t* jobs,
                                       size_t max_jobs, zxc_b200_frame_info_t* info);

/* Bytes of device scratch zxc_b200_decode_blocks needs for blocks of at most
 * block_size decoded bytes (RLE / Huffman literal sections are expanded there). */
ZXC_EXPORT size_t zxc_b200_decode_scratch_size(uint32_t block_size);

/* Decode n_jobs blocks, device to device, on `stream` (asynchronous).
 *   d_src     base of the compressed bytes the jobs index into
 *   d_dst     base of the output
 *   d_jobs    job table in device memory
 *   d_status  one int32 per job: decoded byte count, or a negative zxc_error_t
 *   d_dict    dictionary content or NULL; d_dict_huf its 128-byte table or NULL
 *   d_scratch zxc_b200_decode_scratch_size(block_size) bytes
 *   verify_checksums  non-zero: jobs carry a trailing rapidhash fold, check it
 * Returns ZXC_OK once the launch is enqueued, or a negative code. */
ZXC_EXPORT int zxc_b200_decode_blocks(const void* d_src, void* d_dst, const zxc_b200_job_t* d_jobs,
                                      uint32_t n_jobs, int32_t* d_status, const void* d_dict,
                                      uint32_t dict_size, const void* d_dict_huf, void* d_scratch,
                                      size_t scratch_size, uint32_t block_size,
                                      int verify_checksums, void* stream);

/* Reduce a status array (device) to the reference's frame verdict: total bytes
 * if every job produced exactly its dst_cap, else the first failing job's code
 * in stream order (ZXC_ERROR_CORRUPT_DATA for a size mismatch).  Synchronises
 * `stream`. */
ZXC_EXPORT int64_t zxc_b200_reduce_status(const int32_t* d_status, const zxc_b200_job_t* d_jobs,
                                          uint32_t n_jobs, void* stream);

/* Device scratch that zxc_b200_compress_device needs to compress src_size bytes at these options with the
 * full resident encode grid (0: invalid options, or no device).  At level 6-7 with 64 KiB blocks that is about
 * 1.3 MiB per warp on top of roughly 2 x src_size; a smaller scratch also works, see below. */
ZXC_EXPORT size_t zxc_b200_encode_scratch_size(uint64_t src_size, const zxc_compress_opts_t* opts);

/* Compress src_size bytes at d_src into a complete ZXC frame at d_dst, on `stream`, asynchronously.
 *   opts       as for zxc_compress: level, block_size, checksum_enabled, seekable, and dict / dict_size /
 *              dict_huf in HOST memory, pageable or page-locked (the dictionary has been read when the call
 *              returns: it is staged through a pageable host copy)
 *   d_scratch  device scratch; with less than zxc_b200_encode_scratch_size(...) bytes the encode runs as many
 *              warps as the scratch holds (same output, slower); below one warp's worth the call fails
 *   d_result   one device int64: the frame size, or ZXC_ERROR_DST_TOO_SMALL when the frame does not fit
 *              dst_capacity (the contents of d_dst are then unspecified)
 *   d_jobs     NULL, or ceil(src_size / block_size) entries in device memory: the decode plan of the emitted
 *              frame (what zxc_b200_plan_frame returns for it), ready for zxc_b200_decode_blocks
 * d_dst[0 .. *d_result) equals what zxc_compress returns for the same bytes and options.  d_src and d_dst may have
 * any alignment; nothing outside [d_src, d_src + src_size) is read, and nothing outside d_dst[0 .. dst_capacity),
 * the scratch, *d_result and d_jobs is written.  There is no host synchronisation, no copy through the host and
 * no allocation in the call; without a dictionary it may be captured in a CUDA graph.  Kernel launches per call
 * (zxc_b200_launch_count): 6 when src_size > 0 (encode, three assembly kernels, compaction, finish), plus one
 * dictionary-seeding kernel with a dictionary; 1 for an empty input.
 * Returns ZXC_OK once enqueued, or what the host decides, in zxc_compress's order: ZXC_ERROR_NULL_INPUT (also for a
 * NULL d_scratch or d_result), ZXC_ERROR_DICT_TOO_LARGE, ZXC_ERROR_BAD_BLOCK_SIZE (also for too many blocks),
 * ZXC_B200_ERROR_NO_DEVICE, ZXC_ERROR_DST_TOO_SMALL (dst_capacity below header + trailer), ZXC_ERROR_CORRUPT_DATA
 * (malformed dict_huf), then ZXC_ERROR_MEMORY when the scratch holds less than one warp. */
ZXC_EXPORT int zxc_b200_compress_device(const void* d_src, uint64_t src_size, void* d_dst, uint64_t dst_capacity,
                                        const zxc_compress_opts_t* opts, void* d_scratch, size_t scratch_size,
                                        int64_t* d_result, zxc_b200_job_t* d_jobs, void* stream);

/* Device scratch for zxc_b200_decompress_device: frames whose file-header block size is at most block_size,
 * decoded into at most dst_capacity bytes (0: bad block size, or no device).  It holds a job table of
 * J = ceil(dst_capacity / ZXC_BLOCK_SIZE_MIN) + 2 entries and the decode kernels' per-warp scratch for block_size;
 * on an H100 (132 SMs), 4 GiB of output takes 150 MiB at 4 KiB blocks and 935 MiB at 64 KiB blocks. */
ZXC_EXPORT size_t zxc_b200_decompress_device_scratch_size(uint64_t dst_capacity, uint32_t block_size);

/* Decompress the frame at d_src[0 .. src_size) into d_dst, on `stream`, asynchronously.
 * *d_result (one device int64) becomes exactly what zxc_decompress returns for the same bytes, capacity and opts,
 * and d_dst[0 .. *d_result) equals its output.
 *   opts       as for zxc_decompress: checksum_enabled, and dict / dict_size / dict_huf in HOST memory, pageable or
 *              page-locked (the dictionary has been read when the call returns: it is staged through a pageable
 *              host copy, then copied into the scratch; a call with a dictionary allocates that host copy, may wait
 *              for the stream, and cannot be captured in a CUDA graph)
 *   d_scratch  at least zxc_b200_decompress_device_scratch_size(dst_capacity, B) bytes for some block size B; frames
 *              with blocks larger than the largest such B get ZXC_ERROR_MEMORY in *d_result
 * Returns ZXC_OK once enqueued, or what the host decides without reading the frame, in zxc_decompress's order:
 * ZXC_ERROR_NULL_INPUT (also for a NULL d_scratch or d_result, or a NULL d_dst with dst_capacity > 0),
 * ZXC_ERROR_SRC_TOO_SMALL (src_size below file header + footer), ZXC_ERROR_DICT_TOO_LARGE, ZXC_B200_ERROR_NO_DEVICE,
 * then ZXC_ERROR_MEMORY when the scratch is smaller than zxc_b200_decompress_device_scratch_size(dst_capacity, 4096).
 * The device decides everything that depends on the frame's bytes, in zxc_decompress's order, and writes it to
 * *d_result: the dst_capacity == 0 shortcut (magic, then footer), the file-header rejects, DICT_REQUIRED /
 * DICT_MISMATCH against the header's dictionary id and a malformed dict_huf, the first failing block, capacity,
 * BAD_HEADER at the end of the block stream, the footer size, and the global hash (checked when
 * opts->checksum_enabled and the frame has checksums).  Two limits of this call also give ZXC_ERROR_MEMORY there:
 *   - a header block size larger than the scratch was sized for (decided right after the file-header checks);
 *   - a frame that needs the general re-plan with more blocks ahead of its end than the job table's J entries.  The
 *     re-plan runs when the regular plan (block i at i * block_size) fails with a size mismatch -- a block that
 *     decodes to another size than planned, or runs out of room -- or when blocks do not fit dst_capacity while the
 *     footer's size does.  zxc_decompress then gives a block's error, DST_TOO_SMALL or a size, this call gives
 *     ZXC_ERROR_MEMORY when the frame has more than J blocks.  That takes hand-stitched frames of many short blocks,
 *     or a frame with more than J blocks whose footer was damaged down to at most dst_capacity; a frame the
 *     reference's encoder writes, undamaged, never needs the re-plan.
 * Nothing outside d_dst[0 .. dst_capacity), the scratch and *d_result is written.  Reads of the frame: the planner
 * reads d_src[0 .. src_size) byte by byte, so d_src may have any alignment.  The decode kernels (those of
 * zxc_b200_decode_blocks) copy literal runs with aligned 4-byte loads that reach at most 6 bytes before and 8 bytes
 * past a run.  In a frame that ends with its EOF block and footer every run lies at least 20 bytes before the end,
 * so those loads stay inside d_src[0 .. src_size).  Only a truncated frame, whose last block runs to src_size, may
 * have up to 8 bytes behind d_src + src_size read: keep 8 readable bytes there when frames come from an untrusted
 * source.  d_src and d_dst must not overlap (in-place decode is zxc_decompress_inplace).  Without a dictionary the call makes no host synchronisation and no allocation and may be
 * captured in a CUDA graph.  Kernel launches per call (zxc_b200_launch_count): 12 + k * (2 + c), where k is the
 * number of block sizes from 4 KiB up to B (B = 64 KiB: k = 5) and c = 1 when opts->checksum_enabled, else 0.  The
 * frame is planned on the device (a parallel plan from its SEK table when it has one, else a sequential walk of its
 * block headers), decoded by the same kernels as zxc_b200_decode_blocks, and, for frames whose non-final blocks
 * decode to less than block_size, re-planned and decoded again at the true offsets (see DESIGN.md). */
ZXC_EXPORT int zxc_b200_decompress_device(const void* d_src, uint64_t src_size, void* d_dst, uint64_t dst_capacity,
                                          const zxc_decompress_opts_t* opts, void* d_scratch, size_t scratch_size,
                                          int64_t* d_result, void* stream);

/* ---- random access into a seekable frame in HBM: the device twin of zxc_seekable_open +
 *      zxc_seekable_decompress_range, for many ranges per call ---- */
typedef struct zxc_b200_seekable_device_s zxc_b200_seekable_device;
/* decoded bytes [offset, offset + len) go to d_dst + dst_off */
typedef struct {
    uint64_t offset;
    uint64_t len;
    uint64_t dst_off;
} zxc_b200_range_t;

/* Opens the seekable frame d_src[0 .. src_size) (device memory, borrowed like zxc_seekable_open's src: it must stay
 * valid and unchanged while the handle is used).  Synchronous: the SEK table is parsed on the host from a few copies
 * made on `stream`, and its block offsets (num_blocks + 1 x 8 bytes) are uploaded once to memory the handle owns, on
 * the current device, to which the handle is bound.  Returns NULL exactly where zxc_seekable_open returns NULL for the
 * same bytes, and when there is no device or an allocation fails. */
ZXC_EXPORT zxc_b200_seekable_device* zxc_b200_seekable_device_open(const void* d_src, uint64_t src_size, void* stream);

/* zxc_seekable_set_dict for the device handle: host pointers, the same verdicts in the same order (NULL_INPUT,
 * DICT_TOO_LARGE, DICT_MISMATCH; a rejected call leaves the handle unchanged), then ZXC_ERROR_MEMORY when the device
 * copy cannot be allocated (the previous dictionary is dropped then, as zxc_seekable_set_dict does).  The dictionary and
 * its 128-byte table are copied to the device here, once; the call waits for the handle's device before it frees a
 * previous copy. */
ZXC_EXPORT int zxc_b200_seekable_device_set_dict(zxc_b200_seekable_device* h, const void* dict, size_t dict_size,
                                                 const void* dict_huf);
ZXC_EXPORT uint32_t zxc_b200_seekable_device_num_blocks(const zxc_b200_seekable_device* h);
ZXC_EXPORT uint64_t zxc_b200_seekable_device_decompressed_size(const zxc_b200_seekable_device* h);
ZXC_EXPORT uint32_t zxc_b200_seekable_device_block_size(const zxc_b200_seekable_device* h);

/* Device scratch for one zxc_b200_seekable_device_decompress_ranges call of at most max_ranges ranges whose lengths
 * add up to at most max_bytes (0: NULL handle, no device, or a size that cannot be planned).  Every range decodes
 * whole blocks: a block it covers whole decodes in place in d_dst, a block it covers in part (at most its first and
 * last) into a slot of block_size bytes in the scratch.  The slots dominate for many small ranges: 2 x max_ranges x
 * block_size, so 1 024 ranges at 64 KiB blocks take 128 MiB and 16 384 ranges 2 GiB.  On top come the job table
 * (28 bytes per block of max_bytes), about 90 bytes per range, and the decode kernels' per-warp scratch: one region
 * of about 2.7 x block_size (180 KiB at 64 KiB blocks, 5.3 MiB at 2 MiB) per warp of the larger of the two decode
 * launches, which run one warp per job up to the resident grid.  That is W = max(ceil(max_bytes / block_size),
 * 2 x max_ranges) warps rounded up to 4, and at most the grid's 4 224 warps on an H100 (132 SMs): a single short range
 * at 2 MiB blocks takes 22 MB, while 2 112 or more ranges, or 4 224 or more blocks of max_bytes, take the full grid:
 * 768 MB at 64 KiB blocks and 23 GB at 2 MiB. */
ZXC_EXPORT size_t zxc_b200_seekable_device_scratch_size(const zxc_b200_seekable_device* h, uint32_t max_ranges,
                                                        uint64_t max_bytes);

/* Decodes n_ranges ranges of the handle's frame on `stream`, asynchronously, with no host synchronisation and no
 * allocation: the call may be captured in a CUDA graph, with or without a dictionary.  A captured call keeps what it
 * read from the handle when it was captured -- the dictionary's device copy, whether one was set, the block table --
 * and the job-table size it took from the scratch: zxc_b200_seekable_device_set_dict or _free invalidates every graph
 * captured on the handle before (a replay would read freed memory, or give the old DICT_REQUIRED), so capture again
 * after either.  The contents of d_ranges, d_dst and d_results may change between replays.  d_ranges (n_ranges entries)
 * and d_results (one int64 per range) are device memory; the call runs on the handle's device and restores the
 * current device.  Calls on different streams with separate scratch may run at the same time.
 * Returns ZXC_OK once enqueued, or what the host decides: ZXC_ERROR_NULL_INPUT for a NULL handle, or for a NULL
 * d_ranges, d_results or d_scratch when n_ranges > 0; ZXC_B200_ERROR_NO_DEVICE; ZXC_ERROR_MEMORY when scratch_size is
 * below zxc_b200_seekable_device_scratch_size(h, n_ranges, 0).  n_ranges == 0 returns ZXC_OK and launches nothing.
 * d_results[i] is what zxc_seekable_decompress_range(s, d_dst + dst_off, cap, offset, len) of this library returns on
 * a handle opened on the same bytes with the same dictionary, where cap = dst_capacity - dst_off (0 when dst_off >
 * dst_capacity), in its order: 0 for len == 0, NULL_INPUT for a NULL d_dst, DST_TOO_SMALL, SRC_TOO_SMALL (also when
 * offset + len wraps), DICT_REQUIRED, then the first covered block in block order that failed (its own code, or
 * CORRUPT_DATA for another size than expected), else len.  Checksums are not verified, as on the host's seekable path.
 * One more verdict of this call comes between DICT_REQUIRED and the blocks: ranges take job-table entries in index
 * order, and from the first range whose blocks no longer fit the table the scratch holds, every range that passed
 * the checks gets ZXC_ERROR_MEMORY and decodes nothing; that happens only when the ranges' lengths add up to more
 * than the max_bytes the scratch was sized for.
 * Nothing outside the union of d_dst[dst_off, dst_off + len) over the ranges, the scratch and d_results is written; a
 * range with a negative result may leave its span partly written, and overlapping spans get unspecified bytes.  Reads
 * of d_src stay inside the bounds documented for zxc_b200_decompress_device.  Kernel launches per call
 * (zxc_b200_launch_count): 8 (plan: 3; the decode kernels' lean and general instance on the blocks decoded in place,
 * then on the slots: 4; finish: 1), whatever the ranges. */
ZXC_EXPORT int zxc_b200_seekable_device_decompress_ranges(zxc_b200_seekable_device* h,
                                                          const zxc_b200_range_t* d_ranges, uint32_t n_ranges,
                                                          void* d_dst, uint64_t dst_capacity, void* d_scratch,
                                                          size_t scratch_size, int64_t* d_results, void* stream);
ZXC_EXPORT void zxc_b200_seekable_device_free(zxc_b200_seekable_device* h);

/* Kernels launched by this library since load (for bench.py's gpu_launches). */
ZXC_EXPORT uint64_t zxc_b200_launch_count(void);

/* Resident CTAs per SM that the occupancy calculator gives the lean and the general block-decode kernel (dictionary-free
 * instances) at the dynamic shared memory they launch with, for profiles/occupancy_probe.py.  0 on success. */
ZXC_EXPORT int zxc_b200_decode_occupancy(int* lean, int* general);

/* Phase times (ms) of the calling thread's last dictionary-training calls, for profiles/train_bench.py: upload,
 * count, segments, host sort, pick (zxc_train_dict); slice upload, histogram encode, code lengths
 * (zxc_train_dict_huf).  Writes min(n, 8) entries and returns their number. */
ZXC_EXPORT int zxc_b200_train_phase_times(double* ms, int n);

#ifdef __cplusplus
}
#endif
#endif /* ZXC_B200_H */
