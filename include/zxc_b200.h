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
#include "zxc_pstream.h"

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
 * source.  d_src and d_dst must not overlap (in-place decode is zxc_b200_decompress_inplace_device).  Without a dictionary the call makes no host synchronisation and no allocation and may be
 * captured in a CUDA graph.  Kernel launches per call (zxc_b200_launch_count): 12 + k * (2 + c), where k is the
 * number of block sizes from 4 KiB up to B (B = 64 KiB: k = 5) and c = 1 when opts->checksum_enabled, else 0.  The
 * frame is planned on the device (a parallel plan from its SEK table when it has one, else a sequential walk of its
 * block headers), decoded by the same kernels as zxc_b200_decode_blocks, and, for frames whose non-final blocks
 * decode to less than block_size, re-planned and decoded again at the true offsets (see DESIGN.md). */
ZXC_EXPORT int zxc_b200_decompress_device(const void* d_src, uint64_t src_size, void* d_dst, uint64_t dst_capacity,
                                          const zxc_decompress_opts_t* opts, void* d_scratch, size_t scratch_size,
                                          int64_t* d_result, void* stream);

/* ---- in-place decode in HBM: the device twin of zxc_decompress_inplace ---- */
/* Device scratch for zxc_b200_decompress_inplace_device with buffers of at most buffer_capacity bytes, frames whose
 * header block size is at most block_size, and a staging window of `window` compressed bytes per round (0: bad block
 * size, no device, or a capacity too large to plan).  It is zxc_b200_decompress_device_scratch_size(buffer_capacity,
 * block_size), plus two round tables of 28 x min(J, window / 8 + 1) bytes, 8 bytes per smallest window of the buffer
 * and a staging area of window + block_size + 76 bytes (rounded up to 256-byte regions).  Windows are whole multiples
 * of 4 KiB: `window` is rounded up to one, raised to the smallest window W_min = 4 x block_size + 4096, and lowered to
 * buffer_capacity rounded up to 4 KiB, which decodes any frame in the buffer in one round. */
ZXC_EXPORT size_t zxc_b200_decompress_inplace_device_scratch_size(uint64_t buffer_capacity, uint32_t block_size,
                                                                 uint64_t window);

/* zxc_decompress_inplace_bound for a frame in device memory, d_src[0 .. src_size): reads its 16 header bytes and its
 * footer with two copies on `stream`, which it synchronises.  0 where zxc_decompress_inplace_bound gives 0, and
 * without a device. */
ZXC_EXPORT size_t zxc_b200_decompress_inplace_device_bound(const void* d_src, uint64_t src_size, void* stream);

/* Decodes the frame of comp_size bytes that lies flush-right in d_buffer[0 .. buffer_capacity) (device memory) into
 * d_buffer[0 ..), on `stream`, asynchronously, with no second buffer: the device memory it takes is the buffer and
 * the scratch, against frame + output + scratch for zxc_b200_decompress_device.
 * *d_result (one device int64) and d_buffer[0 .. *d_result) when it is not negative become exactly what this
 * library's zxc_decompress_inplace returns and writes for the same buffer contents, buffer_capacity, comp_size and
 * opts, but for the two limits below; frames the reference's encoder writes never reach them.  (The reference's
 * zxc_decompress_inplace also rejects buffer_capacity - comp_size < block_size + 2112; neither call does.)
 *   opts       as for zxc_b200_decompress_device: checksum_enabled, and a dictionary in HOST memory, staged the same
 *              way (a host copy: the call then may wait for the stream and cannot be captured in a CUDA graph)
 *   d_scratch  zxc_b200_decompress_inplace_device_scratch_size(buffer_capacity, b, window) bytes; the call finds the
 *              block size B and the window W from scratch_size and buffer_capacity alone: B is the largest block size
 *              whose layout with the smallest window fits, and W the largest window (a multiple of 4 KiB, up to
 *              buffer_capacity rounded up to 4 KiB) that then fits.  Frames with blocks larger than B get ZXC_ERROR_MEMORY in *d_result, as from
 *              zxc_b200_decompress_device.  A scratch sized for (b, window) gives B = b and W = window unless the
 *              window is larger than the growth of the decode kernels' per-warp scratch from b to 2b, about 2.7 x b
 *              per warp for one warp per 4 KiB of buffer_capacity, up to the resident grid (4 224 warps on an H100):
 *              never for buffers below about 17 MiB, else above about 47 MiB at 4 KiB blocks and 730 MiB at 64 KiB.
 *              Such a window gives a larger B and a smaller W: the same result, in more rounds.
 * Returns ZXC_OK once enqueued, or what the host decides without reading the buffer, in this order:
 * ZXC_ERROR_NULL_INPUT (a NULL d_buffer, comp_size below file header + footer or above buffer_capacity, as
 * zxc_decompress_inplace; also a NULL d_scratch or d_result), ZXC_ERROR_DICT_TOO_LARGE, ZXC_B200_ERROR_NO_DEVICE, then
 * ZXC_ERROR_MEMORY when the scratch is below zxc_b200_decompress_inplace_device_scratch_size(buffer_capacity, 4096, 0).
 * The device writes the rest to *d_result, in zxc_decompress_inplace's order: its own checks first (BAD_MAGIC,
 * BAD_HEADER for any file-header reject, CORRUPT_DATA for a footer size the frame cannot hold, DST_TOO_SMALL when
 * buffer_capacity is below the decoded size plus zxc_decompress_inplace_bound's margin), then everything
 * zxc_b200_decompress_device decides for d_src = d_buffer + buffer_capacity - comp_size, d_dst = d_buffer and
 * dst_capacity = buffer_capacity, with that call's limits.  Two limits of this call give ZXC_ERROR_MEMORY as well:
 *   (a) the round schedule cannot decode the frame without overwriting compressed bytes a later round still has to
 *       stage, or a block is longer on disk than B + 12 bytes (the largest block the reference's encoder writes) and
 *       would not fit its round's staged copy.  This is decided after the plan and before the first byte of the buffer
 *       is written: the buffer is then unchanged.  Only a frame with more than one round can reach it;
 *   (b) the frame needs zxc_b200_decompress_device's general re-plan (non-final blocks that decode to less than the
 *       block size) and the call runs more than one round.
 * With one round (W >= comp_size) neither applies.  On any other negative result the buffer's contents are
 * unspecified: the decode is in place, so the frame is consumed.
 * How it works (DESIGN.md section 7j): the frame is planned where it lies; then, in R = ceil(comp_size / W) rounds,
 * round k copies frame bytes [k W - 8, min((k + 1) W + B + 20, comp_size)) into the scratch and decodes the blocks
 * whose headers lie in [k W, (k + 1) W) from that copy into the buffer.
 * Nothing outside d_buffer[0 .. buffer_capacity), the scratch and *d_result is written, and nothing outside
 * d_buffer[0 .. buffer_capacity) is read: the decode kernels read the staged copy, so their read-past stays inside
 * the scratch; d_buffer may have any alignment.  Without a dictionary there is no host synchronisation and no
 * allocation, and the call may be captured in a CUDA graph; a replay consumes the frame, so restore the buffer before
 * each one.  Kernel launches per call (zxc_b200_launch_count): 16 + R * (1 + k * (2 + c)), k and c as for
 * zxc_b200_decompress_device with the B above (plan: 6, the in-place probe and the round plan: 2; per round one table
 * kernel and the decode kernels; the last round's gather, check, decide, the re-plan limit: 4; the general split: 4);
 * R and k follow from (comp_size, buffer_capacity, scratch_size).  Each round also makes one device-to-device copy. */
ZXC_EXPORT int zxc_b200_decompress_inplace_device(void* d_buffer, uint64_t buffer_capacity, uint64_t comp_size,
                                                  const zxc_decompress_opts_t* opts, void* d_scratch,
                                                  size_t scratch_size, int64_t* d_result, void* stream);

/* ---- many device-resident frames in one call: zxc_b200_decompress_device over a batch ---- */
/* one frame of a batch; the array of them lives in DEVICE memory */
typedef struct {
    const void* src;       /* the frame, device memory */
    uint64_t src_size;
    void* dst;             /* its output, device memory */
    uint64_t dst_capacity;
} zxc_b200_frame_t;

/* Device scratch for one zxc_b200_decompress_device_batch call of at most max_frames frames whose dst_capacity values
 * add up to at most max_total_capacity, with blocks of at most block_size bytes (0: bad block size, no device, more
 * than 2^30 frames, or a table too large to plan).  It holds a job table of
 * Jt = ceil(max_total_capacity / ZXC_BLOCK_SIZE_MIN) + 3 x max_frames entries: 28 bytes each for the plan and the
 * split, and a window of 28 bytes each per launch slot (2 per block size from 4 KiB up to block_size: 10 at 64 KiB);
 * about 170 bytes per frame; and the decode kernels' per-warp scratch for the full resident grid at block_size
 * (on an H100, 132 SMs: 83 MiB at 4 KiB blocks, 732 MiB at 64 KiB, whatever the batch). */
ZXC_EXPORT size_t zxc_b200_decompress_device_batch_scratch_size(uint32_t max_frames, uint64_t max_total_capacity,
                                                                uint32_t block_size);

/* Decompresses n_frames independent frames on `stream`, asynchronously: d_frames[i] names frame i's bytes
 * src[0 .. src_size) and its output dst[0 .. dst_capacity), all in device memory.  d_results[i] (one device int64
 * per frame) becomes exactly what zxc_b200_decompress_device returns in *d_result for that frame with the same opts
 * and a scratch of zxc_b200_decompress_device_scratch_size(dst_capacity, B), and dst[0 .. d_results[i]) equals its
 * output; B is the block size the scratch was sized for (below).  The device also makes that call's host checks per
 * frame, in zxc_decompress's order: ZXC_ERROR_NULL_INPUT for a NULL src, or a NULL dst with dst_capacity > 0, then
 * ZXC_ERROR_SRC_TOO_SMALL for src_size below file header + footer.
 * Returns ZXC_OK once enqueued, or a verdict for the whole call that replaces every frame's own (d_results is then
 * not written), in this order: ZXC_ERROR_NULL_INPUT for a NULL d_frames, d_results or d_scratch when n_frames > 0;
 * ZXC_ERROR_DICT_TOO_LARGE; ZXC_B200_ERROR_NO_DEVICE; ZXC_ERROR_MEMORY when scratch_size is below
 * zxc_b200_decompress_device_batch_scratch_size(n_frames, 0, 4096).  n_frames == 0 returns ZXC_OK (after the
 * dictionary and device checks) and launches nothing.
 * The scratch: B is the largest block size whose layout with the smallest table (max_total_capacity 0) fits
 * scratch_size, and the call then takes the largest job table that fits at B.  A scratch from
 * zxc_b200_decompress_device_batch_scratch_size(n, C, b) gives B = b as long as the table's share of it is below the
 * per-warp regions' step to 2b (C below about 2 GiB at 4 KiB blocks, 9 GiB at 64 KiB).  Frames take ceil(dst_capacity /
 * ZXC_BLOCK_SIZE_MIN) + 2 table entries each, in index order (frames that fail the argument checks take none); from
 * the first frame whose entries no longer fit the table, every later frame that passed the argument checks gets
 * ZXC_ERROR_MEMORY and decodes nothing.  That happens only when the capacities add up to more than the
 * max_total_capacity the scratch was sized for.
 * Nothing outside the union of the frames' dst[0 .. dst_capacity), the scratch and d_results is written; overlapping
 * outputs get unspecified bytes.  Reads of each src stay inside the bounds documented for zxc_b200_decompress_device.
 * There is no host synchronisation and no allocation without a dictionary, and the call may then be captured in a
 * CUDA graph; d_frames, the frames' bytes and d_results may change between replays.  A dictionary (one for the whole
 * batch, host memory) is staged as in zxc_b200_decompress_device: a host copy, not capturable.  Kernel launches per
 * call (zxc_b200_launch_count): 14 + k * (2 + c) whatever the frames, k and c as for zxc_b200_decompress_device with
 * the B above (plan: 8; the decode kernels' lean and general instance per slot; check and decide: 2; the general
 * split: 4, which exit at once when no frame needs it). */
ZXC_EXPORT int zxc_b200_decompress_device_batch(const zxc_b200_frame_t* d_frames, uint32_t n_frames,
                                                const zxc_decompress_opts_t* opts, void* d_scratch,
                                                size_t scratch_size, int64_t* d_results, void* stream);

/* ---- many device-resident buffers in one call: zxc_b200_compress_device over a batch ---- */
/* Device scratch for one zxc_b200_compress_device_batch call of at most max_frames buffers whose src_size values add
 * up to at most max_total_src, at these options (0: invalid options, no device, more than 2^30 buffers, or more than
 * 2^50 bytes).  It holds about 112 bytes per buffer; a pool with each buffer's share (below); 12 bytes per block the
 * pool can hold; and one encode slot per warp (zxc_b200_encode_scratch_size's per-warp share) for the full resident
 * grid, or for one warp per block the pool can hold when that is fewer.  On an H100 (132 SMs, 4 224 warps), 4 096
 * buffers of 64 KiB take about 2.8 GB at level 3 and 6.1 GB at level 6. */
ZXC_EXPORT size_t zxc_b200_compress_device_batch_scratch_size(uint32_t max_frames, uint64_t max_total_src,
                                                              const zxc_compress_opts_t* opts);

/* Compresses n_frames independent buffers on `stream`, asynchronously, into one ZXC frame each: d_frames[i] (device
 * memory) names buffer i's bytes src[0 .. src_size) and its frame's room dst[0 .. dst_capacity), all in device memory.
 * d_results[i] (one device int64 per buffer) becomes exactly what zxc_b200_compress_device gives that buffer alone in
 * *d_result with the same opts, and dst[0 .. d_results[i]) equals its frame, so both equal zxc_compress's result and
 * bytes.  One set of opts applies to the whole batch: level, block_size, checksum_enabled, seekable and one dictionary
 * in HOST memory (read before the call returns, as for zxc_b200_compress_device).
 * Per buffer, the device makes zxc_b200_compress_device's host checks in its order: ZXC_ERROR_NULL_INPUT for a NULL
 * dst, dst_capacity 0, or a NULL src with src_size > 0; ZXC_ERROR_BAD_BLOCK_SIZE for more than 2^32 - 3 blocks;
 * ZXC_ERROR_DST_TOO_SMALL for dst_capacity below header + trailer (which depends on the block count and seekable).
 * Then the pool rule below (ZXC_ERROR_MEMORY), and last ZXC_ERROR_DST_TOO_SMALL for a frame whose body does not fit
 * (dst is then left untouched).
 * Returns ZXC_OK once enqueued, or a verdict for the whole call that replaces every buffer's own (d_results is then
 * not written), in zxc_b200_compress_device's order: ZXC_ERROR_NULL_INPUT for a NULL d_frames, d_results or d_scratch
 * when n_frames > 0; ZXC_ERROR_DICT_TOO_LARGE; ZXC_ERROR_BAD_BLOCK_SIZE from the options; ZXC_B200_ERROR_NO_DEVICE;
 * ZXC_ERROR_CORRUPT_DATA for a malformed dict_huf; ZXC_ERROR_MEMORY when scratch_size is below
 * zxc_b200_compress_device_batch_scratch_size(n_frames, 0, opts).  n_frames == 0 returns ZXC_OK after those option,
 * dictionary and device checks and launches nothing.
 * The scratch: past about 112 bytes per buffer and the dictionary comes the room: a pool of P bytes, then one encode
 * slot.  A non-empty buffer's share of the pool is its padded input copy, r256(src_size + 64) bytes, plus one staging
 * slot of r256(block_size + 80) bytes per block; an empty buffer takes none.  Buffers take their shares in index order;
 * from the first buffer whose share no longer fits, every later buffer that passed the checks gets ZXC_ERROR_MEMORY
 * and nothing is written for it.  P is a function of (scratch_size, n_frames, opts) alone: the largest pool whose
 * layout fits, where the layout holds, beside the room, a 4-byte size and an 8-byte offset for each of the
 * nb_max = max(1, P / (r256(block_size + 80) + 256)) blocks such a pool can hold.  The encode runs up to
 * W = min(resident encode grid, nb_max) warps (rounded down to a multiple of 4 from 4 up), one encode slot each,
 * counted down from the room's end: every slot that fits in the part of the room the batch's shares leave free runs a
 * warp, so a scratch from zxc_b200_compress_device_batch_scratch_size(n, T, opts) gives any batch of at most n
 * buffers of at most T bytes no ZXC_ERROR_MEMORY and W warps, and a smaller one that still holds the shares runs fewer
 * warps (down to one: same output, slower).
 * Nothing outside [src, src + src_size) of each buffer is read, whatever its alignment; nothing outside the union of
 * the dst[0 .. dst_capacity), the scratch and d_results is written, and overlapping outputs get unspecified bytes.
 * There is no host synchronisation, no copy through the host and no allocation without a dictionary, and the call may
 * then be captured in a CUDA graph; d_frames, the buffers' bytes and d_results may change between replays.  Kernel
 * launches per call (zxc_b200_launch_count): 12 whatever the buffers (plan: 3; gather; encode; assembly: 5;
 * compaction; finish), plus one dictionary-seeding kernel with a dictionary. */
ZXC_EXPORT int zxc_b200_compress_device_batch(const zxc_b200_frame_t* d_frames, uint32_t n_frames,
                                              const zxc_compress_opts_t* opts, void* d_scratch, size_t scratch_size,
                                              int64_t* d_results, void* stream);

/* ---- the block API in HBM: zxc_compress_block / zxc_decompress_block(_safe) over a batch of frameless blocks ---- */
/* Device scratch for one zxc_b200_compress_blocks_device call of at most max_blocks items whose src_size values add
 * up to at most max_total_src, none above max_src_size bytes, at these options (0: a dictionary above
 * ZXC_DICT_SIZE_MAX, no device, more than 2^30 items, more than 2^50 bytes, or max_src_size above
 * ZXC_BLOCK_SIZE_MAX).  It is about 72 bytes per item, the dictionary's region, a pool of at most 2 x max_total_src +
 * 586 x max_blocks bytes (each item's share, below), and one encode slot (zxc_b200_encode_scratch_size's per-warp
 * share at block size B = zxf_block_size_ceil(max_src_size)) for each of W = min(max_blocks, max_total_src, resident
 * encode grid) warps (at least one), rounded down to a multiple of 4 from 4 up: on an H100 (132 SMs, 4 224 warps), 2^20 items of 4 KiB at level 5
 * take about 10.3 GB. */
ZXC_EXPORT size_t zxc_b200_compress_blocks_device_scratch_size(uint32_t max_blocks, uint64_t max_total_src,
                                                               uint32_t max_src_size, const zxc_compress_opts_t* opts);

/* Compresses n_items independent frameless blocks on `stream`, asynchronously: d_items[i] (device memory) names item
 * i's bytes src[0 .. src_size) and its block's room dst[0 .. dst_capacity), all in device memory.  d_results[i] (one
 * device int64 per item) and dst[0 .. d_results[i]) become exactly what this library's zxc_compress_block returns and
 * writes for item i on a fresh zxc_create_cctx(NULL) context with the same opts, and so what the reference's
 * zxc_compress_block gives (a block's bytes depend on its content, level, checksum flag and dictionary only, not on
 * opts->block_size).  opts == NULL means level 3 without checksums; the call uses level, checksum_enabled and one
 * dictionary (dict / dict_size in HOST memory, read before the call returns, as for zxc_b200_compress_device);
 * dict_huf and block_size are ignored, as by the host block API.
 * Per item, in zxc_compress_block's order: ZXC_ERROR_NULL_INPUT for a NULL src or dst, src_size 0 or dst_capacity 0;
 * ZXC_ERROR_BAD_BLOCK_SIZE for src_size above ZXC_BLOCK_SIZE_MAX; ZXC_ERROR_MEMORY by the room rule below; last
 * ZXC_ERROR_DST_TOO_SMALL when the block does not fit dst_capacity (dst is then left untouched).
 * Returns ZXC_OK once enqueued, or a verdict for the whole call that replaces every item's own (d_results is then not
 * written), in this order: ZXC_ERROR_NULL_INPUT for a NULL d_items, d_results or d_scratch when n_items > 0;
 * ZXC_ERROR_DICT_TOO_LARGE; ZXC_B200_ERROR_NO_DEVICE; ZXC_ERROR_MEMORY when scratch_size is below
 * zxc_b200_compress_blocks_device_scratch_size(n_items, 0, 0, opts): the item records and one encode slot at 4 KiB.  n_items == 0 returns ZXC_OK after those checks and launches nothing.
 * The scratch: past about 72 bytes per item and the dictionary comes the room.  Items that pass the checks take their
 * share of it in index order from its start: an input copy of r256(src_size + 64) bytes and a staging slot of
 * r256(src_size + 12) bytes (the most the encoder writes for a block: a RAW block with its checksum).  The encode
 * slots are laid out for B, the largest zxf_block_size_ceil(src_size) among the admitted items, and counted down from
 * the room's end.  Item i is admitted when the shares of the admitted items up to it plus one encode slot at B fit the
 * room; from the first item that is not, it and every later item that passed the checks get ZXC_ERROR_MEMORY and
 * nothing is written for them.  B and the room follow from scratch_size and the items alone: there is no block size
 * to choose.  The call launches W warps (W as in the size query, for n_items), and every one whose slot fits the part
 * of the room the admitted shares leave free runs (W for n_items items: min(n_items, resident grid)), so a scratch
 * from zxc_b200_compress_blocks_device_scratch_size(n, T, m, opts) gives any batch of at most n items of at most T bytes
 * in all and m bytes each no ZXC_ERROR_MEMORY and that query's W warps, and a smaller one runs fewer warps (down to
 * one: same output, slower).
 * Nothing outside [src, src + src_size) of each item is read, whatever its alignment; nothing outside the union of the
 * dst[0 .. dst_capacity), the scratch and d_results is written, and overlapping outputs get unspecified bytes.  There
 * is no host synchronisation and no allocation without a dictionary, and the call may then be captured in a CUDA
 * graph; d_items, the items' bytes and d_results may change between replays.  Kernel launches per call
 * (zxc_b200_launch_count): 5 whatever the items (checks and shares, scan, gather, encode, fit and copy-out), plus one
 * dictionary-seeding kernel with a dictionary. */
ZXC_EXPORT int zxc_b200_compress_blocks_device(const zxc_b200_frame_t* d_items, uint32_t n_items,
                                               const zxc_compress_opts_t* opts, void* d_scratch, size_t scratch_size,
                                               int64_t* d_results, void* stream);

/* Device scratch for one zxc_b200_decompress_blocks_device call of at most max_blocks items, none with a dst_capacity
 * above max_dst_capacity (0: no device, or more than 2^30 items).  B = zxf_block_size_ceil(max_dst_capacity); it
 * holds, per item, 16 bytes and one job and status word in each of the k x 2 launch slots (k block sizes from 4 KiB up
 * to B, 28 bytes each), the dictionary's region (ZXC_DICT_SIZE_MAX) and the decode kernels' per-warp scratch at B for
 * max_blocks jobs (one warp per job up to the resident grid): on an H100, 2^20 items at 4 KiB take about 160 MiB. */
ZXC_EXPORT size_t zxc_b200_decompress_blocks_device_scratch_size(uint32_t max_blocks, uint64_t max_dst_capacity);

/* Decompresses n_items independent frameless blocks on `stream`, asynchronously: d_items[i] (device memory) names item
 * i's block src[0 .. src_size) and its output dst[0 .. dst_capacity), all in device memory.  d_results[i] (one device
 * int64 per item) and dst[0 .. d_results[i]) become exactly what this library's zxc_decompress_block returns and
 * writes for item i (zxc_decompress_block_safe when safe != 0) with the same opts: checksums verified when
 * opts->checksum_enabled, dict / dict_size (HOST memory, one for the batch, staged as for zxc_b200_decompress_device)
 * used as there, dict_huf ignored as there.  On a negative result the item's dst holds unspecified bytes.
 * Per item: ZXC_ERROR_NULL_INPUT for a NULL src or dst, src_size below 8 or dst_capacity 0; ZXC_ERROR_BAD_BLOCK_SIZE
 * for dst_capacity above ZXC_BLOCK_SIZE_MAX + 2112 (safe: above ZXC_BLOCK_SIZE_MAX); ZXC_ERROR_MEMORY when
 * zxf_block_size_ceil(dst_capacity) is above the block size B the scratch was sized for; then the block's own verdict
 * from the decode kernels of zxc_b200_decode_blocks, run on the job {src, dst, min(src_size, 2^32 - 1), dst_capacity}
 * at block size zxf_block_size_ceil(dst_capacity), exactly as zxc_decompress_block builds it.
 * Returns ZXC_OK once enqueued, or a verdict for the whole call that replaces every item's own (d_results is then not
 * written): ZXC_ERROR_NULL_INPUT for a NULL d_items, d_results or d_scratch when n_items > 0;
 * ZXC_ERROR_DICT_TOO_LARGE; ZXC_B200_ERROR_NO_DEVICE; ZXC_ERROR_MEMORY when scratch_size is below
 * zxc_b200_decompress_blocks_device_scratch_size(n_items, 4096).  n_items == 0 returns ZXC_OK after those checks and
 * launches nothing.  B is the largest block size whose layout for n_items items fits scratch_size, so a scratch from
 * zxc_b200_decompress_blocks_device_scratch_size(n, C) gives every batch of at most n items of capacity at most C a B
 * of at least zxf_block_size_ceil(C), and the job table always holds every item.
 * Reads: the decode kernels copy literal runs with aligned 4-byte loads that reach at most 6 bytes before and 8 bytes
 * past a run.  A run starts behind the 8-byte block header, and in a GLO or GHI block the encoder's format keeps every
 * literal at least 32 bytes before the payload's end, but a RAW block's run ends where the payload ends: without a
 * checksum that is src + src_size.  So keep 8 readable bytes behind src + src_size (blocks packed back to back in one
 * allocation have them, but for the last); nothing before src is read.  d_items and d_results must not overlap the
 * outputs.  Nothing outside the union of the dst[0 .. dst_capacity), the scratch and d_results is written.  There is no
 * host synchronisation and no allocation without a dictionary, and the call may then be captured in a CUDA graph;
 * d_items, the blocks' bytes and d_results may change between replays.  Kernel launches per call
 * (zxc_b200_launch_count): 4 + k x (2 + c) whatever the items, k the number of block sizes from 4 KiB up to B and c = 1
 * when opts->checksum_enabled, else 0 (plan: 3; per block size the decode kernels' lean and general instance, and the
 * verifying instance with checksums; finish: 1). */
ZXC_EXPORT int zxc_b200_decompress_blocks_device(const zxc_b200_frame_t* d_items, uint32_t n_items,
                                                 const zxc_decompress_opts_t* opts, int safe, void* d_scratch,
                                                 size_t scratch_size, int64_t* d_results, void* stream);

/* ---- prepared dictionaries in HBM: load a dictionary once, use it in every device-to-device call ---- */
typedef struct zxc_b200_dict_device_s zxc_b200_dict_device;

/* Prepares the dictionary dict[0 .. dict_size) and its optional 128-byte literal table dict_huf (HOST memory, pageable
 * or page-locked; read before the call returns, so the caller may free or overwrite them afterwards) for the
 * _using_dict calls below.  Synchronous on `stream` (a cudaStream_t, NULL = legacy default stream): the call returns
 * once the device copy is complete.  The handle owns one device allocation on the CUDA device current at creation, to
 * which it is bound, of about 2 x dict_size + 520 KiB: the dictionary as the decode calls stage it (its table right
 * behind it when the table is usable), and as the compress calls stage it (zero-padded, with the match tables that
 * zxc_seed_kernel seeds for levels 1-2 and for levels 3-7, and the table's 256 code lengths).  Creation runs two
 * seeding kernels.  A malformed dict_huf is not rejected here: the handle keeps the verdicts the calls would make about
 * it, and every _using_dict call gives them where its base call does (ZXC_ERROR_CORRUPT_DATA from the frame compress
 * calls, the device verdict of the frame decode calls).
 * Returns NULL and sets *err (err may be NULL; ZXC_OK on success), in this order: ZXC_ERROR_NULL_INPUT for a NULL dict
 * or dict_size 0; ZXC_ERROR_DICT_TOO_LARGE above ZXC_DICT_SIZE_MAX; ZXC_B200_ERROR_NO_DEVICE; ZXC_ERROR_MEMORY or
 * ZXC_B200_ERROR_CUDA when the device memory cannot be allocated or filled. */
ZXC_EXPORT zxc_b200_dict_device* zxc_b200_dict_device_create(const void* dict, size_t dict_size, const void* dict_huf,
                                                             int* err, void* stream);
/* zxc_dict_id(dict, dict_size, dict_huf) of the bytes the handle was created from (0 for NULL) */
ZXC_EXPORT uint32_t zxc_b200_dict_device_id(const zxc_b200_dict_device* dd);
/* the dictionary's content bytes (0 for NULL) */
ZXC_EXPORT size_t zxc_b200_dict_device_size(const zxc_b200_dict_device* dd);
/* Waits for the handle's device (calls in flight on any stream may still read the handle), then frees it.  Graphs
 * captured with the handle are invalid afterwards.  NULL is a no-op. */
ZXC_EXPORT void zxc_b200_dict_device_free(zxc_b200_dict_device* dd);

/* The _using_dict variants.  Each takes its base call's arguments plus dd right after opts, and returns, writes to its
 * result words and writes to its outputs exactly what the base call does when opts->dict, dict_size and dict_huf are
 * replaced by the bytes dd was created from; with dd == NULL, what the base call does without a dictionary.  opts' own
 * dictionary fields are ignored, so the base call's DICT_TOO_LARGE never comes.  The differences:
 *   - No staging: the call makes no host copy, allocation or synchronisation, with or without a handle, so it may be
 *     captured in a CUDA graph (which keeps reading the handle: free it only after the graph's last replay).
 *   - Kernel launches (zxc_b200_launch_count): the compress variants launch no seeding kernel, so they make the base
 *     call's dictionary-free count (6 for zxc_b200_compress_device, 1 for an empty input; 12 for _batch; 5 for
 *     _blocks); the decode variants make the base call's count.
 *   - Scratch: the compress variants' layouts are the base call's layouts for opts without a dictionary, so the size
 *     queries with opts->dict = NULL give their scratch, and the pool and admission rules of _batch and _blocks are
 *     those of a dictionary-free call (a larger scratch works too).  The results equal the base call's wherever
 *     neither call reaches a scratch-capacity ZXC_ERROR_MEMORY.  The decode layouts are unchanged; their dictionary
 *     region is left unused.
 *   - A handle bound to another device than the current one gives ZXC_B200_ERROR_NO_DEVICE where the base call checks
 *     for a device.
 * The handle is only read by the calls: any number of calls on any streams and threads may share it. */
ZXC_EXPORT int zxc_b200_compress_device_using_dict(const void* d_src, uint64_t src_size, void* d_dst,
                                                   uint64_t dst_capacity, const zxc_compress_opts_t* opts,
                                                   const zxc_b200_dict_device* dd, void* d_scratch, size_t scratch_size,
                                                   int64_t* d_result, zxc_b200_job_t* d_jobs, void* stream);
ZXC_EXPORT int zxc_b200_compress_device_batch_using_dict(const zxc_b200_frame_t* d_frames, uint32_t n_frames,
                                                         const zxc_compress_opts_t* opts,
                                                         const zxc_b200_dict_device* dd, void* d_scratch,
                                                         size_t scratch_size, int64_t* d_results, void* stream);
/* as zxc_b200_compress_blocks_device, the handle's literal table is not attached */
ZXC_EXPORT int zxc_b200_compress_blocks_device_using_dict(const zxc_b200_frame_t* d_items, uint32_t n_items,
                                                          const zxc_compress_opts_t* opts,
                                                          const zxc_b200_dict_device* dd, void* d_scratch,
                                                          size_t scratch_size, int64_t* d_results, void* stream);
ZXC_EXPORT int zxc_b200_decompress_device_using_dict(const void* d_src, uint64_t src_size, void* d_dst,
                                                     uint64_t dst_capacity, const zxc_decompress_opts_t* opts,
                                                     const zxc_b200_dict_device* dd, void* d_scratch,
                                                     size_t scratch_size, int64_t* d_result, void* stream);
ZXC_EXPORT int zxc_b200_decompress_inplace_device_using_dict(void* d_buffer, uint64_t buffer_capacity,
                                                             uint64_t comp_size, const zxc_decompress_opts_t* opts,
                                                             const zxc_b200_dict_device* dd, void* d_scratch,
                                                             size_t scratch_size, int64_t* d_result, void* stream);
ZXC_EXPORT int zxc_b200_decompress_device_batch_using_dict(const zxc_b200_frame_t* d_frames, uint32_t n_frames,
                                                           const zxc_decompress_opts_t* opts,
                                                           const zxc_b200_dict_device* dd, void* d_scratch,
                                                           size_t scratch_size, int64_t* d_results, void* stream);
/* as zxc_b200_decompress_blocks_device, the handle's literal table is not attached */
ZXC_EXPORT int zxc_b200_decompress_blocks_device_using_dict(const zxc_b200_frame_t* d_items, uint32_t n_items,
                                                            const zxc_decompress_opts_t* opts,
                                                            const zxc_b200_dict_device* dd, int safe, void* d_scratch,
                                                            size_t scratch_size, int64_t* d_results, void* stream);

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

/* ---- push streaming in HBM: the device twins of zxc_cstream_* / zxc_dstream_* (include/zxc_pstream.h) ---- */
typedef struct zxc_b200_cstream_device_s zxc_b200_cstream_device;
typedef struct zxc_b200_dstream_device_s zxc_b200_dstream_device;

/* Streams whose chunks live in device memory: in->src and out->dst are device pointers on the handle's device (any
 * alignment); the pos / size fields are host values, as for the host streams.
 * Call for call identical to the reference: fed the same chunks and out capacities in the same order as the
 * reference's zxc_cstream_* / zxc_dstream_*, every call gives the same return value, in->pos and out->pos, the same
 * bytes in out->dst[0 .. out->pos), and the same _finished result and _in_size / _out_size hints.  Bytes past out->pos
 * are unspecified.  The compressed stream is zxc_compress's non-seekable frame.
 * Creation follows zxc_cstream_create / zxc_dstream_create: dictionary options give NULL, so does a bad block_size;
 * level 0 means the default level and other levels are clamped; seekable, n_threads and the progress callback are
 * ignored.  NULL also when there is no device or an allocation fails.  The handle is bound to the CUDA device current
 * at creation; calls switch to it and back.
 * Synchronous and ordered on `stream` (a cudaStream_t, NULL = legacy default stream): a call's work follows what is
 * already enqueued on `stream` (a chunk a kernel just wrote there is seen), and the call returns once all its work is
 * complete: the caller may then overwrite `in` and read `out` without waiting.  Not capturable in a CUDA graph.  The
 * handle owns device buffers, grown to the largest batch a call has used and freed by _free.  Errors are sticky, as in
 * the reference.  One handle must not be used by two threads at once; separate handles may run on separate streams.
 * Reads: nothing outside in->src[in->pos .. in->size) is read.  Writes: nothing outside out->dst[0 .. out->size) and
 * the handle's own memory is written; `in` is not written.
 * Work per call (DESIGN.md section 7l).  Blocks go in batches of at most 64 MiB of decoded bytes, sized from the out
 * room as on the host streams.
 *   cstream, per batch: 3 kernel launches (zxc_b200_launch_count): encode, trailers, and the gather into `out`, plus
 *     one gather before the batch when bytes were drained ahead of it in the call (the file header, a held block);
 *     and 1 host synchronisation (the block sizes and trailers come back in one copy).
 *   dstream, per batch: 4 launches: the header walk, the decode kernels' lean and general instance, and the gather;
 *     3 when checksums are verified (opts->checksum_enabled and a frame with checksums), where the verifying instance
 *     alone replaces the pair; and 2 host synchronisations (the walk's result in one copy, the decode statuses in
 *     one copy).
 *   Either: at most a few small copies per call for bytes cut by a chunk's end (file header, a block header, the
 *   footer) and one synchronisation at the end.  None of this grows with the number of blocks in a batch. */
ZXC_EXPORT zxc_b200_cstream_device* zxc_b200_cstream_device_create(const zxc_compress_opts_t* opts);
ZXC_EXPORT int64_t zxc_b200_cstream_device_compress(zxc_b200_cstream_device* cs, zxc_outbuf_t* out, zxc_inbuf_t* in,
                                                    void* stream);
ZXC_EXPORT int64_t zxc_b200_cstream_device_end(zxc_b200_cstream_device* cs, zxc_outbuf_t* out, void* stream);
ZXC_EXPORT size_t zxc_b200_cstream_device_in_size(const zxc_b200_cstream_device* cs);
ZXC_EXPORT size_t zxc_b200_cstream_device_out_size(const zxc_b200_cstream_device* cs);
ZXC_EXPORT void zxc_b200_cstream_device_free(zxc_b200_cstream_device* cs);

ZXC_EXPORT zxc_b200_dstream_device* zxc_b200_dstream_device_create(const zxc_decompress_opts_t* opts);
ZXC_EXPORT int64_t zxc_b200_dstream_device_decompress(zxc_b200_dstream_device* ds, zxc_outbuf_t* out,
                                                      zxc_inbuf_t* in, void* stream);
ZXC_EXPORT int zxc_b200_dstream_device_finished(const zxc_b200_dstream_device* ds);
ZXC_EXPORT size_t zxc_b200_dstream_device_in_size(const zxc_b200_dstream_device* ds);
ZXC_EXPORT size_t zxc_b200_dstream_device_out_size(const zxc_b200_dstream_device* ds);
ZXC_EXPORT void zxc_b200_dstream_device_free(zxc_b200_dstream_device* ds);

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
