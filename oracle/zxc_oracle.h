/*
 * zxc_oracle.h -- TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C, scalar restatement of the ZXC v8 decode path (frame walk, block
 * decode, hashes).  It exists to CHECK the CUDA path in tests/, in
 * __graft_entry__.smoke() and as bench.py's cpu_baseline "port" leg.  Nothing
 * under zxc_b200/ includes, links or calls it, and libzxc.so has no CPU codec.
 *
 * Parity status: PINNED.  tests/test_oracle.py checks this restatement against
 * every conformance/valid vector and every conformance/invalid error code the
 * reference's tests hold for the path (copied as fixtures into tests/golden/),
 * and differentially against oracle/_ref/libzxc_ref.so (the unmodified
 * reference compiled by oracle/Makefile) on seeded synthetic inputs.
 */
#ifndef ZXC_ORACLE_H
#define ZXC_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* error codes: the reference's zxc_error_t values (include/zxc_error.h:39-76) */
#define ZXO_OK 0
#define ZXO_E_MEMORY (-1)
#define ZXO_E_DST_TOO_SMALL (-2)
#define ZXO_E_SRC_TOO_SMALL (-3)
#define ZXO_E_BAD_MAGIC (-4)
#define ZXO_E_BAD_VERSION (-5)
#define ZXO_E_BAD_HEADER (-6)
#define ZXO_E_BAD_CHECKSUM (-7)
#define ZXO_E_CORRUPT_DATA (-8)
#define ZXO_E_BAD_OFFSET (-9)
#define ZXO_E_OVERFLOW (-10)
#define ZXO_E_NULL_INPUT (-12)
#define ZXO_E_BAD_BLOCK_TYPE (-13)
#define ZXO_E_BAD_BLOCK_SIZE (-14)
#define ZXO_E_DICT_REQUIRED (-15)
#define ZXO_E_DICT_MISMATCH (-16)

/* hashes (src/lib/zxc_internal.h:1188-1214, :1353-1393; vendors/rapidhash.h V3) */
uint8_t zxo_hash8(const uint8_t* p8);
uint16_t zxo_hash16(const uint8_t* p16);
uint64_t zxo_rapidhash(const void* key, size_t len, uint64_t seed);
uint32_t zxo_checksum(const void* p, size_t len);
uint32_t zxo_checksum_seed(const void* p, size_t len, uint32_t seed);
uint32_t zxo_dict_id(const void* dict, size_t dict_size, const void* huf128);

/* One on-disk block (8-byte header + payload [+4 checksum if has_checksum]).
 * Returns decoded bytes or a negative code.  `dict` (may be NULL) is the
 * window prefix matches may reach into.  src/lib/zxc_decompress.c:1646-1695.
 * `block_size` is the frame's block size, which bounds the Huffman-coded token count; zxo_decode_block takes it from
 * dst_cap rounded up to a block size, as the block API zxc_decompress_block does. */
int zxo_decode_block_bs(const uint8_t* blk, size_t blk_size, uint8_t* dst, size_t dst_cap,
                        const uint8_t* dict, size_t dict_size, const uint8_t* dict_huf,
                        int verify_checksum, size_t block_size);
int zxo_decode_block(const uint8_t* blk, size_t blk_size, uint8_t* dst, size_t dst_cap,
                     const uint8_t* dict, size_t dict_size, const uint8_t* dict_huf,
                     int verify_checksum);

/* Whole frame, the behaviour of zxc_decompress (src/lib/zxc_dispatch.c:842-1005). */
int64_t zxo_decompress(const uint8_t* src, size_t src_size, uint8_t* dst, size_t dst_cap,
                       int checksum_enabled, const uint8_t* dict, size_t dict_size,
                       const uint8_t* dict_huf);

/* Per-block sequence statistics of a frame (kernel-sizing aid for tests/bench). */
typedef struct {
    uint64_t blocks, raw_blocks, glo_blocks, ghi_blocks;
    uint64_t sequences, literals, extras_bytes, comp_bytes, decoded_bytes;
    uint64_t ll_escapes, ml_escapes, off_lt32, off_lt_ml, rle_blocks, huf_blocks, off8_blocks;
    uint64_t ml_sum, max_seq_per_block;
} zxo_stats_t;
int zxo_frame_stats(const uint8_t* src, size_t src_size, zxo_stats_t* out);

/* SEK table: returns number of blocks (>0) and fills block_size/total, or a negative code.
 * comp_sizes (may be NULL) receives up to cap entries.  src/lib/zxc_seekable.c:270-396. */
int64_t zxo_seek_parse(const uint8_t* src, size_t src_size, uint32_t* block_size,
                       uint64_t* total, uint32_t* comp_sizes, size_t cap);

#ifdef __cplusplus
}
#endif
#endif
