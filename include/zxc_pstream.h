/*
 * zxc_pstream.h -- push-streaming (caller-driven) API.
 *
 * Call for call identical to the reference (include/zxc_pstream.h:70-296,
 * src/lib/zxc_pstream.c): fed the same input chunks and output capacities in
 * the same order, every call returns the same value, leaves the same in->pos
 * and out->pos and writes the same bytes out->dst[0 .. out->pos); bytes past
 * out->pos are unspecified.  zxc_dstream_finished and the *_in_size /
 * *_out_size hints agree as well.
 *
 * Creation follows the reference's options: dictionary options are rejected
 * (NULL), an invalid block_size is rejected, level 0 means the default level
 * and other levels are clamped; seekable, n_threads and the progress callback
 * are ignored.  The compressed stream is zxc_compress's non-seekable frame for
 * the same level, block size and checksum flag.  Errors are sticky; after the
 * end, zxc_cstream_* return ZXC_ERROR_NULL_INPUT and zxc_dstream_decompress 0.
 *
 * GPU: creation never touches the device.  Each stream owns one device
 * context, created by the first call that has to encode or decode a block, on
 * the CUDA device current at that moment; the stream stays on that device
 * (later calls switch to it for their GPU work and back).  Without a device
 * that first call latches ZXC_B200_ERROR_NO_DEVICE as the stream's error;
 * what needs no block (headers, their verdicts, an empty stream's header,
 * EOF block and footer, an empty frame up to its end) works without one.
 * A call batches every whole block it can reach into one launch and still
 * ends in the state the reference's block-by-block loop reaches.  One stream
 * must not be driven from two threads at once; distinct streams are
 * independent.
 */
#ifndef ZXC_PSTREAM_H
#define ZXC_PSTREAM_H

#include <stddef.h>
#include <stdint.h>

#include "zxc_export.h"
#include "zxc_opts.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
    const void* src;
    size_t size;
    size_t pos;
} zxc_inbuf_t;

typedef struct {
    void* dst;
    size_t size;
    size_t pos;
} zxc_outbuf_t;

typedef struct zxc_cstream_s zxc_cstream;
typedef struct zxc_dstream_s zxc_dstream;

ZXC_EXPORT zxc_cstream* zxc_cstream_create(const zxc_compress_opts_t* opts);
ZXC_EXPORT void zxc_cstream_free(zxc_cstream* cs);
ZXC_EXPORT int64_t zxc_cstream_compress(zxc_cstream* cs, zxc_outbuf_t* out, zxc_inbuf_t* in);
ZXC_EXPORT int64_t zxc_cstream_end(zxc_cstream* cs, zxc_outbuf_t* out);
ZXC_EXPORT size_t zxc_cstream_in_size(const zxc_cstream* cs);
ZXC_EXPORT size_t zxc_cstream_out_size(const zxc_cstream* cs);

ZXC_EXPORT zxc_dstream* zxc_dstream_create(const zxc_decompress_opts_t* opts);
ZXC_EXPORT void zxc_dstream_free(zxc_dstream* ds);
ZXC_EXPORT int64_t zxc_dstream_decompress(zxc_dstream* ds, zxc_outbuf_t* out, zxc_inbuf_t* in);
ZXC_EXPORT int zxc_dstream_finished(const zxc_dstream* ds);
ZXC_EXPORT size_t zxc_dstream_in_size(const zxc_dstream* ds);
ZXC_EXPORT size_t zxc_dstream_out_size(const zxc_dstream* ds);

#ifdef __cplusplus
}
#endif
#endif /* ZXC_PSTREAM_H */
