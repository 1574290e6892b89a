/*
 * zxc_error.h -- negative return codes shared by every entry point.
 *
 * Replaces: reference include/zxc_error.h:39-76 (enum) and :88 (zxc_error_name).
 * Codes -1..-18 are the reference's; ZXC_B200_ERROR_* are additive (the
 * reference's ABI policy allows added symbols/values, .github/workflows/abi-check.yml:128).
 */
#ifndef ZXC_ERROR_H
#define ZXC_ERROR_H

#include "zxc_export.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    ZXC_OK = 0,
    ZXC_ERROR_MEMORY = -1,
    ZXC_ERROR_DST_TOO_SMALL = -2,
    ZXC_ERROR_SRC_TOO_SMALL = -3,
    ZXC_ERROR_BAD_MAGIC = -4,
    ZXC_ERROR_BAD_VERSION = -5,
    ZXC_ERROR_BAD_HEADER = -6,
    ZXC_ERROR_BAD_CHECKSUM = -7,
    ZXC_ERROR_CORRUPT_DATA = -8,
    ZXC_ERROR_BAD_OFFSET = -9,
    ZXC_ERROR_OVERFLOW = -10,
    ZXC_ERROR_IO = -11,
    ZXC_ERROR_NULL_INPUT = -12,
    ZXC_ERROR_BAD_BLOCK_TYPE = -13,
    ZXC_ERROR_BAD_BLOCK_SIZE = -14,
    ZXC_ERROR_DICT_REQUIRED = -15,
    ZXC_ERROR_DICT_MISMATCH = -16,
    ZXC_ERROR_DICT_TOO_LARGE = -17,
    ZXC_ERROR_BAD_LEVEL = -18,
    /* additive: the CUDA device / runtime is missing or failed.  There is no
     * CPU fallback behind this library, so codec entry points report this. */
    ZXC_B200_ERROR_NO_DEVICE = -100,
    ZXC_B200_ERROR_CUDA = -101,
    /* additive: memory the call cannot work on, e.g. a host room that is not
     * page-locked memory mapped for the device
     * (zxc_b200_compress_device_to_host). */
    ZXC_B200_ERROR_UNSUPPORTED = -102
} zxc_error_t;

ZXC_EXPORT const char* zxc_error_name(const int code);

#ifdef __cplusplus
}
#endif
#endif /* ZXC_ERROR_H */
