/*
 * zxc_dict.h -- dictionary identity, .zxd container, trainers.
 *
 * On the hot path: zxc_dict_id (binds a frame to its dictionary), load/save/
 * get_id/huf (the .zxd container).  The trainers run their data-parallel work
 * on the GPU (k-gram count, candidate segments, greedy pick; the level-6 parses
 * whose literals make the shared table) and return the reference's bytes and
 * codes; without a device a valid call returns ZXC_B200_ERROR_NO_DEVICE
 * (DESIGN.md section 7d).
 *
 * Reference interface replaced (file:line in /root/reference):
 *   zxc_dict_id          include/zxc_dict.h:52    src/lib/zxc_dict.c:35
 *   zxc_dict_load        include/zxc_dict.h:92    src/lib/zxc_dict.c:133
 *   zxc_dict_save[_bound] include/zxc_dict.h:110-121 src/lib/zxc_dict.c:80-121
 *   zxc_dict_get_id      include/zxc_dict.h:131   src/lib/zxc_dict.c:70
 *   zxc_dict_huf         include/zxc_dict.h:205   src/lib/zxc_dict.c:185
 *   trainers             include/zxc_dict.h:150-195 src/lib/zxc_dict.c:231-638
 */
#ifndef ZXC_DICT_H
#define ZXC_DICT_H

#include <stddef.h>
#include <stdint.h>

#include "zxc_export.h"

#ifdef __cplusplus
extern "C" {
#endif

/* fold32(rapidhash(content)); when huf_lengths != NULL the 128-byte table is
 * hashed with that value as seed.  0 for an empty / NULL dictionary. */
ZXC_EXPORT uint32_t zxc_dict_id(const void* dict, size_t dict_size, const void* huf_lengths);

/* Parse a .zxd image; outputs are views into `buf`. */
ZXC_EXPORT int zxc_dict_load(const void* buf, size_t buf_size, const void** content_out,
                             size_t* content_size_out, const void** huf_out, uint32_t* dict_id_out);

ZXC_EXPORT int64_t zxc_dict_save(const void* content, size_t content_size, const void* huf_lengths,
                                 void* buf, size_t buf_capacity);
ZXC_EXPORT size_t zxc_dict_save_bound(size_t content_size);
ZXC_EXPORT uint32_t zxc_dict_get_id(const void* buf, size_t buf_size);

ZXC_EXPORT int64_t zxc_train_dict(const void* const* samples, const size_t* sample_sizes,
                                  size_t n_samples, void* dict_buf, size_t dict_capacity);
ZXC_EXPORT int zxc_train_dict_huf(const void* const* samples, const size_t* sample_sizes,
                                  size_t n_samples, const void* dict, size_t dict_size,
                                  uint8_t* huf_lengths_out);
ZXC_EXPORT int64_t zxc_dict_train(const void* const* samples, const size_t* sample_sizes,
                                  size_t n_samples, void* zxd_buf, size_t zxd_capacity);

ZXC_EXPORT const void* zxc_dict_huf(const void* buf, size_t buf_size);

#ifdef __cplusplus
}
#endif
#endif /* ZXC_DICT_H */
