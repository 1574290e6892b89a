"""compute-sanitizer driver for the push streams in HBM (zxc_b200_cstream_device / _dstream_device): chunks in exactly
sized allocations at offsets 1 and 15, RAW blocks that end at a chunk's end, small and large out capacities, and
mutated frames -- memcheck must stay silent and every transcript must equal the host streams' (zxc_cstream_* /
zxc_dstream_*).  Usage on a GPU machine:
    compute-sanitizer --tool memcheck python tests/sanitize_pstream_device.py"""
import os
import sys

os.environ.setdefault("PYTORCH_NO_CUDA_MEMORY_CACHING", "1")  # every tensor its own cudaMalloc: exact bounds

import numpy as np  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import zxc_corpus as zc  # noqa: E402
import zxc_ctypes as z  # noqa: E402
import zxc_pstream_driver as pd  # noqa: E402
from test_decompress_device import _mutants  # noqa: E402
from test_pstream_device import bind_device, drive_dev  # noqa: E402

prod = z.ZxcLib(z.PRODUCT_SO)
P = bind_device(pd.bind(prod.lib))
n = bad = 0


def check(make, sched, end_cap=None, offset=1):
    global n, bad
    tp = drive_dev(P, make, sched, end_cap=end_cap, offset=offset)
    th = pd.drive(P, make, sched, end_cap=end_cap)
    n += 1
    if tp != th:
        bad += 1
        print("MISMATCH", make[0], len(sched), offset, tp[-1][:3] if tp else None, th[-1][:3] if th else None)


data = zc.silesia_shaped(1 << 20, seed=5)[:300001]
raw = np.random.default_rng(7).integers(0, 256, 40000, dtype=np.uint8)
for level, bs, cks in ((1, 4096, 1), (3, 65536, 0), (6, 4096, 1)):
    for offset in (1, 15):
        for cap in (pd.UNLIMITED, 13, bs + 2112):
            check(("c", z.CompressOpts(level=level, block_size=bs, checksum_enabled=cks)),
                  [(data[i:i + 70001].tobytes(), cap) for i in range(0, data.size, 70001)], cap, offset)
    for src in (data, raw):
        frame = prod.compress(src, level=level, block_size=bs, checksum=cks)
        fb = frame.tobytes()
        for offset in (1, 15):
            for step, cap in ((len(fb), pd.UNLIMITED), (5001, 13), (bs + 20, bs + 2112)):
                check(("d", z.DecompressOpts(checksum_enabled=cks)),
                      [(fb[i:i + step], cap) for i in range(0, len(fb), step)], cap, offset)
        for _, m in _mutants(frame, 20, seed=level):
            check(("d", z.DecompressOpts(checksum_enabled=1)), [(m.tobytes(), pd.UNLIMITED)], offset=15)
# RAW blocks that end exactly at a chunk's end, chunks cut at every block boundary
bs = 4096
for cks in (0, 1):
    fb = prod.compress(raw, level=1, block_size=bs, checksum=cks).tobytes()
    cuts, p = [0], 16
    while p + 8 <= len(fb) and fb[p] != 255:
        cuts.append(p)
        p += 8 + int.from_bytes(fb[p + 3:p + 7], "little") + 4 * cks
    cuts += [p, len(fb)]
    for offset in (1, 15):
        check(("d", z.DecompressOpts(checksum_enabled=cks)),
              [(fb[a:b], pd.UNLIMITED) for a, b in zip(cuts, cuts[1:]) if b > a], offset=offset)
print("sanitize_pstream_device: ran", n, "streams, mismatches:", bad)
sys.exit(1 if bad else 0)
