"""compute-sanitizer driver for zxc_b200_compress_device: unaligned inputs and outputs, inputs that end at the end of
their allocation, capacities from exact down to one byte short, one-warp scratch, a dictionary -- memcheck must stay
silent and every frame must equal zxc_compress's.  Usage on the GPU machine:
    compute-sanitizer --tool memcheck python tests/sanitize_compress_device.py"""
import ctypes as C
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import zxc_ctypes as z  # noqa: E402
from test_compress_device import Dev, opts  # noqa: E402
from test_oracle import golden_dicts, make_case  # noqa: E402

prod = z.ZxcLib(z.PRODUCT_SO)
dev = Dev(prod)
n = bad = 0
d, h = next(iter(golden_dicts().values()))
for kind, size in (("tiny", 1), ("small", 37), ("text", 4095), ("text", 4097), ("runs", 30000), ("silesia", 140001)):
    data = make_case(kind, size)
    for level, bs, dd, hh in ((1, 4096, None, None), (3, 65536, None, None), (6, 4096, None, None), (7, 65536, d, h)):
        want = prod.compress(data, level=level, block_size=bs, checksum=1, seekable=1, dict=dd, dict_huf=hh)
        for src_off, dst_off in ((0, 0), (1, 3), (15, 1)):
            o = opts(level, bs, 1, 1, dd, hh)
            r, fr, _ = dev.compress(data, o, src_off=src_off, dst_off=dst_off, jobs=True)
            n += 1
            if r != want.size or not np.array_equal(fr, want):
                bad += 1
                print("MISMATCH", kind, size, level, bs, src_off, dst_off, r)
        # capacities around the frame size, the dst tensor ending exactly at dst_capacity
        src = torch.from_numpy(data).cuda()
        o = opts(level, bs, 1, 1, dd, hh)
        scratch = torch.empty(dev.scratch_size(data.size, o), dtype=torch.uint8, device="cuda")
        res = torch.zeros(1, dtype=torch.int64, device="cuda")
        for cap in (want.size, want.size - 1, want.size - 50, 60):
            if cap <= 0:
                continue
            dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
            rc = dev.enqueue(src.data_ptr(), data.size, dst.data_ptr(), cap, o, scratch, res)
            torch.cuda.synchronize()
            got = int(res.item()) if rc == 0 else rc
            n += 1
            if (cap >= want.size) != (got == want.size) or (cap < want.size and got != -2):
                bad += 1
                print("CAPACITY", kind, size, level, bs, cap, got)
print("sanitize_compress_device: ran", n, "calls, mismatches:", bad)
