"""compute-sanitizer driver for the dictionary trainers on samples in HBM (zxc_b200_train_dict_device,
zxc_b200_train_dict_huf_device, zxc_b200_dict_train_device): every sample in its own exactly sized allocation, flush
against its end, starting at offsets 0 (aligned) and 1-15 (misaligned), with sizes around the gather's 16-byte vectors
and its 64 KiB pieces, and NULL samples.  memcheck must stay silent and every result must equal the host trainers'.
Usage on a GPU machine:
    compute-sanitizer --tool memcheck python tests/sanitize_train_device.py"""
import ctypes as C
import os
import sys

os.environ.setdefault("PYTORCH_NO_CUDA_MEMORY_CACHING", "1")  # every tensor its own cudaMalloc: exact bounds

import numpy as np  # noqa: E402
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_train_gpu as T  # noqa: E402
import zxc_ctypes as z  # noqa: E402
from test_train_device_host import Twins  # noqa: E402

prod = z.ZxcLib(z.PRODUCT_SO)
H, D = T.bind(prod), Twins(prod)
n = bad = 0


class Flush:
    """sample i copied into an allocation of exactly offsets[i] + sizes[i] bytes, ending flush with it"""

    def __init__(self, data, sizes, offsets, nulls=()):
        self.keep, ptrs, hp, o = [], [], [], 0
        for i, (s, off) in enumerate(zip(sizes, offsets)):
            if i in nulls:
                ptrs.append(None)
                hp.append(None)
                continue
            t = torch.empty(off + s, dtype=torch.uint8, device="cuda")
            if s:
                t[off:] = torch.from_numpy(data[o:o + s]).cuda()
            self.keep.append(t)
            ptrs.append(t.data_ptr() + off)
            hp.append(data.ctypes.data + o)
            o += s
        self.n = len(sizes)
        self.ptrs = (C.c_void_p * self.n)(*ptrs)
        self.hptrs = (C.c_void_p * self.n)(*hp)
        self.sizes = (C.c_size_t * self.n)(*sizes)


class View:
    def __init__(self, ptrs, sizes, n):
        self.ptrs, self.sizes, self.n = ptrs, sizes, n


def check(data, sizes, offsets, cap, nulls=()):
    global n, bad
    F = Flush(data, sizes, offsets, nulls)
    hv = View(F.hptrs, F.sizes, F.n)
    want = [T.train_content(H, hv, cap), T.train_zxd(H, hv)]
    got = [T.train_content(D, F, cap), T.train_zxd(D, F)]
    if want[0][0] > 0:
        want.append(T.train_table(H, hv, want[0][1]))
        got.append(T.train_table(D, F, want[0][1]))
    n += 1
    if got != want:
        bad += 1
        print("MISMATCH", len(sizes), offsets[:4], cap, [g[0] for g in got], [w[0] for w in want])


rng = np.random.default_rng(3)
data = T.corpus("records", 1 << 21)
edge = [1, 2, 15, 16, 17, 31, 32, 33, 47, 48, 63, 64, 65, 4095, 4096, 4097, 65535, 65536, 65537, 131073]
for base in range(16):
    offs = [(base + i) % 16 for i in range(len(edge))]
    check(data, edge, offs, 4096)
sizes = [int(x) for x in rng.integers(1, 300, 2000)]
for base in (0, 1, 7, 15):
    check(data, sizes, [base] * len(sizes), 16384)
    check(data, sizes, [(base + i) % 16 for i in range(len(sizes))], 16384)
check(data, [100, 5000, 100, 70000, 100], [3, 0, 9, 1, 15], 1024, nulls=(1, 3))
print("sanitize_train_device: ran", n, "cases, mismatches:", bad)
sys.exit(1 if bad else 0)
