"""compute-sanitizer driver for seekable frames in page-locked host memory (zxc_b200_seekable_device_open_host and
its range calls): frames at every offset 0-15 inside exact-size cudaHostAlloc allocations, and flush against their
end, with the standard range mix, payload damage and a scratch sized for fewer bytes than the ranges ask -- memcheck
must stay silent and every result and byte must equal zxc_seekable_decompress_range's.  Usage on a GPU machine:
    compute-sanitizer --tool memcheck python tests/sanitize_seekable_host.py"""
import ctypes as C
import os
import sys

os.environ.setdefault("PYTORCH_NO_CUDA_MEMORY_CACHING", "1")  # every tensor its own cudaMalloc: exact bounds

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import zxc_corpus as zc  # noqa: E402
import zxc_ctypes as z  # noqa: E402
from test_seekable_device import host_ranges, standard_ranges  # noqa: E402
from test_seekable_host import bind_host  # noqa: E402

torch.cuda.init()
rt = C.CDLL("libcudart.so.12")
rt.cudaHostAlloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t, C.c_uint]
rt.cudaFreeHost.argtypes = [C.c_void_p]
prod = z.ZxcLib(z.PRODUCT_SO)
L = bind_host(prod.lib)
n = bad = 0


def check(frame, place, rs, cap, max_bytes=None):
    """the frame in an exact-size pinned allocation, at offset `place` (or flush against its end for None)"""
    global n, bad
    off = 0 if place is None else place
    size = frame.size + off
    p = C.c_void_p()
    assert rt.cudaHostAlloc(C.byref(p), size, 0) == 0
    try:
        C.memmove(p.value + off, frame.ctypes.data, frame.size)
        h = L.zxc_b200_seekable_device_open_host(p.value + off, frame.size, None)
        assert h
        max_bytes = sum(k for _, k, _ in rs) if max_bytes is None else max_bytes
        ss = int(L.zxc_b200_seekable_device_scratch_size(h, len(rs), max_bytes))
        scr = torch.empty(ss, dtype=torch.uint8, device="cuda")
        dst = torch.zeros(max(cap, 1), dtype=torch.uint8, device="cuda")
        res = torch.zeros(len(rs), dtype=torch.int64, device="cuda")
        rr = torch.from_numpy(np.array(rs, np.uint64).reshape(-1, 3).view(np.int64)).cuda()
        assert L.zxc_b200_seekable_device_decompress_ranges(h, rr.data_ptr(), len(rs), dst.data_ptr(), cap,
                                                            scr.data_ptr(), ss, res.data_ptr(), None) == 0
        torch.cuda.synchronize()
        L.zxc_b200_seekable_device_free(h)
        got, out = res.tolist(), dst.cpu().numpy()
        want = host_ranges(prod.lib, frame, rs, cap)
        for i, ((o, k, dd), r, (r0, o0)) in enumerate(zip(rs, got, want)):
            n += 1
            ok = r == r0 or (r == -1 and max_bytes < sum(x for _, x, _ in rs))
            if ok and r0 > 0 and r > 0:
                ok = np.array_equal(out[dd:dd + k], o0)
            if not ok:
                bad += 1
                print("MISMATCH", place, i, o, k, r, r0)
    finally:
        rt.cudaFreeHost(p)


for bs, level in ((4096, 1), (65536, 3)):
    data = zc.silesia_shaped(6 * bs + 999, seed=bs)
    frame = prod.compress(data, level=level, block_size=bs, checksum=1, seekable=1)
    rs, cap = standard_ranges(data.size, bs, 17)
    damaged = frame.copy()
    damaged[16 + bs // 3] ^= 0x33
    for place in list(range(16)) + [None]:
        check(frame, place, rs, cap)
    for place in (0, 5, None):
        check(damaged, place, rs, cap)
        check(frame, place, rs, cap, max_bytes=bs)
print("sanitize_seekable_host: ran", n, "checks, mismatches:", bad)
sys.exit(1 if bad else 0)
