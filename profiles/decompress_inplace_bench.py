"""zxc_b200_decompress_inplace_device against zxc_b200_decompress_device on one 4 GiB frame.

Silesia-shaped input (a 64 MiB piece repeated to 4 GiB), compressed on the device at level 3 with 64 KiB blocks, once
seekable and once not.  The in-place call runs with windows of 64 MiB, 256 MiB, 1 GiB and the whole frame, in a buffer
of zxc_decompress_inplace_bound bytes with a scratch from zxc_b200_decompress_inplace_device_scratch_size.  Each round
restores the frame at the buffer's end (not timed), times one in-place call, then one out-of-place call of the same
frame into a separate output (CUDA events around each call on one stream); medians of --rounds after a warm-up.
Reported per window: both medians, the device bytes each needs (buffer + scratch against frame + output + scratch),
the launches of one in-place call (16 + R (1 + k (2 + c)), so the rounds it ran) and a check of every output against
the input.  The card's name, power limit and SM clock are read in the same run.
Usage (GPU machine): python profiles/decompress_inplace_bench.py [--rounds 5] [--gib 4]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "profiles"))
sys.path.insert(0, ROOT)
import zxc_corpus as zc  # noqa: E402
import zxc_ctypes as z  # noqa: E402
from decompress_batch_bench import card  # noqa: E402
from zxc_b200 import device  # noqa: E402
from test_decompress_inplace_device import bind  # noqa: E402

BS = 65536
MIB = 1 << 20


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def workload(L, src, seek, rounds):
    total = src.numel()
    s = torch.cuda.current_stream()
    frame = device.compress(src, level=3, block_size=BS, seekable=bool(seek)).frame
    n = frame.numel()
    cap = int(L.zxc_b200_decompress_inplace_device_bound(frame.data_ptr(), n, s.cuda_stream))
    buf = torch.empty(cap, dtype=torch.uint8, device="cuda")
    out = torch.empty(total, dtype=torch.uint8, device="cuda")
    res = torch.zeros(2, dtype=torch.int64, device="cuda")
    oop = torch.empty(int(L.zxc_b200_decompress_device_scratch_size(total, BS)), dtype=torch.uint8, device="cuda")
    rows = []
    for window in (64 * MIB, 256 * MIB, 1024 * MIB, n):
        scr = torch.empty(int(L.zxc_b200_decompress_inplace_device_scratch_size(cap, BS, window)), dtype=torch.uint8,
                          device="cuda")

        def inplace():
            assert L.zxc_b200_decompress_inplace_device(buf.data_ptr(), cap, n, None, scr.data_ptr(), scr.numel(),
                                                        res.data_ptr(), s.cuda_stream) == 0

        def out_of_place():
            assert L.zxc_b200_decompress_device(frame.data_ptr(), n, out.data_ptr(), total, None, oop.data_ptr(),
                                                oop.numel(), res.data_ptr() + 8, s.cuda_stream) == 0

        t_in, t_out, launches = [], [], 0
        for r in range(rounds + 1):
            buf[cap - n:].copy_(frame)
            torch.cuda.synchronize()
            before = int(L.zxc_b200_launch_count())
            ti = timed(inplace)
            launches = int(L.zxc_b200_launch_count()) - before
            assert int(res[0].item()) == total and torch.equal(buf[:total], src), ("in place", window)
            to = timed(out_of_place)
            assert int(res[1].item()) == total and torch.equal(out, src), "out of place"
            out.zero_()
            if r > 0:  # the first is the warm-up
                t_in.append(ti)
                t_out.append(to)
        row = {"seekable": bool(seek), "compressed_bytes": n, "decoded_bytes": total, "window": window,
               "inplace_launches": launches,
               "inplace_ms": round(statistics.median(t_in), 2), "out_of_place_ms": round(statistics.median(t_out), 2),
               "inplace_device_bytes": cap + scr.numel(), "out_of_place_device_bytes": n + total + oop.numel(),
               "outputs_checked": True}
        row["inplace_gbps"] = round(total / row["inplace_ms"] / 1e6, 1)
        row["out_of_place_gbps"] = round(total / row["out_of_place_ms"] / 1e6, 1)
        print(json.dumps(row), flush=True)
        rows.append(row)
        del scr
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--gib", type=float, default=4.0)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    L = bind(z.ZxcLib(z.PRODUCT_SO).lib)
    L.zxc_b200_decompress_device_scratch_size.restype = C.c_size_t
    L.zxc_b200_decompress_device_scratch_size.argtypes = [C.c_uint64, C.c_uint32]
    L.zxc_b200_decompress_device.restype = C.c_int
    L.zxc_b200_decompress_device.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                             C.c_size_t, C.c_void_p, C.c_void_p]
    piece = zc.silesia_shaped(64 << 20, seed=3)
    src = torch.from_numpy(np.resize(piece, int(a.gib * (1 << 30)))).cuda()
    for seek in (0, 1):
        workload(L, src, seek, a.rounds)


if __name__ == "__main__":
    main()
