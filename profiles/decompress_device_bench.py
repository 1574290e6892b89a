"""zxc_b200_decompress_device against the two host-planned ways of decoding the same frame.

A 4 GiB silesia-shaped input at level 3 with 64 KiB blocks, compressed on the device, once seekable and once not.
Per frame, alternated, median of --rounds:
  device   zxc_b200_decompress_device (CUDA events around the call on one stream)
  plan     zxc_b200_plan_frame on a host copy of the frame + job upload + zxc_b200_decode_blocks + reduce_status
           (host clock: what bench.py's HBM-resident decode does, with the walk it needs first)
  pinned   zxc_decompress from page-locked host memory into page-locked host memory
Every output is checked against the input.  torch.profiler then gives the planner and verdict kernels' share of one
device call.  Usage (GPU machine): python profiles/decompress_device_bench.py [--gib 4] [--rounds 3]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import zxc_corpus as zc  # noqa: E402
import zxc_ctypes as z  # noqa: E402
from zxc_b200 import device  # noqa: E402
from test_decompress_device import bind, dopts  # noqa: E402


class Job(C.Structure):
    _fields_ = [("src_off", C.c_uint64), ("dst_off", C.c_uint64), ("src_len", C.c_uint32), ("dst_cap", C.c_uint32)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    prod = z.ZxcLib(z.PRODUCT_SO)
    L = bind(prod.lib)
    L.zxc_b200_plan_frame.restype = C.c_int64
    L.zxc_b200_plan_frame.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    n = int(a.gib * (1 << 30))
    piece = zc.silesia_shaped(256 << 20, seed=3)
    src = torch.from_numpy(np.resize(piece, n)).cuda()
    del piece
    bs = 65536
    res = {"gpu": torch.cuda.get_device_name(), "input_bytes": n, "level": 3, "block_size": bs}
    out = torch.empty(n, dtype=torch.uint8, device="cuda")
    scr = torch.empty(L.zxc_b200_decompress_device_scratch_size(n, bs), dtype=torch.uint8, device="cuda")
    result = torch.zeros(1, dtype=torch.int64, device="cuda")
    L.zxc_b200_decode_scratch_size.restype = C.c_size_t
    L.zxc_b200_decode_scratch_size.argtypes = [C.c_uint32]
    dscr_size = int(L.zxc_b200_decode_scratch_size(bs))
    dscr = torch.empty(dscr_size, dtype=torch.uint8, device="cuda")
    pin_out = torch.empty(n, dtype=torch.uint8).pin_memory()
    s = torch.cuda.current_stream()
    for seek in (1, 0):
        f = device.compress(src, level=3, block_size=bs, checksum=False, seekable=bool(seek))
        frame = f.frame
        host = frame.cpu().pin_memory()
        hnp = host.numpy()
        nb = f.n_blocks
        jobs = torch.empty(nb * 24, dtype=torch.uint8, device="cuda")
        status = torch.empty(nb, dtype=torch.int32, device="cuda")
        jh = (Job * nb)()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def run_device():
            out.zero_()
            e0.record()
            assert L.zxc_b200_decompress_device(frame.data_ptr(), frame.numel(), out.data_ptr(), n, None,
                                                scr.data_ptr(), scr.numel(), result.data_ptr(), s.cuda_stream) == 0
            e1.record()
            torch.cuda.synchronize()
            assert int(result.item()) == n and torch.equal(out, src)
            return e0.elapsed_time(e1)

        def run_plan():
            out.zero_()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            assert L.zxc_b200_plan_frame(hnp.ctypes.data, hnp.size, jh, nb, None) == nb
            jobs.copy_(torch.frombuffer(jh, dtype=torch.uint8), non_blocking=False)
            assert prod.lib.zxc_b200_decode_blocks(frame.data_ptr(), out.data_ptr(), jobs.data_ptr(), nb,
                                                   status.data_ptr(), None, 0, None, dscr.data_ptr(), dscr_size, bs,
                                                   0, s.cuda_stream) == 0
            r = prod.lib.zxc_b200_reduce_status(C.c_void_p(status.data_ptr()), C.c_void_p(jobs.data_ptr()), nb,
                                                C.c_void_p(s.cuda_stream))
            ms = (time.perf_counter() - t0) * 1e3
            assert r == n and torch.equal(out, src)
            return ms

        def run_pinned():
            t0 = time.perf_counter()
            r = prod.lib.zxc_decompress(C.c_void_p(host.data_ptr()), host.numel(), C.c_void_p(pin_out.data_ptr()), n,
                                        None)
            ms = (time.perf_counter() - t0) * 1e3
            assert r == n and torch.equal(pin_out[: 1 << 20].cuda(), src[: 1 << 20])
            return ms

        prod.lib.zxc_b200_decode_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                                    C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t,
                                                    C.c_uint32, C.c_int, C.c_void_p]
        prod.lib.zxc_b200_reduce_status.restype = C.c_int64
        run_device(), run_plan(), run_pinned()  # warm-up
        t = {"device": [], "plan": [], "pinned": []}
        for _ in range(a.rounds):
            t["device"].append(run_device())
            t["plan"].append(run_plan())
            t["pinned"].append(run_pinned())
        assert torch.equal(pin_out.cuda(), src)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run_device()
        k = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                name = ev.name
                key = "plan" if "dplan" in name else "split" if "dsplit" in name else "decode" if "decode" in name \
                    else "other"
                k[key] = k.get(key, 0.0) + ev.device_time_total / 1e3
        res["seekable" if seek else "non_seekable"] = {
            "frame_bytes": frame.numel(), "blocks": nb,
            **{m + "_ms": round(statistics.median(v), 3) for m, v in t.items()},
            **{m + "_gbps": round(n / statistics.median(v) / 1e6, 1) for m, v in t.items()},
            "kernel_ms": {q: round(v, 3) for q, v in k.items()},
        }
        print(json.dumps(res["seekable" if seek else "non_seekable"]), flush=True)
        del f, frame, host, jobs, status
    print(json.dumps(res))


if __name__ == "__main__":
    main()
