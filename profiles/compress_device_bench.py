"""zxc_b200_compress_device (HBM to HBM, frame assembled on the device) against zxc_compress host to host.

1 GiB silesia-shaped input (tests/zxc_corpus.py), 64 KiB blocks, levels 3 and 6.  Per level, in one run and
alternated rep by rep: the device call (CUDA events around the whole call), zxc_compress from and to pinned host
buffers, and from and to pageable ones (host clock; the call ends in a stream synchronise).  Every frame is checked
against the host path's.  Then, in a separate pass, torch.profiler gives the kernels' own times of one device call
per level, so the assembly kernels' share can be read off.  Prints the card and its power limit, and one JSON line.

    python profiles/compress_device_bench.py [--size-mib 1024] [--reps 3] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
import zxc_corpus as zc  # noqa: E402
import zxc_ctypes as z  # noqa: E402

ASSEMBLY = ("zxc_asm_tile_sums", "zxc_asm_scan_tiles", "zxc_asm_blocks", "zxc_compact_kernel", "zxc_asm_finish")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-mib", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--levels", type=int, nargs="+", default=[3, 6])
    ap.add_argument("--out", default=None, help="directory for the profiler tables")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("compress_device_bench: no CUDA device")
    prod = z.ZxcLib(z.PRODUCT_SO)
    L = prod.lib
    L.zxc_b200_encode_scratch_size.restype = C.c_size_t
    L.zxc_b200_encode_scratch_size.argtypes = [C.c_uint64, C.c_void_p]
    L.zxc_b200_compress_device.restype = C.c_int
    L.zxc_b200_compress_device.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                           C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    n = a.size_mib << 20
    bs = 65536
    data = zc.silesia_shaped(n, seed=1)
    cap = int(L.zxc_compress_bound(n))
    d_src = torch.from_numpy(data).cuda()
    d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    d_res = torch.zeros(1, dtype=torch.int64, device="cuda")
    h_src_pin = torch.from_numpy(data).pin_memory()
    h_dst_pin = torch.empty(cap, dtype=torch.uint8).pin_memory()
    h_dst = np.empty(cap, np.uint8)
    stream = torch.cuda.current_stream()
    card_info = card()
    print("card:", card_info, flush=True)
    rows = {}
    for level in a.levels:
        o = z.CompressOpts(level=level, block_size=bs)
        ss = int(L.zxc_b200_encode_scratch_size(n, C.byref(o)))
        scratch = torch.empty(ss, dtype=torch.uint8, device="cuda")

        def device_call():
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record(stream)
            rc = L.zxc_b200_compress_device(d_src.data_ptr(), n, d_dst.data_ptr(), cap, C.byref(o), scratch.data_ptr(),
                                            ss, d_res.data_ptr(), None, stream.cuda_stream)
            ev1.record(stream)
            assert rc == 0, z.ERR.get(rc, rc)
            ev1.synchronize()
            return ev0.elapsed_time(ev1) / 1e3, int(d_res.item())

        def host_call(src_ptr, dst_ptr):
            t0 = time.perf_counter()
            r = L.zxc_compress(src_ptr, n, dst_ptr, cap, C.byref(o))
            t1 = time.perf_counter()
            assert r > 0, z.ERR.get(r, r)
            return t1 - t0, r

        paths = {
            "device": device_call,
            "host_pinned": lambda: host_call(h_src_pin.data_ptr(), h_dst_pin.data_ptr()),
            "host_pageable": lambda: host_call(data.ctypes.data, h_dst.ctypes.data),
        }
        for f in paths.values():  # warm-up: module load, context buffers, pinned bounce buffers
            f()
        times = {k: [] for k in paths}
        size = None
        for _ in range(a.reps):
            for k, f in paths.items():
                t, r = f()
                times[k].append(t)
                size = r if size is None else size
                assert r == size, (k, r, size)
        ok = (np.array_equal(d_dst[:size].cpu().numpy(), h_dst[:size])
              and np.array_equal(h_dst_pin[:size].numpy(), h_dst[:size]))
        assert ok, "device frame differs from the host path's"
        rows[level] = {"frame_bytes": size, "identical": ok,
                       **{f"{k}_s_median": float(np.median(v)) for k, v in times.items()},
                       **{f"{k}_s_all": [round(x, 5) for x in v] for k, v in times.items()},
                       **{f"{k}_GBps": n / float(np.median(v)) / 1e9 for k, v in times.items()}}
        print(f"L{level}: " + ", ".join(f"{k} {n / np.median(v) / 1e9:.2f} GB/s (median of {len(v)})"
                                        for k, v in times.items()), flush=True)
        del scratch
        torch.cuda.empty_cache()
    # kernel times from the profiler, in a pass of their own
    from torch.profiler import ProfilerActivity, profile
    for level in a.levels:
        o = z.CompressOpts(level=level, block_size=bs)
        ss = int(L.zxc_b200_encode_scratch_size(n, C.byref(o)))
        scratch = torch.empty(ss, dtype=torch.uint8, device="cuda")
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            assert L.zxc_b200_compress_device(d_src.data_ptr(), n, d_dst.data_ptr(), cap, C.byref(o), scratch.data_ptr(),
                                              ss, d_res.data_ptr(), None, stream.cuda_stream) == 0
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():  # kernels, memcpy and memset: the device activities of the call
            t = getattr(e, "self_device_time_total", 0.0)
            if t > 0:
                kern[e.key] = t / 1e3  # us -> ms
        total = sum(kern.values())
        asm = sum(v for k, v in kern.items() if any(s in k for s in ASSEMBLY))
        rows[level]["kernel_ms"] = {k: round(v, 4) for k, v in kern.items() if v > 0}
        rows[level]["assembly_ms"] = round(asm, 4)
        rows[level]["assembly_share_of_device_time"] = asm / total if total else None
        print(f"L{level}: device time {total:.2f} ms, of which assembly (scan, blocks, compaction, finish) {asm:.3f} ms",
              flush=True)
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, f"compress_device_L{level}_kernels.txt"), "w") as fh:
                fh.write(prof.key_averages().table(sort_by="self_device_time_total", row_limit=30))
        del scratch
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "compress_device", "card": card_info, "input_bytes": n, "block_size": bs,
                      "levels": rows}), flush=True)


if __name__ == "__main__":
    main()
