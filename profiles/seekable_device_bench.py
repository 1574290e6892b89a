"""zxc_b200_seekable_device_decompress_ranges on three gather workloads, against the ways there were before it.

Input: --gib GiB (default 4) silesia-shaped at level 3 with 64 KiB blocks, seekable, compressed on the device.
Workloads: minibatch (1 024 x 4 KiB at seeded random offsets), many tiny (65 536 x 256 B), one large (one 1 GiB range
at an odd offset into an odd dst_off).  Per workload, one JSON line with:
  call_ms            the range call (CUDA events, median of --calls after warm-up)
  graph_ms           the same call replayed from a CUDA graph
  useful_gbs         sum of the lengths / call time
  decoded_gbs        blocks decoded (whole blocks, once per range that covers them) x block size / call time
  host_loop_ms       zxc_seekable_decompress_range over the same ranges on a page-locked host copy of the frame
  whole_frame_ms     one zxc_b200_decompress_device of the whole frame (CUDA events)
Every output is checked against the input.  The card, its power limit and max SM clock are read in the same run.
Usage (GPU machine): python profiles/seekable_device_bench.py [--gib 4] [--calls 20]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
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
from test_decompress_device import bind as bind_dd, dopts  # noqa: E402
from test_seekable_device import bind  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def events_ms(fn, calls):
    ts = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--host-calls", type=int, default=2)
    a = ap.parse_args()
    prod = z.ZxcLib(z.PRODUCT_SO)
    L = bind(bind_dd(prod.lib))
    info = card()
    n = int(a.gib * (1 << 30))
    piece = zc.silesia_shaped(256 << 20, seed=3)
    src = torch.from_numpy(np.resize(piece, n)).cuda()
    del piece
    bs = 65536
    f = device.compress(src, level=3, block_size=bs, seekable=True)
    frame = f.frame
    s = torch.cuda.current_stream()
    h = L.zxc_b200_seekable_device_open(frame.data_ptr(), frame.numel(), s.cuda_stream)
    assert h
    pin_frame = torch.empty(frame.numel(), dtype=torch.uint8).pin_memory()
    pin_frame.copy_(frame)
    hs = prod.lib.zxc_seekable_open(pin_frame.data_ptr(), pin_frame.numel())
    assert hs
    # the whole frame, once per call
    out_all = torch.empty(n, dtype=torch.uint8, device="cuda")
    dscr = torch.empty(L.zxc_b200_decompress_device_scratch_size(n, bs), dtype=torch.uint8, device="cuda")
    dres = torch.zeros(1, dtype=torch.int64, device="cuda")
    o = dopts()

    def whole():
        assert L.zxc_b200_decompress_device(frame.data_ptr(), frame.numel(), out_all.data_ptr(), n, C.byref(o),
                                            dscr.data_ptr(), dscr.numel(), dres.data_ptr(), s.cuda_stream) == 0

    whole()
    torch.cuda.synchronize()
    assert int(dres.item()) == n and torch.equal(out_all, src)
    whole_ms = events_ms(whole, 5)
    del out_all, dscr

    rng = np.random.default_rng(2026)
    work = {
        "minibatch": (rng.integers(0, n - 4096, 1024), np.full(1024, 4096)),
        "many_tiny": (rng.integers(0, n - 256, 65536), np.full(65536, 256)),
        "one_large": (np.array([12345677]), np.array([1 << 30])),
    }
    for name, (offs, lens) in work.items():
        offs = offs.astype(np.int64)
        lens = lens.astype(np.int64)
        m = offs.size
        dst_off = np.cumsum(lens) - lens + (13 if name == "one_large" else 0)
        cap = int(dst_off[-1] + lens[-1])
        ranges = torch.from_numpy(np.stack([offs, lens, dst_off], 1)).cuda()
        ss = int(L.zxc_b200_seekable_device_scratch_size(h, m, int(lens.sum())))
        scr = torch.empty(ss, dtype=torch.uint8, device="cuda")
        dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        res = torch.zeros(m, dtype=torch.int64, device="cuda")

        def call():
            assert L.zxc_b200_seekable_device_decompress_ranges(h, ranges.data_ptr(), m, dst.data_ptr(), cap,
                                                                scr.data_ptr(), ss, res.data_ptr(), s.cuda_stream) == 0

        for _ in range(3):
            call()
        torch.cuda.synchronize()
        assert torch.equal(res.cpu(), torch.from_numpy(lens))
        if m == 1:
            assert torch.equal(dst[int(dst_off[0]):], src[int(offs[0]):int(offs[0] + lens[0])]), name
        else:
            rel = np.arange(int(lens.sum())) - np.repeat(np.cumsum(lens) - lens, lens)
            pos = torch.from_numpy(np.repeat(dst_off, lens) + rel).cuda()
            idx = torch.from_numpy(np.repeat(offs, lens) + rel).cuda()
            assert torch.equal(dst[pos], src[idx]), name
            del idx, pos
        call_ms = events_ms(call, a.calls)
        g = torch.cuda.CUDAGraph()
        gs = torch.cuda.Stream()
        gs.wait_stream(s)
        with torch.cuda.graph(g, stream=gs):
            assert L.zxc_b200_seekable_device_decompress_ranges(
                h, ranges.data_ptr(), m, dst.data_ptr(), cap, scr.data_ptr(), ss, res.data_ptr(),
                torch.cuda.current_stream().cuda_stream) == 0
        g.replay()
        torch.cuda.synchronize()
        graph_ms = events_ms(g.replay, a.calls)
        # blocks decoded: whole blocks, once per range that covers them
        b0 = offs // bs
        b1 = (offs + lens - 1) // bs
        decoded = int((b1 - b0 + 1).sum()) * bs
        # the host loop over the same ranges, from the page-locked frame into page-locked memory
        pin_out = torch.zeros(cap, dtype=torch.uint8).pin_memory()
        base = pin_out.data_ptr()
        host = []
        for _ in range(a.host_calls):
            t0 = time.perf_counter()
            for k in range(m):
                r = prod.lib.zxc_seekable_decompress_range(hs, base + int(dst_off[k]), int(lens[k]), int(offs[k]),
                                                           int(lens[k]))
                assert r == lens[k]
            host.append((time.perf_counter() - t0) * 1e3)
        assert torch.equal(pin_out.cuda(), dst), (name, "host loop")
        print(json.dumps({
            "workload": name, "card": info, "input_bytes": n, "frame_bytes": frame.numel(), "level": 3,
            "block_size": bs, "ranges": m, "bytes": int(lens.sum()), "call_ms": round(call_ms, 4),
            "graph_ms": round(graph_ms, 4), "useful_gbs": round(lens.sum() / call_ms / 1e6, 2),
            "decoded_gbs": round(decoded / call_ms / 1e6, 2), "host_loop_ms": round(statistics.median(host), 3),
            "whole_frame_ms": round(whole_ms, 3), "scratch_bytes": ss}), flush=True)
        del g, scr, dst, pin_out
    prod.lib.zxc_seekable_free(hs)
    L.zxc_b200_seekable_device_free(h)


if __name__ == "__main__":
    main()
