"""Random access into a seekable frame in page-locked host memory (zxc_b200_seekable_device_open_host), against the
frame in HBM and against the host seekable handle.

Input: --gib GiB (default 4) silesia-shaped at level 3 with 64 KiB blocks, seekable, compressed on the device and copied
into a pinned host buffer.  Workloads: minibatch (1 024 x 4 KiB at seeded random offsets), many tiny (65 536 x 256 B),
one large (one 1 GiB range at an odd offset into an odd dst_off), whole frame (one range over everything).  Per
workload, one JSON line with:
  call_ms          the host-backed range call (CUDA events, median of --calls after warm-up)
  graph_ms         the same call replayed from a CUDA graph
  staged_bytes     the compressed bytes the call moves over PCIe: each range's span of blocks, from the SEK offsets
  fetch_ms         zxc_dseek_fetch's mean kernel time, from torch.profiler in a separate run; fetch_gbs = staged / it
  copy_engine_ms   a pinned host-to-device cudaMemcpy of staged_bytes (CUDA events); copy_engine_gbs
  device_call_ms   the same ranges on the device handle with the frame in HBM (the lower bound)
  host_loop_ms     the way before: zxc_seekable_decompress_range per range into pinned memory, then one host-to-device
                   copy of the decoded bytes (wall clock, median of --host-calls)
Every output is checked against the input.  The card, its power limit and max SM clock are read in the same run.
Usage (GPU machine): python profiles/seekable_host_bench.py [--gib 4] [--calls 20]
"""
import argparse
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
from test_seekable_host import bind_host  # noqa: E402


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


def sek_offsets(frame, bs):
    """the blocks' frame offsets from the SEK table: 16 + the prefix sums of its entries"""
    total = int.from_bytes(frame[-12:-4].tobytes(), "little")
    nb = -(-total // bs)
    ent = frame.size - 12 - 4 * nb
    sizes = np.frombuffer(frame[ent:ent + 4 * nb].tobytes(), "<u4").astype(np.int64)
    return np.concatenate([[16], 16 + np.cumsum(sizes)])


def fetch_kernel_ms(call, reps):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    ts = [e.device_time for e in p.events() if "zxc_dseek_fetch" in e.name]
    return (sum(ts) / len(ts) / 1e3) if ts else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--host-calls", type=int, default=2)
    a = ap.parse_args()
    prod = z.ZxcLib(z.PRODUCT_SO)
    L = bind_host(prod.lib)
    info = card()
    n = int(a.gib * (1 << 30))
    piece = zc.silesia_shaped(256 << 20, seed=3)
    src = torch.from_numpy(np.resize(piece, n)).cuda()
    del piece
    bs = 65536
    frame = device.compress(src, level=3, block_size=bs, seekable=True).frame
    pin_frame = torch.empty(frame.numel(), dtype=torch.uint8).pin_memory()
    pin_frame.copy_(frame)
    offs_tab = sek_offsets(pin_frame.numpy(), bs)
    s = torch.cuda.current_stream()
    hh = L.zxc_b200_seekable_device_open_host(pin_frame.data_ptr(), pin_frame.numel(), s.cuda_stream)
    hd = L.zxc_b200_seekable_device_open(frame.data_ptr(), frame.numel(), s.cuda_stream)
    hs = prod.lib.zxc_seekable_open(pin_frame.data_ptr(), pin_frame.numel())
    assert hh and hd and hs

    rng = np.random.default_rng(2026)
    work = {
        "minibatch": (rng.integers(0, n - 4096, 1024), np.full(1024, 4096)),
        "many_tiny": (rng.integers(0, n - 256, 65536), np.full(65536, 256)),
        "one_large": (np.array([12345677]), np.array([1 << 30])),
        "whole_frame": (np.array([0]), np.array([n])),
    }
    for name, (offs, lens) in work.items():
        offs = offs.astype(np.int64)
        lens = lens.astype(np.int64)
        m = offs.size
        dst_off = np.cumsum(lens) - lens + (13 if name == "one_large" else 0)
        cap = int(dst_off[-1] + lens[-1])
        ranges = torch.from_numpy(np.stack([offs, lens, dst_off], 1)).cuda()
        dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        res = torch.zeros(m, dtype=torch.int64, device="cuda")
        b0, b1 = offs // bs, (offs + lens - 1) // bs
        staged = int((offs_tab[b1 + 1] - offs_tab[b0]).sum())

        def maker(h):
            ss = int(L.zxc_b200_seekable_device_scratch_size(h, m, int(lens.sum())))
            scr = torch.empty(ss, dtype=torch.uint8, device="cuda")

            def call(stream=s):
                assert L.zxc_b200_seekable_device_decompress_ranges(h, ranges.data_ptr(), m, dst.data_ptr(), cap,
                                                                    scr.data_ptr(), ss, res.data_ptr(),
                                                                    stream.cuda_stream) == 0
            return call, scr

        def verify(what):
            torch.cuda.synchronize()
            assert torch.equal(res.cpu(), torch.from_numpy(lens)), (name, what)
            if m == 1:
                assert torch.equal(dst[int(dst_off[0]):], src[int(offs[0]):int(offs[0] + lens[0])]), (name, what)
            else:
                rel = np.arange(int(lens.sum())) - np.repeat(np.cumsum(lens) - lens, lens)
                pos = torch.from_numpy(np.repeat(dst_off, lens) + rel).cuda()
                idx = torch.from_numpy(np.repeat(offs, lens) + rel).cuda()
                assert torch.equal(dst[pos], src[idx]), (name, what)

        # the device handle, frame in HBM
        call_d, scr_d = maker(hd)
        for _ in range(3):
            call_d()
        verify("device handle")
        device_ms = events_ms(call_d, a.calls)
        del scr_d
        # the host handle
        dst.zero_()
        call, scr = maker(hh)
        for _ in range(3):
            call()
        verify("host handle")
        call_ms = events_ms(call, a.calls)
        g = torch.cuda.CUDAGraph()
        gs = torch.cuda.Stream()
        gs.wait_stream(s)
        with torch.cuda.graph(g, stream=gs):
            call(torch.cuda.current_stream())
        dst.zero_()
        g.replay()
        verify("graph")
        graph_ms = events_ms(g.replay, a.calls)
        fetch_ms = fetch_kernel_ms(call, 5)
        # the copy engine on the same byte count, pinned to device
        ce_src = pin_frame[:min(staged, pin_frame.numel())]
        ce_dst = torch.empty(ce_src.numel(), dtype=torch.uint8, device="cuda")
        ce_ms = events_ms(lambda: ce_dst.copy_(ce_src, non_blocking=True), a.calls)
        del ce_dst
        # the way before: the host handle per range into pinned memory, then the decoded bytes uploaded
        pin_out = torch.zeros(cap, dtype=torch.uint8).pin_memory()
        base = pin_out.data_ptr()
        dst2 = torch.empty(cap, dtype=torch.uint8, device="cuda")
        host = []
        for _ in range(a.host_calls if name != "whole_frame" else 1):
            t0 = time.perf_counter()
            for k in range(m):
                r = prod.lib.zxc_seekable_decompress_range(hs, base + int(dst_off[k]), int(lens[k]), int(offs[k]),
                                                           int(lens[k]))
                assert r == lens[k]
            dst2.copy_(pin_out, non_blocking=True)
            torch.cuda.synchronize()
            host.append((time.perf_counter() - t0) * 1e3)
        assert torch.equal(dst2[int(dst_off[0]):], dst[int(dst_off[0]):]), (name, "host loop")
        print(json.dumps({
            "workload": name, "card": info, "input_bytes": n, "frame_bytes": frame.numel(), "level": 3,
            "block_size": bs, "ranges": m, "bytes": int(lens.sum()), "staged_bytes": staged,
            "call_ms": round(call_ms, 4), "graph_ms": round(graph_ms, 4),
            "fetch_ms": round(fetch_ms, 4), "fetch_gbs": round(staged / fetch_ms / 1e6, 2),
            "copy_engine_ms": round(ce_ms, 4), "copy_engine_gbs": round(staged / ce_ms / 1e6, 2),
            "device_call_ms": round(device_ms, 4), "host_loop_ms": round(statistics.median(host), 3),
            "scratch_bytes": scr.numel()}), flush=True)
        del g, scr, dst, dst2, pin_out
    prod.lib.zxc_seekable_free(hs)
    L.zxc_b200_seekable_device_free(hh)
    L.zxc_b200_seekable_device_free(hd)


if __name__ == "__main__":
    main()
