"""zxc_b200_decompress_device_batch against a loop of zxc_b200_decompress_device and against one frame of the same size.

Silesia-shaped input at level 3 with 64 KiB blocks, compressed on the device.  Workloads:
  a   4 096 frames x 64 KiB, once seekable and once not
  b   65 536 frames x 4 KiB
  c   8 frames x 512 MiB
For the small-frame workloads 256 distinct pieces are compressed and the batch's frames are copies of them, each in
its own place of one buffer (the decode work does not depend on which piece a frame holds).  Per workload:
  batch    one batch call (CUDA events around it on one stream), median of --rounds after a warm-up call
  graph    the same call captured once in a CUDA graph and replayed, median of --rounds
  loop     zxc_b200_decompress_device once per frame on the same stream (events around the loop), median of
           --loop-rounds: the host enqueues 12 + 5 x 2 = 22 launches per frame, so the loop runs as fast as the host
           launches
  single   one zxc_b200_decompress_device of one frame of the whole input (the same total size)
Every output is checked against the input.  The card's name, power limit and SM clock are read in the same run.
Usage (GPU machine): python profiles/decompress_batch_bench.py [--rounds 20] [--loop-rounds 5] [--only a,b,c]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import zxc_corpus as zc  # noqa: E402
import zxc_ctypes as z  # noqa: E402
from zxc_b200 import device  # noqa: E402
from test_decompress_batch import bind_batch  # noqa: E402

BS = 65536
DISTINCT = 256


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return f"{torch.cuda.get_device_name()} (nvidia-smi: {e})"


def events_ms(fn, rounds):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()  # warm-up
    torch.cuda.synchronize()
    t = []
    for _ in range(rounds):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        t.append(e0.elapsed_time(e1))
    return statistics.median(t)


def workload(L, name, n_frames, frame_bytes, seek, a, piece):
    total = n_frames * frame_bytes
    src = torch.from_numpy(np.resize(piece, total)).cuda()
    s = torch.cuda.current_stream()
    # the frames: DISTINCT compressed pieces replicated, or every frame compressed when there are few
    k = min(n_frames, DISTINCT)
    comp = [device.compress(src[i * frame_bytes:(i + 1) * frame_bytes], level=3, block_size=BS,
                            seekable=bool(seek)).frame for i in range(k)]
    if k == n_frames:
        frames = comp
    else:
        sizes = [comp[i % k].numel() for i in range(n_frames)]
        offs = np.concatenate([[0], np.cumsum(sizes)[:-1]])
        blob = torch.empty(int(sum(sizes)), dtype=torch.uint8, device="cuda")
        frames = []
        for i in range(n_frames):
            v = blob[int(offs[i]):int(offs[i]) + sizes[i]]
            v.copy_(comp[i % k])
            frames.append(v)
        # the expected output repeats the first k pieces
        src = src[:k * frame_bytes].repeat((n_frames + k - 1) // k)[:total]
    out = torch.empty(total, dtype=torch.uint8, device="cuda")
    desc = torch.tensor([[f.data_ptr(), f.numel(), out.data_ptr() + i * frame_bytes, frame_bytes]
                         for i, f in enumerate(frames)], dtype=torch.int64).cuda()
    res = torch.zeros(n_frames, dtype=torch.int64, device="cuda")
    scr = torch.empty(int(L.zxc_b200_decompress_device_batch_scratch_size(n_frames, total, BS)), dtype=torch.uint8,
                      device="cuda")

    def batch():
        assert L.zxc_b200_decompress_device_batch(desc.data_ptr(), n_frames, None, scr.data_ptr(), scr.numel(),
                                                  res.data_ptr(), s.cuda_stream) == 0

    def check():
        assert bool((res == frame_bytes).all()), res.unique()
        assert torch.equal(out, src)
        out.zero_()
        res.zero_()

    r = {"workload": name, "frames": n_frames, "frame_bytes": frame_bytes, "seekable": bool(seek),
         "compressed_bytes": int(sum(f.numel() for f in frames))}
    r["batch_ms"] = events_ms(batch, a.rounds)
    check()
    g = torch.cuda.CUDAGraph()
    gs = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=gs):
        assert L.zxc_b200_decompress_device_batch(desc.data_ptr(), n_frames, None, scr.data_ptr(), scr.numel(),
                                                  res.data_ptr(), gs.cuda_stream) == 0
    r["graph_ms"] = events_ms(g.replay, a.rounds)
    check()
    del g
    one = torch.empty(int(L.zxc_b200_decompress_device_scratch_size(frame_bytes, BS)), dtype=torch.uint8,
                      device="cuda")

    def loop():
        for i, f in enumerate(frames):
            assert L.zxc_b200_decompress_device(f.data_ptr(), f.numel(), out.data_ptr() + i * frame_bytes,
                                                frame_bytes, None, one.data_ptr(), one.numel(),
                                                res.data_ptr() + 8 * i, s.cuda_stream) == 0

    r["loop_ms"] = events_ms(loop, a.loop_rounds)
    check()
    del one, scr
    whole = device.compress(src, level=3, block_size=BS, seekable=bool(seek)).frame
    one = torch.empty(int(L.zxc_b200_decompress_device_scratch_size(total, BS)), dtype=torch.uint8, device="cuda")

    def single():
        assert L.zxc_b200_decompress_device(whole.data_ptr(), whole.numel(), out.data_ptr(), total, None,
                                            one.data_ptr(), one.numel(), res.data_ptr(), s.cuda_stream) == 0

    r["single_ms"] = events_ms(single, a.rounds)
    assert int(res[0].item()) == total and torch.equal(out, src)
    for m in ("batch", "graph", "loop", "single"):
        r[m + "_gbps"] = round(total / r[m + "_ms"] / 1e6, 1)
        r[m + "_ms"] = round(r[m + "_ms"], 3)
    r["loop_over_batch"] = round(r["loop_ms"] / r["batch_ms"], 1)
    r["loop_over_graph"] = round(r["loop_ms"] / r["graph_ms"], 1)
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--loop-rounds", type=int, default=5)
    ap.add_argument("--only", default="a,b,c")
    a = ap.parse_args()
    L = bind_batch(z.ZxcLib(z.PRODUCT_SO).lib)
    piece = zc.silesia_shaped(64 << 20, seed=3)
    res = {"card": card(), "level": 3, "block_size": BS, "rounds": a.rounds, "loop_rounds": a.loop_rounds,
           "runs": []}
    print(json.dumps({"card": res["card"]}), flush=True)
    only = set(a.only.split(","))
    if "a" in only:
        for seek in (0, 1):
            res["runs"].append(workload(L, "a", 4096, 64 << 10, seek, a, piece))
    if "b" in only:
        res["runs"].append(workload(L, "b", 65536, 4 << 10, 0, a, piece))
    if "c" in only:
        res["runs"].append(workload(L, "c", 8, 512 << 20, 0, a, piece))
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
