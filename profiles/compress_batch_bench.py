"""zxc_b200_compress_device_batch against a loop of zxc_b200_compress_device and against one frame of the same size.

Silesia-shaped input (tests/zxc_corpus.py).  Workloads:
  a   4 096 buffers x 64 KiB, level 3, 64 KiB blocks
  b   65 536 buffers x 4 KiB, level 3, 4 KiB blocks
  c   4 096 buffers x 64 KiB, level 6, 64 KiB blocks
  d   8 buffers x 128 MiB, level 3, 64 KiB blocks, against one 1 GiB frame
For a to c the buffers are copies of 256 distinct pieces of the corpus, each in its own place of one input buffer
(the work of a buffer does not depend on which piece it holds), so every frame is checked against the single call's
frame of its piece.  Per workload:
  batch    one batch call (CUDA events around it on one stream), median of --rounds after a warm-up call
  graph    the same call captured once in a CUDA graph and replayed, median of --rounds
  loop     zxc_b200_compress_device once per buffer on the same stream (events around the loop).  The loop keeps one
           encode warp busy per call and is far too slow to run over a whole small-buffer workload, so for a to c it
           runs over the first --loop-sample buffers and the time is scaled up by n / sample (marked "scaled")
  single   one zxc_b200_compress_device over one buffer of the whole input (the same total bytes)
The card's name, power limit and SM clocks are read in the same run.
Usage (GPU machine): python profiles/compress_batch_bench.py [--rounds 5] [--loop-sample 32] [--only a,b,c,d]
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
from test_compress_batch import bind_batch  # noqa: E402
from test_compress_device import opts  # noqa: E402

DISTINCT = 256
WORKLOADS = {"a": (4096, 64 << 10, 3, 65536), "b": (65536, 4 << 10, 3, 4096), "c": (4096, 64 << 10, 6, 65536),
             "d": (8, 128 << 20, 3, 65536)}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return f"{torch.cuda.get_device_name()} (nvidia-smi: {e})"


def events_ms(fn, rounds, warm=True):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if warm:
        fn()
        torch.cuda.synchronize()
    t = []
    for _ in range(rounds):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        t.append(e0.elapsed_time(e1))
    return statistics.median(t)


class Single:
    """zxc_b200_compress_device on the current stream with a scratch and a result reused across calls"""

    def __init__(self, L, n, o):
        self.L, self.o = L, o
        self.size = int(L.zxc_b200_encode_scratch_size(n, C.byref(o)))
        self.scratch = torch.empty(self.size, dtype=torch.uint8, device="cuda")
        self.res = torch.zeros(1, dtype=torch.int64, device="cuda")

    def __call__(self, sp, n, dp, cap):
        rc = self.L.zxc_b200_compress_device(sp, n, dp, cap, C.byref(self.o), self.scratch.data_ptr(), self.size,
                                             self.res.data_ptr(), None, torch.cuda.current_stream().cuda_stream)
        assert rc == 0, rc


def run(L, key, rounds, sample):
    n, size, level, bs = WORKLOADS[key]
    o = opts(level, bs)
    total = n * size
    bound = int(L.zxc_compress_bound(size))
    if key == "d":
        data = torch.from_numpy(zc.silesia_shaped(total, seed=17)).cuda()
        pick = np.arange(n)
        offs = np.arange(n, dtype=np.int64) * size
        src = data
    else:
        corpus = torch.from_numpy(zc.silesia_shaped(DISTINCT * size, seed=17)).cuda()
        pick = np.random.default_rng(5).integers(0, DISTINCT, n)
        src = corpus.view(DISTINCT, size)[torch.from_numpy(pick).cuda()].reshape(-1).contiguous()
        offs = np.arange(n, dtype=np.int64) * size
    out = torch.empty(n * bound, dtype=torch.uint8, device="cuda")
    desc = torch.stack([src.data_ptr() + torch.from_numpy(offs), torch.full((n,), size, dtype=torch.int64),
                        out.data_ptr() + torch.arange(n, dtype=torch.int64) * bound,
                        torch.full((n,), bound, dtype=torch.int64)], 1).cuda()
    ssz = int(L.zxc_b200_compress_device_batch_scratch_size(n, total, C.byref(o)))
    scratch = torch.empty(ssz, dtype=torch.uint8, device="cuda")
    res = torch.zeros(n, dtype=torch.int64, device="cuda")

    def call(stream=None):
        rc = L.zxc_b200_compress_device_batch(desc.data_ptr(), n, C.byref(o), scratch.data_ptr(), ssz,
                                              res.data_ptr(), (stream or torch.cuda.current_stream()).cuda_stream)
        assert rc == 0, rc

    t_batch = events_ms(call, rounds)
    # every frame against the single call's frame of its piece (workload d: of its 128 MiB part)
    one = Single(L, size, o)
    dst = torch.empty(bound, dtype=torch.uint8, device="cuda")
    r = res.cpu().numpy()
    assert (r > 0).all(), r[r <= 0][:5]
    ob = out.view(n, bound)
    for p in np.unique(pick):
        i = int(np.nonzero(pick == p)[0][0])
        one(src.data_ptr() + int(offs[i]), size, dst.data_ptr(), bound)
        torch.cuda.synchronize()
        k = int(one.res.item())
        sel = torch.from_numpy(np.nonzero(pick == p)[0]).cuda()
        assert (res[sel] == k).all().item(), ("size", key, p)
        assert (ob[sel, :k] == dst[:k]).all().item(), ("bytes", key, p)
    # graph replay of the same call
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        call(s)
    res.zero_()
    t_graph = events_ms(g.replay, rounds)
    assert (res.cpu().numpy() == r).all()
    # the loop of single calls, over a sample for a to c
    m = n if key == "d" else min(sample, n)

    def loop():
        for i in range(m):
            one(src.data_ptr() + int(offs[i]), size, out.data_ptr() + i * bound, bound)

    t_loop = events_ms(loop, 1, warm=False) * n / m  # the single call is warm from the checks above
    # one frame of the whole input
    big = Single(L, total, o)
    bigout = torch.empty(int(L.zxc_compress_bound(total)), dtype=torch.uint8, device="cuda")
    t_single = events_ms(lambda: big(src.data_ptr(), total, bigout.data_ptr(), bigout.numel()), rounds)
    gb = total / 1e9
    row = {"workload": key, "frames": n, "frame_bytes": size, "level": level, "block_size": bs,
           "batch_ms": round(t_batch, 3), "batch_GBps": round(gb / t_batch * 1e3, 2),
           "graph_ms": round(t_graph, 3), "loop_ms": round(t_loop, 1), "loop_frames_run": m,
           "loop_scaled": m < n, "single_ms": round(t_single, 3), "single_GBps": round(gb / t_single * 1e3, 2),
           "loop_over_batch": round(t_loop / t_batch, 1), "frames_checked": n}
    del scratch, big, bigout, out
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--loop-sample", type=int, default=32)
    ap.add_argument("--only", default="a,b,c,d")
    ap.add_argument("--out", default=None, help="also write the rows as JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("compress_batch_bench: no CUDA device")
    L = bind_batch(z.ZxcLib(z.PRODUCT_SO).lib)
    rows = {"card": card(), "rows": []}
    print("card:", rows["card"], flush=True)
    for key in a.only.split(","):
        row = run(L, key, a.rounds, a.loop_sample)
        rows["rows"].append(row)
        print(json.dumps(row), flush=True)
    rows["card_after"] = card()
    print("card after:", rows["card_after"])
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
