"""zxc_b200_add_seek_table_device on a large frame without a table, and the decode it speeds up.

Input: --gib GiB (default 4) silesia-shaped at level 3, compressed on the device without a table, at 64 KiB and 4 KiB
blocks.  Per block size, one JSON line with:
  seal_ms           zxc_b200_add_seek_table_device (CUDA events, median of --calls, the frame restored in between)
  decode_plain_ms   zxc_b200_decompress_device on the frame without its table
  decode_sealed_ms  the same call on the sealed frame
  seal_plus_sealed_ms, and the path that decided the chain (1: speculation, 2: walk)
  kernels_ms        per-kernel time of one sealing call, from torch.profiler
  fallback_ms       the worst case: a frame of the same size whose scratch holds too few candidates, so the walk decides
The sealed frame is checked byte for byte against zxc_b200_compress_device with seekable = 1, and both decodes against
the input.  The card's name, power limit and max SM clock are read in the same run.
Usage (GPU machine): python profiles/seek_table_device_bench.py [--gib 4] [--calls 10]
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
from test_decompress_device import bind as bind_dd, dopts  # noqa: E402
from test_seek_table_device import bind  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def events_ms(fn, calls, before=None):
    ts = []
    for _ in range(calls):
        if before is not None:
            before()
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
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--block-sizes", default="65536,4096")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    prod = z.ZxcLib(z.PRODUCT_SO)
    L = bind(bind_dd(prod.lib))
    info = card()
    n = int(a.gib * (1 << 30))
    piece = zc.silesia_shaped(256 << 20, seed=3)
    src = torch.from_numpy(np.resize(piece, n)).cuda()
    del piece
    s = torch.cuda.current_stream()
    for bs in [int(x) for x in a.block_sizes.split(",")]:
        plain = device.compress(src, level=3, block_size=bs).frame
        want = device.compress(src, level=3, block_size=bs, seekable=True).frame
        size, nb = plain.numel(), -(-n // bs)
        buf = torch.empty(want.numel(), dtype=torch.uint8, device="cuda")
        ss = int(L.zxc_b200_seek_table_device_scratch_size(size, nb))
        scr = torch.empty(ss, dtype=torch.uint8, device="cuda")
        res = torch.zeros(1, dtype=torch.int64, device="cuda")

        def restore():
            buf[:size].copy_(plain)

        def seal(scratch=scr, scratch_size=ss):
            assert L.zxc_b200_add_seek_table_device(buf.data_ptr(), size, buf.numel(), scratch.data_ptr(),
                                                    scratch_size, res.data_ptr(), s.cuda_stream) == 0

        restore()
        seal()
        torch.cuda.synchronize()
        assert int(res.item()) == want.numel() and torch.equal(buf, want), "sealed frame"
        path = int(scr[:4].cpu().numpy().view(np.uint32)[0]) if scr.data_ptr() % 256 == 0 else -1
        seal_ms = events_ms(seal, a.calls, restore)

        out = torch.empty(n, dtype=torch.uint8, device="cuda")
        dscr = torch.empty(L.zxc_b200_decompress_device_scratch_size(n, bs), dtype=torch.uint8, device="cuda")
        dres = torch.zeros(1, dtype=torch.int64, device="cuda")
        o = dopts()

        def decode(frame):
            assert L.zxc_b200_decompress_device(frame.data_ptr(), frame.numel(), out.data_ptr(), n, C.byref(o),
                                                dscr.data_ptr(), dscr.numel(), dres.data_ptr(), s.cuda_stream) == 0

        timings = {}
        for name, frame in (("plain", plain), ("sealed", want)):
            decode(frame)
            torch.cuda.synchronize()
            assert int(dres.item()) == n and torch.equal(out, src), name
            timings[name] = events_ms(lambda: decode(frame), a.calls)
        del out, dscr

        # the per-kernel split of one sealing call
        restore()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            seal()
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.events():
            if "zxc_dindex" in e.name:
                k = e.name.split("(")[0].replace("void ", "")
                kernels[k] = kernels.get(k, 0.0) + e.device_time_total / 1000.0

        # the worst case: the walk decides.  Every block's payload is overwritten with valid-looking RAW headers of
        # 16-byte blocks, the block headers kept: the chain, and so the result, stay as they are, but the candidates
        # outnumber the list of a scratch sized for the frame's blocks, so the guess is abandoned.
        v = 16 << 24
        h = v ^ 0x9E3779B97F4A7C15
        h ^= (h << 13) & (2 ** 64 - 1)
        h ^= h >> 7
        h ^= (h << 17) & (2 ** 64 - 1)
        fake = np.frombuffer((v | ((((h >> 32) ^ h) & 0xFF) << 56)).to_bytes(8, "little"), np.uint8)
        hostile = plain.cpu().numpy().copy()
        pos, planted = 16, 0
        while planted < 2 * nb + 4096 and hostile[pos] != 255:
            comp = int.from_bytes(hostile[pos + 3:pos + 7].tobytes(), "little")
            k = comp // 8 * 8
            hostile[pos + 8:pos + 8 + k] = np.tile(fake, k // 8)
            planted += k // 8
            pos += 8 + comp
        hostile = torch.from_numpy(hostile).cuda()

        def restore_hostile():
            buf[:size].copy_(hostile)

        restore_hostile()
        seal()
        torch.cuda.synchronize()
        fpath = int(scr[:4].cpu().numpy().view(np.uint32)[0]) if scr.data_ptr() % 256 == 0 else -1
        fres = int(res.item())
        assert fres == want.numel() and torch.equal(buf[size - 12:], want[size - 12:]), "fallback result"
        fallback_ms = events_ms(seal, max(2, a.calls // 5), restore_hostile)
        print(json.dumps({
            "block_size": bs, "input_bytes": n, "frame_bytes": size, "blocks": nb, "scratch_bytes": ss,
            "path": path, "seal_ms": round(seal_ms, 3), "decode_plain_ms": round(timings["plain"], 3),
            "decode_sealed_ms": round(timings["sealed"], 3),
            "seal_plus_sealed_ms": round(seal_ms + timings["sealed"], 3),
            "kernels_ms": {k: round(v, 4) for k, v in sorted(kernels.items(), key=lambda x: -x[1])},
            "fallback": {"path": fpath, "result": fres, "ms": round(fallback_ms, 3), "planted": planted},
            "card": info}), flush=True)
        del plain, want, buf, scr, hostile


if __name__ == "__main__":
    main()
