"""Push streaming in HBM: zxc_b200_cstream_device / _dstream_device against the host streams (zxc_cstream_* /
zxc_dstream_*) on the same chunks, and one zxc_b200_compress_device / zxc_b200_decompress_device call on the whole
buffer.

    python profiles/pstream_device_bench.py [--mib 1024] [--rounds 3] [--chunks 1,16,64,256] [--out results.json]
    python profiles/pstream_device_bench.py --phases [--mib 256] [--chunks 64,256]

--phases times one device dstream and cstream per case under torch.profiler instead: device time of the header walk,
the decode or encode kernels, the trailers and the gather, beside the stream's wall time (the rest is host work,
copies and synchronisations).

Input: zxc_corpus.silesia_shaped (seeded), levels 1 and 3, 64 KiB and 512 KiB blocks.  Chunks of 1, 16, 64 and 256 MiB
with an out capacity equal to the chunk.  GB/s = uncompressed bytes / host-clock time of the whole stream (every
device-stream call returns with its work complete; the one-shot calls are timed around a stream synchronise), median
of --rounds alternating rounds.  Every stream's output is checked against the one-shot result.  Prints one line per
case, then one JSON line with the GPU's name, power limit and max SM clock beside the numbers.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import zxc_corpus as zc  # noqa: E402
import zxc_ctypes as z  # noqa: E402
import zxc_pstream_driver as pd  # noqa: E402
from test_pstream_device import bind_device  # noqa: E402

MIB = 1 << 20


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def dev_stream(P, kind, opts, src, chunk, out, st):
    """seconds and output bytes of one device stream over src (a CUDA uint8 tensor) in chunks of `chunk` bytes"""
    h = getattr(P, f"zxc_b200_{kind}stream_device_create")(C.byref(opts))
    call = P.zxc_b200_cstream_device_compress if kind == "c" else P.zxc_b200_dstream_device_decompress
    total = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for off in range(0, src.numel(), chunk):
        n = min(chunk, src.numel() - off)
        ib = pd.InBuf(src.data_ptr() + off, n, 0)
        while True:
            ob = pd.OutBuf(out.data_ptr(), chunk, 0)
            r = call(h, C.byref(ob), C.byref(ib), st)
            assert r >= 0, r
            total += ob.pos
            if (kind == "c" and r == 0) or (kind == "d" and ob.pos < chunk):
                break
    while True:
        ob = pd.OutBuf(out.data_ptr(), chunk, 0)
        if kind == "c":
            r = P.zxc_b200_cstream_device_end(h, C.byref(ob), st)
        else:
            r = P.zxc_b200_dstream_device_decompress(h, C.byref(ob), C.byref(pd.InBuf(None, 0, 0)), st)
        assert r >= 0, r
        total += ob.pos
        if r == 0 or (kind == "d" and ob.pos < chunk):
            break
    dt = time.perf_counter() - t0
    getattr(P, f"zxc_b200_{kind}stream_device_free")(h)
    return dt, total


def host_stream(P, kind, opts, src, chunk, out):
    h = getattr(P, f"zxc_{kind}stream_create")(C.byref(opts))
    call = P.zxc_cstream_compress if kind == "c" else P.zxc_dstream_decompress
    base, optr = src.ctypes.data, out.ctypes.data
    total = 0
    t0 = time.perf_counter()
    for off in range(0, src.size, chunk):
        ib = pd.InBuf(base + off, min(chunk, src.size - off), 0)
        while True:
            ob = pd.OutBuf(optr, chunk, 0)
            r = call(h, C.byref(ob), C.byref(ib))
            assert r >= 0, r
            total += ob.pos
            if (kind == "c" and r == 0) or (kind == "d" and ob.pos < chunk):
                break
    while True:
        ob = pd.OutBuf(optr, chunk, 0)
        r = P.zxc_cstream_end(h, C.byref(ob)) if kind == "c" else \
            P.zxc_dstream_decompress(h, C.byref(ob), C.byref(pd.InBuf(None, 0, 0)))
        assert r >= 0, r
        total += ob.pos
        if r == 0 or (kind == "d" and ob.pos < chunk):
            break
    dt = time.perf_counter() - t0
    getattr(P, f"zxc_{kind}stream_free")(h)
    return dt, total


def phases(P, data, d_data, chunks, st):
    """per-kernel device time of one device stream per case, from torch.profiler"""
    import zxc_b200.device as dv
    from torch.profiler import ProfilerActivity, profile
    groups = (("walk", "zxc_ps_walk"), ("gather", "zxc_ps_gather"), ("trailers", "zxc_ps_trailers"),
              ("decode", "zxc_decode_kernel"), ("encode", "zxc_encode_kernel"))
    rows = []
    for level, bs in ((1, 64 << 10), (3, 64 << 10), (1, 512 << 10)):
        frame = dv.compress(d_data, level=level, block_size=bs).frame
        for ch in chunks:
            out = torch.empty(ch, dtype=torch.uint8, device="cuda")
            for kind, src, opts in (("d", frame, z.DecompressOpts()), ("c", d_data, z.CompressOpts(level=level,
                                                                                                  block_size=bs))):
                dev_stream(P, kind, opts, src, ch, out, st.cuda_stream)  # warm-up: buffers grown
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    wall, _ = dev_stream(P, kind, opts, src, ch, out, st.cuda_stream)
                ms = {g: 0.0 for g, _ in groups}
                other = 0.0
                for e in prof.key_averages():
                    t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1e3
                    g = next((g for g, k in groups if k in e.key), None)
                    if g:
                        ms[g] += t
                    elif "Memcpy" in e.key or "Memset" in e.key:
                        other += t
                r = {"level": level, "block_size": bs, "chunk_mib": ch // MIB, "stream": kind,
                     "gbs": round(data.size / wall / 1e9, 2), "wall_ms": round(wall * 1e3, 2),
                     **{g + "_ms": round(v, 2) for g, v in ms.items() if v}, "copies_ms": round(other, 2)}
                print(json.dumps(r))
                rows.append(r)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--chunks", default="1,16,64,256")
    ap.add_argument("--host", type=int, default=1, help="also time the host streams")
    ap.add_argument("--phases", action="store_true", help="per-kernel device time instead of the rate table")
    ap.add_argument("--out")
    a = ap.parse_args()
    import zxc_b200.device as dv
    prod = z.ZxcLib(z.PRODUCT_SO)
    P = bind_device(pd.bind(prod.lib))
    info = gpu_info()
    print("gpu:", info)
    data = zc.silesia_shaped(a.mib * MIB, seed=1)[: a.mib * MIB]
    n = data.size
    d_data = torch.from_numpy(data).cuda()
    st = torch.cuda.current_stream()
    if a.phases:
        rows = phases(P, data, d_data, [int(x) * MIB for x in a.chunks.split(",")], st)
        print(json.dumps({"gpu": info, "mib": a.mib, "phases": rows}))
        return
    rows = []
    for level in (1, 3):
        for bs in (64 << 10, 512 << 10):
            fr = dv.compress(d_data, level=level, block_size=bs)
            frame = fr.frame
            h_frame = frame.cpu().numpy()
            t_one_c, t_one_d = [], []
            res = {}
            for rnd in range(a.rounds):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                dv.compress(d_data, level=level, block_size=bs)
                t_one_c.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                dv.decompress_frame(frame, capacity=n)
                torch.cuda.synchronize()
                t_one_d.append(time.perf_counter() - t0)
                for ch in [int(x) * MIB for x in a.chunks.split(",")]:
                    out = torch.empty(ch, dtype=torch.uint8, device="cuda")
                    hout = np.empty(ch, np.uint8)
                    co = z.CompressOpts(level=level, block_size=bs)
                    do = z.DecompressOpts()
                    for what, fn in (("dev_c", lambda: dev_stream(P, "c", co, d_data, ch, out, st.cuda_stream)),
                                     ("dev_d", lambda: dev_stream(P, "d", do, frame, ch, out, st.cuda_stream)),
                                     ("host_c", lambda: host_stream(P, "c", co, data, ch, hout)),
                                     ("host_d", lambda: host_stream(P, "d", do, h_frame, ch, hout))):
                        if what.startswith("host") and not a.host:
                            continue
                        dt, total = fn()
                        assert total == (frame.numel() if what.endswith("c") else n), (what, total)
                        res.setdefault((what, ch), []).append(dt)
            gb = lambda ts: n / statistics.median(ts) / 1e9  # noqa: E731
            one = {"level": level, "block_size": bs, "oneshot_compress_gbs": round(gb(t_one_c), 2),
                   "oneshot_decompress_gbs": round(gb(t_one_d), 2)}
            print(json.dumps(one))
            rows.append(one)
            for (what, ch), ts in sorted(res.items()):
                r = {"level": level, "block_size": bs, "chunk_mib": ch // MIB, "what": what, "gbs": round(gb(ts), 2)}
                print(json.dumps(r))
                rows.append(r)
    result = {"gpu": info, "mib": a.mib, "rounds": a.rounds, "rows": rows}
    print(json.dumps(result))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
