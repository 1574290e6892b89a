"""Push-streaming throughput: the product's zxc_cstream_* / zxc_dstream_* (blocks batched into one launch per call)
against the reference's pstream on the same host CPU, and one-shot zxc_compress / zxc_decompress of both.

    python profiles/pstream_bench.py [--mib 64] [--reps 3] [--out results.json]

Input: zxc_corpus.silesia_shaped (seeded).  Chunks: the stream's own in_size() / out_size() hint (one block per
call) and 64 MiB.  Levels 1 and 3, 64 KiB and 512 KiB blocks.  MB/s = uncompressed bytes / wall time of the whole
stream (host clock; every product call ends in a device synchronise), median of --reps after one warm-up run.
Every stream's output is checked against the one-shot result.  Prints a Markdown table, then one JSON line with the
GPU name and power limit beside the numbers (also written to --out, when given).
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

import zxc_corpus as zc  # noqa: E402
import zxc_ctypes as z  # noqa: E402
import zxc_pstream_driver as pd  # noqa: E402

CHUNK_BIG = 64 << 20


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def run_c(L, src, level, bs, chunk):
    """(seconds, output) of one compress stream fed `chunk` bytes per call (0: the in_size() hint)"""
    s = pd.Stream(L, "c", z.CompressOpts(level=level, block_size=bs))
    n_in = chunk or L.zxc_cstream_in_size(s.h)
    cap = max(L.zxc_cstream_out_size(s.h), n_in + n_in // 8 + 4096) if chunk else L.zxc_cstream_out_size(s.h)
    out = (C.c_uint8 * cap)()
    sbuf = C.create_string_buffer(src, len(src))
    base = C.cast(sbuf, C.c_void_p).value
    parts = []
    t0 = time.perf_counter()
    for off in range(0, len(src), n_in):
        n = min(n_in, len(src) - off)
        ib = pd.InBuf(base + off, n, 0)
        while True:
            ob = pd.OutBuf(C.cast(out, C.c_void_p), cap, 0)
            r = L.zxc_cstream_compress(s.h, C.byref(ob), C.byref(ib))
            assert r >= 0, r
            parts.append(C.string_at(C.addressof(out), ob.pos))
            if r == 0:
                break
    while True:
        ob = pd.OutBuf(C.cast(out, C.c_void_p), cap, 0)
        r = L.zxc_cstream_end(s.h, C.byref(ob))
        assert r >= 0, r
        parts.append(C.string_at(C.addressof(out), ob.pos))
        if r == 0:
            break
    dt = time.perf_counter() - t0
    s.close()
    return dt, b"".join(parts)


def run_d(L, frame, chunk, total):
    """(seconds, output) of one decompress stream fed `chunk` bytes per call (0: in_size() / out_size() hints)"""
    s = pd.Stream(L, "d", z.DecompressOpts())
    fbuf = C.create_string_buffer(frame, len(frame))
    base = C.cast(fbuf, C.c_void_p).value
    big = (C.c_uint8 * max(CHUNK_BIG, 1))()
    parts = []
    off = 0
    t0 = time.perf_counter()
    while not L.zxc_dstream_finished(s.h):
        n_in = chunk or L.zxc_dstream_in_size(s.h)
        cap = chunk or L.zxc_dstream_out_size(s.h)
        n = min(n_in, len(frame) - off)
        ib = pd.InBuf(base + off, n, 0)
        while True:
            ob = pd.OutBuf(C.cast(big, C.c_void_p), cap, 0)
            r = L.zxc_dstream_decompress(s.h, C.byref(ob), C.byref(ib))
            assert r >= 0, r
            parts.append(C.string_at(C.addressof(big), ob.pos))
            if L.zxc_dstream_finished(s.h) or (ib.pos == ib.size and ob.pos < cap):
                break
        off += ib.pos
    dt = time.perf_counter() - t0
    s.close()
    out = b"".join(parts)
    assert len(out) == total
    return dt, out


def timed(f):
    t0 = time.perf_counter()
    r = f()
    return time.perf_counter() - t0, r


def med(f, reps):
    f()  # warm-up: context creation, buffer growth, module load
    ts = []
    res = None
    for _ in range(reps):
        t, res = f()
        ts.append(t)
    return statistics.median(ts), res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    P = pd.bind(C.CDLL(z.PRODUCT_SO))
    if P.zxc_b200_device_count() <= 0:
        sys.exit("pstream_bench: no CUDA device")
    if not z.have_ref():
        sys.exit("pstream_bench: oracle/_ref/libzxc_ref.so is missing")
    prod, ref = z.ZxcLib(z.PRODUCT_SO), z.ZxcLib(z.REF_SO)
    R = pd.bind(ref.lib)
    src = zc.silesia_shaped(a.mib << 20, seed=1)
    sb = src.tobytes()
    mb = len(sb) / 1e6
    rows = []
    for level in (1, 3):
        for bs in (64 << 10, 512 << 10):
            frame = ref.compress(src, level=level, block_size=bs).tobytes()
            t_pc, f_pc = med(lambda: timed(lambda: prod.compress(src, level=level, block_size=bs)), a.reps)
            t_rc, _ = med(lambda: timed(lambda: ref.compress(src, level=level, block_size=bs)), a.reps)
            t_pd, _ = med(lambda: timed(lambda: prod.decompress(frame, len(sb))), a.reps)
            t_rd, _ = med(lambda: timed(lambda: ref.decompress(frame, len(sb))), a.reps)
            assert f_pc.tobytes() == frame
            for chunk, cname in ((0, "hint"), (CHUNK_BIG, "64 MiB")):
                tc_p, out_c = med(lambda: run_c(P, sb, level, bs, chunk), a.reps)
                tc_r, _ = med(lambda: run_c(R, sb, level, bs, chunk), a.reps)
                td_p, out_d = med(lambda: run_d(P, frame, chunk, len(sb)), a.reps)
                td_r, _ = med(lambda: run_d(R, frame, chunk, len(sb)), a.reps)
                assert out_c == frame and out_d == sb
                rows.append(dict(level=level, block_size=bs, chunk=cname,
                                 cstream_gpu=mb / tc_p, cstream_ref=mb / tc_r, dstream_gpu=mb / td_p, dstream_ref=mb / td_r,
                                 compress_gpu=mb / t_pc, compress_ref=mb / t_rc, decompress_gpu=mb / t_pd,
                                 decompress_ref=mb / t_rd))
                r = rows[-1]
                print(f"| {level} | {bs >> 10} KiB | {cname} | {r['cstream_gpu']:.0f} | {r['cstream_ref']:.0f} | "
                      f"{r['dstream_gpu']:.0f} | {r['dstream_ref']:.0f} | {r['compress_gpu']:.0f} | {r['compress_ref']:.0f} | "
                      f"{r['decompress_gpu']:.0f} | {r['decompress_ref']:.0f} |", flush=True)
    info = dict(gpu=gpu_info(), input_mib=a.mib, reps=a.reps, host_cpus=os.cpu_count(), rows=rows)
    print(json.dumps(info))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
