"""Dictionary training, product (GPU) against the reference library on the same host.

    python profiles/train_bench.py [--cases bench,records4g,small100] [--repeat N]

Each case trains the content (zxc_train_dict) and then the shared literal table from it (zxc_train_dict_huf), with
both libraries, after one warm-up call of the product.  Whole calls are timed with the host clock; the product's
per-phase device times (CUDA events) and host times come from zxc_b200_train_phase_times.  Prints one JSON line.
Needs oracle/_ref/libzxc_ref.so (built from the reference sources) and a CUDA device.

Cases:
  bench      the bench's dictionary corpus: the first 4 096 x 4 KiB records, 16 KiB content
  records4g  1 Mi x 4 KiB records (4 GiB), 64 KiB content
  small100   1 Mi samples of 100 bytes, 64 KiB content: the table trainer parses about 80 k slices, each against the
             whole dictionary
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zxc_corpus as zc  # noqa: E402
import zxc_ctypes as z  # noqa: E402

PHASES = ["upload", "count", "segments", "host_sort", "pick", "slice_upload", "histogram_encode", "code_lengths"]


def bind(path):
    L = C.CDLL(path)
    L.zxc_train_dict.restype = C.c_int64
    L.zxc_train_dict.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    L.zxc_train_dict_huf.restype = C.c_int
    L.zxc_train_dict_huf.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    return L


def samples(data, size):
    n = data.size // size
    ptrs = (C.c_void_p * n)(*range(data.ctypes.data, data.ctypes.data + n * size, size))
    sizes = (C.c_size_t * n)(*([size] * n))
    return ptrs, sizes, n


def train(L, S, cap):
    ptrs, sizes, n = S
    out = np.zeros(cap, np.uint8)
    huf = np.zeros(128, np.uint8)
    t0 = time.perf_counter()
    r = L.zxc_train_dict(ptrs, sizes, n, out.ctypes.data, cap)
    t1 = time.perf_counter()
    assert r > 0, r
    h = L.zxc_train_dict_huf(ptrs, sizes, n, out.ctypes.data, r, huf.ctypes.data)
    t2 = time.perf_counter()
    assert h == 0, h
    return out[:r].tobytes() + huf.tobytes(), t1 - t0, t2 - t1


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, pl = [s.strip() for s in q.split(",")]
        return name, pl
    except Exception:
        return "unknown", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="bench,records4g,small100")
    ap.add_argument("--repeat", type=int, default=3, help="timed product runs per case (best is reported)")
    a = ap.parse_args()
    prod, ref = bind(z.PRODUCT_SO), bind(z.REF_SO)
    prod.zxc_b200_train_phase_times.restype = C.c_int
    prod.zxc_b200_train_phase_times.argtypes = [C.c_void_p, C.c_int]
    name, pl = card()
    res = {"card": name, "power_limit": pl, "cases": {}}
    for case in a.cases.split(","):
        if case == "bench":
            data, size, cap = zc.records(4096, 4096), 4096, 16384
        elif case == "records4g":
            data, size, cap = zc.records(1 << 20, 4096), 4096, 65535
        elif case == "small100":
            data, size, cap = zc.records(1 << 20, 100, seed=5), 100, 65535
        else:
            raise SystemExit(f"unknown case {case}")
        S = samples(data, size)
        train(prod, samples(data[: 1 << 20], size), cap)  # warm-up: device context, buffers
        best = None
        for _ in range(a.repeat):
            out_p, tc, th = train(prod, S, cap)
            ms = np.zeros(len(PHASES))
            prod.zxc_b200_train_phase_times(ms.ctypes.data, len(PHASES))
            if best is None or tc + th < best[0]:
                best = (tc + th, tc, th, ms.copy())
        out_r, rc_, rh_ = train(ref, S, cap)
        res["cases"][case] = {
            "samples": S[2], "bytes": int(data.size), "capacity": cap,
            "product_s": round(best[0], 4), "product_content_s": round(best[1], 4), "product_table_s": round(best[2], 4),
            "reference_s": round(rc_ + rh_, 4), "reference_content_s": round(rc_, 4), "reference_table_s": round(rh_, 4),
            "phases_ms": {p: round(float(v), 3) for p, v in zip(PHASES, best[3])},
            "identical": out_p == out_r,
        }
        del data, S
        print(f"# {case}: {json.dumps(res['cases'][case])}", file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
