"""Dictionary training on samples in HBM (zxc_b200_train_dict_device + zxc_b200_train_dict_huf_device) against the
same samples through the host trainers (zxc_train_dict + zxc_train_dict_huf), and the records pipeline end to end.

    python profiles/train_device_bench.py [--cases bench,records4g,small100] [--repeat 3] [--no-pipeline]

Cases (DESIGN.md section 6):
  bench      the bench's dictionary corpus: the first 4 096 x 4 KiB records, 16 KiB content
  records4g  1 Mi x 4 KiB records (4 GiB), 64 KiB content
  small100   1 Mi samples of 100 bytes, 64 KiB content
Each case trains the content and then the table from it, from host memory and from one CUDA tensor holding the same
samples back to back, after one warm-up call of each.  Whole calls are timed with the host clock (the calls are
synchronous), best of --repeat; per-phase device times come from zxc_b200_train_phase_times.  The device path runs
twice: with the samples at the tensor's start (every 4 KiB record 16-byte aligned in source and corpus) and one byte
in (every piece misaligned).  One more device run per layout goes under torch.profiler to time the zxc_ps_gather
kernel alone; its GB/s counts the corpus bytes once (each is read once and written once).

Pipeline (records4g's records): DeviceDict.train on the records in HBM (content and table), then one
zxc_b200_compress_blocks_device_using_dict call at level 5 over all records, each into its own slot of one arena.

Prints one line per case, then one JSON line with the GPU's name, power limit and max SM clock read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import zxc_b200.device as dv  # noqa: E402
import zxc_corpus as zc  # noqa: E402

L = dv.lib
PHASES = ["upload", "count", "segments", "host_sort", "pick", "slice_upload", "histogram_encode", "code_lengths"]
for name in ("zxc_train_dict", "zxc_train_dict_huf"):
    getattr(L, name).argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t] + (
        [C.c_void_p] if name.endswith("huf") else [])
L.zxc_train_dict.restype = C.c_int64
L.zxc_train_dict_huf.restype = C.c_int
L.zxc_b200_train_phase_times.restype = C.c_int
L.zxc_b200_train_phase_times.argtypes = [C.c_void_p, C.c_int]
L.zxc_b200_compress_blocks_device_scratch_size.restype = C.c_size_t
L.zxc_b200_compress_blocks_device_scratch_size.argtypes = [C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def arrays(base, n, size):
    ptrs = np.uint64(base) + np.arange(n, dtype=np.uint64) * np.uint64(size)
    return ptrs, np.full(n, size, np.uint64)


def train(dev, ptrs, sizes, cap):
    """(content + table bytes, content s, table s, phase ms) of one content + table training"""
    n = ptrs.size
    out = C.create_string_buffer(cap)
    huf = C.create_string_buffer(128)
    st = torch.cuda.current_stream().cuda_stream
    t0 = time.perf_counter()
    if dev:
        r = L.zxc_b200_train_dict_device(ptrs.ctypes.data, sizes.ctypes.data, n, out, cap, st)
    else:
        r = L.zxc_train_dict(ptrs.ctypes.data, sizes.ctypes.data, n, out, cap)
    t1 = time.perf_counter()
    assert r > 0, r
    if dev:
        h = L.zxc_b200_train_dict_huf_device(ptrs.ctypes.data, sizes.ctypes.data, n, out, r, huf, st)
    else:
        h = L.zxc_train_dict_huf(ptrs.ctypes.data, sizes.ctypes.data, n, out, r, huf)
    t2 = time.perf_counter()
    assert h == 0, h
    ms = np.zeros(len(PHASES))
    L.zxc_b200_train_phase_times(ms.ctypes.data, len(PHASES))
    return out.raw[:r] + huf.raw, t1 - t0, t2 - t1, ms


def best_of(k, fn):
    best = None
    for _ in range(k):
        r = fn()
        if best is None or r[1] + r[2] < best[1] + best[2]:
            best = r
    return best


def gather_kernel_ms(ptrs, sizes, cap):
    """device time of the zxc_ps_gather launches of one content training, from torch.profiler"""
    out = C.create_string_buffer(cap)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        assert L.zxc_b200_train_dict_device(ptrs.ctypes.data, sizes.ctypes.data, ptrs.size, out, cap, None) > 0
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "zxc_ps_gather" in e.key)
    return us / 1e3


def case_row(case, data, size, cap, repeat, d_data, d_mis):
    n = data.size // size
    hp, hs = arrays(data.ctypes.data, n, size)
    warm = min(n, max(1, (1 << 20) // size))
    train(False, hp[:warm].copy(), hs[:warm].copy(), cap)
    host = best_of(repeat, lambda: train(False, hp, hs, cap))
    row = {"samples": n, "bytes": int(data.size), "capacity": cap,
           "host_s": round(host[1] + host[2], 4), "host_content_s": round(host[1], 4),
           "host_table_s": round(host[2], 4), "host_phases_ms": {p: round(float(v), 3) for p, v in zip(PHASES, host[3])}}
    for label, base in (("aligned", d_data.data_ptr()), ("misaligned", d_mis.data_ptr() + 1)):
        dp, ds = arrays(base, n, size)
        train(True, dp[:warm].copy(), ds[:warm].copy(), cap)
        dev = best_of(repeat, lambda: train(True, dp, ds, cap))
        gk = gather_kernel_ms(dp, ds, cap)
        row[label] = {"device_s": round(dev[1] + dev[2], 4), "device_content_s": round(dev[1], 4),
                      "device_table_s": round(dev[2], 4),
                      "phases_ms": {p: round(float(v), 3) for p, v in zip(PHASES, dev[3])},
                      "gather_kernel_ms": round(gk, 3),
                      "gather_kernel_gbs": round(data.size / (gk / 1e3) / 1e9, 1) if gk > 0 else None,
                      "upload_slot_gbs": round(data.size / (dev[3][0] / 1e3) / 1e9, 1) if dev[3][0] > 0 else None,
                      "identical": dev[0] == host[0]}
    return row


def pipeline(data, size):
    """records in HBM -> DeviceDict.train -> compress_blocks (level 5), timed per stage and in all"""
    n = data.size // size
    d_in = torch.from_numpy(data).cuda()
    stride = (size + 8 + 68 + 4 + 15) // 16 * 16  # zxc_compress_block_bound, 16-byte aligned slots
    arena = torch.empty(n * stride, dtype=torch.uint8, device="cuda")
    idx = torch.arange(n, dtype=torch.int64, device="cuda")
    desc = torch.stack([d_in.data_ptr() + idx * size, torch.full_like(idx, size), arena.data_ptr() + idx * stride,
                        torch.full_like(idx, stride)], 1).contiguous()
    co = dv._Opts(level=5)
    ss = int(L.zxc_b200_compress_blocks_device_scratch_size(n, data.size, size, C.byref(co)))
    scr = torch.empty(ss, dtype=torch.uint8, device="cuda")
    res = torch.empty(n, dtype=torch.int64, device="cuda")
    sizes = np.full(n, size, np.int64)

    def run():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dd = dv.DeviceDict.train(d_in, sizes)
        t1 = time.perf_counter()
        rc = L.zxc_b200_compress_blocks_device_using_dict(desc.data_ptr(), n, C.byref(co), dd.handle, scr.data_ptr(),
                                                          ss, res.data_ptr(), None)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        assert rc == 0 and bool((res > 0).all()), rc
        dd.close()
        return t1 - t0, t2 - t1

    run()
    t = min((run() for _ in range(2)), key=sum)
    return {"records": n, "bytes": int(data.size), "train_s": round(t[0], 4), "compress_blocks_s": round(t[1], 4),
            "total_s": round(sum(t), 4), "compressed_bytes": int(res.sum().item())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="bench,records4g,small100")
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--no-pipeline", action="store_true")
    a = ap.parse_args()
    res = {"gpu": gpu_info(), "cases": {}}
    for case in a.cases.split(","):
        if case == "bench":
            data, size, cap = zc.records(4096, 4096), 4096, 16384
        elif case == "records4g":
            data, size, cap = zc.records(1 << 20, 4096), 4096, 65535
        elif case == "small100":
            data, size, cap = zc.records(1 << 20, 100, seed=5), 100, 65535
        else:
            raise SystemExit(f"unknown case {case}")
        d_data = torch.from_numpy(data).cuda()
        d_mis = torch.empty(data.size + 1, dtype=torch.uint8, device="cuda")
        d_mis[1:] = d_data
        res["cases"][case] = case_row(case, data, size, cap, a.repeat, d_data, d_mis)
        print(f"# {case}: {json.dumps(res['cases'][case])}", file=sys.stderr, flush=True)
        del d_data, d_mis
        if case == "records4g" and not a.no_pipeline:
            res["pipeline"] = pipeline(data, size)
            print(f"# pipeline: {json.dumps(res['pipeline'])}", file=sys.stderr, flush=True)
        del data
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
