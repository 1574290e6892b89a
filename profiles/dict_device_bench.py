"""Prepared device dictionaries against host dictionary bytes, in the block API and in small calls.

Three measurements, all printed as one JSON object with the card's name, power limit and SM clocks read in the same
run:
  records   BASELINE.json configs[3]'s shape: 1 Mi records of 4 KiB (zxc_corpus.records), a 16 KiB dictionary from
            the reference's trainer, level 5, through zxc_b200_compress_blocks_device / _decompress_blocks_device with
            the dictionary as host bytes (staged per call) and through the _using_dict variants with one handle.  Per
            round each of the four calls runs once between CUDA events on one stream, alternating; medians over
            --rounds.  Outputs of the two forms are compared.
  small     --calls calls of --small records of 4 KiB each, compress then decompress per call, run three ways: eager
            with host bytes, eager with the handle, and with the handle captured once in a CUDA graph and replayed.
            Wall time per call is the host clock over all calls up to a final synchronize.  "host_blocked" says
            whether one call, enqueued behind a device sleep (sleep_ms), took more than half the sleep to return.
  seed      in a separate torch.profiler run: the device time of zxc_seed_kernel, the per-call dictionary seeding that
            the handle removes, for 16 384- and 65 535-byte dictionaries (record bytes), over --seed-calls calls of
            zxc_b200_compress_blocks_device on 64 records.
Usage (GPU machine): python profiles/dict_device_bench.py [--records 1048576] [--rounds 5] [--small 64] [--calls 1000]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "profiles"))
sys.path.insert(0, ROOT)
import zxc_corpus as zc  # noqa: E402
import zxc_ctypes as z  # noqa: E402
from compress_batch_bench import card  # noqa: E402
from test_compress_device import opts  # noqa: E402
from test_dict_device_host import bind  # noqa: E402

REC = 4096


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def dopts(d=None):
    o = z.DecompressOpts()
    o._keep = None
    if d is not None:
        o._keep = bytes(d)
        o.dict, o.dict_size = C.cast(C.c_char_p(o._keep), C.c_void_p), len(o._keep)
    return o


class Records:
    """n records of 4 KiB in one arena, their blocks in slots of another, and both calls in both forms"""

    def __init__(self, L, data, n, d, dd):
        self.L, self.n, self.dd = L, n, dd
        self.d_in = torch.from_numpy(data[:n * REC]).cuda()
        stride = (REC + 8 + 68 + 4 + 15) // 16 * 16
        self.arena = torch.empty(n * stride, dtype=torch.uint8, device="cuda")
        self.d_out = torch.empty(n * REC, dtype=torch.uint8, device="cuda")
        idx = torch.arange(n, dtype=torch.int64, device="cuda")
        self.cdesc = torch.stack([self.d_in.data_ptr() + idx * REC, torch.full_like(idx, REC),
                                  self.arena.data_ptr() + idx * stride, torch.full_like(idx, stride)], 1).contiguous()
        self.ddesc = torch.stack([self.arena.data_ptr() + idx * stride, torch.zeros_like(idx),
                                  self.d_out.data_ptr() + idx * REC, torch.full_like(idx, REC)], 1).contiguous()
        self.co, self.cnone, self.do = opts(5, d=d), opts(5), dopts(d)
        total = n * REC
        self.c_ss = {False: int(L.zxc_b200_compress_blocks_device_scratch_size(n, total, REC, C.byref(self.co))),
                     True: int(L.zxc_b200_compress_blocks_device_scratch_size(n, total, REC, C.byref(self.cnone)))}
        self.d_ss = int(L.zxc_b200_decompress_blocks_device_scratch_size(n, REC))
        self.c_scr = torch.empty(max(self.c_ss.values()), dtype=torch.uint8, device="cuda")
        self.d_scr = torch.empty(self.d_ss, dtype=torch.uint8, device="cuda")
        self.cres = torch.empty(n, dtype=torch.int64, device="cuda")
        self.dres = torch.empty(n, dtype=torch.int64, device="cuda")

    def compress(self, handle, st=None):
        L, head = self.L, (self.cdesc.data_ptr(), self.n, C.byref(self.co))
        tail = (self.c_scr.data_ptr(), self.c_ss[handle], self.cres.data_ptr(), st)
        rc = (L.zxc_b200_compress_blocks_device_using_dict(*head, self.dd, *tail) if handle
              else L.zxc_b200_compress_blocks_device(*head, *tail))
        assert rc == 0, rc

    def decompress(self, handle, st=None):
        L, head = self.L, (self.ddesc.data_ptr(), self.n, C.byref(self.do))
        tail = (0, self.d_scr.data_ptr(), self.d_ss, self.dres.data_ptr(), st)
        rc = (L.zxc_b200_decompress_blocks_device_using_dict(*head, self.dd, *tail) if handle
              else L.zxc_b200_decompress_blocks_device(*head, *tail))
        assert rc == 0, rc

    def check(self, handle):
        """one round trip; -> (the blocks, their sizes)"""
        self.compress(handle)
        torch.cuda.synchronize()
        assert bool((self.cres > 0).all())
        self.ddesc[:, 1] = self.cres
        self.d_out.zero_()
        self.decompress(handle)
        torch.cuda.synchronize()
        assert bool((self.dres == REC).all()) and torch.equal(self.d_out, self.d_in)
        return self.arena.clone(), self.cres.clone()


def records_leg(L, data, n, d, dd, rounds):
    R = Records(L, data, n, d, dd)
    a0, s0 = R.check(False)
    a1, s1 = R.check(True)
    assert torch.equal(s0, s1) and torch.equal(a0, a1), "host bytes and handle give different blocks"
    t = {k: [] for k in ("compress_host", "compress_handle", "decompress_host", "decompress_handle")}
    for _ in range(rounds):
        t["compress_host"].append(timed(lambda: R.compress(False)))
        t["compress_handle"].append(timed(lambda: R.compress(True)))
        t["decompress_host"].append(timed(lambda: R.decompress(False)))
        t["decompress_handle"].append(timed(lambda: R.decompress(True)))
    total = n * REC
    out = {k + "_ms": [round(x, 3) for x in v] for k, v in t.items()}
    out.update({k + "_gbps": round(total / statistics.median(v) / 1e6, 2) for k, v in t.items()})
    out["compress_scratch_bytes"] = {"host": R.c_ss[False], "handle": R.c_ss[True]}
    return out


def small_leg(L, data, n, d, dd, calls):
    R = Records(L, data, n, d, dd)
    R.check(False)
    R.check(True)
    out = {}

    def eager(handle):
        def one():
            R.compress(handle)
            R.decompress(handle)
        return one

    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            R.compress(True, s.cuda_stream)
            R.decompress(True, s.cuda_stream)
    torch.cuda.synchronize()
    ways = {"eager_host_bytes": eager(False), "eager_handle": eager(True), "graph_handle": g.replay}
    # how long the sleep of the blocking probe takes on this card
    cycles = 50_000_000
    sleep_ms = timed(lambda: torch.cuda._sleep(cycles))
    for name, fn in ways.items():
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) / calls * 1e3
        torch.cuda._sleep(cycles)
        t1 = time.perf_counter()
        fn()
        enq = (time.perf_counter() - t1) * 1e3
        torch.cuda.synchronize()
        out[name] = {"wall_ms_per_call": round(wall, 4), "enqueue_ms_behind_sleep": round(enq, 3),
                     "host_blocked": enq > 0.5 * sleep_ms}
    out["sleep_ms"] = round(sleep_ms, 2)
    # the graph's last replay wrote the same bytes as the eager calls
    torch.cuda.synchronize()
    assert bool((R.dres == REC).all()) and torch.equal(R.d_out, R.d_in)
    return out


def seed_leg(L, data, d16, d64, calls):
    """device time of zxc_seed_kernel per call, from torch.profiler, for each dictionary size"""
    from torch.profiler import ProfilerActivity, profile
    res = {}
    for name, d in (("16KiB", d16), ("64KiB", d64)):
        R = Records(L, data, 64, d, None)
        R.compress(False)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                R.compress(False)
            torch.cuda.synchronize()
        times = [e.device_time for e in prof.events() if "zxc_seed_kernel" in e.name]
        enc = [e.device_time for e in prof.events() if "zxc_blocks_encode" in e.name]
        res[name] = {"dict_bytes": len(d), "seed_kernels": len(times),
                     "seed_us_mean": round(statistics.mean(times), 2) if times else None,
                     "seed_us_median": round(statistics.median(times), 2) if times else None,
                     "encode_us_median_64x4KiB": round(statistics.median(enc), 2) if enc else None}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1 << 20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--small", type=int, default=64)
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--seed-calls", type=int, default=50)
    ap.add_argument("--legs", default="records,small,seed")
    args = ap.parse_args()
    prod, ref = z.ZxcLib(z.PRODUCT_SO), z.ZxcLib(z.REF_SO)
    L = bind(prod.lib)
    for name, at in (("compress_blocks_device_scratch_size", [C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p]),
                     ("decompress_blocks_device_scratch_size", [C.c_uint32, C.c_uint64])):
        getattr(L, "zxc_b200_" + name).restype = C.c_size_t
        getattr(L, "zxc_b200_" + name).argtypes = at
    data = zc.records(args.records, REC)
    d = zc.train_dict_ref(ref, data, REC)
    # the seeding kernel's time depends on the dictionary's length, not its bytes: record bytes of the two sizes
    d16, d64 = data[:16384].tobytes(), data[:65535].tobytes()
    err = C.c_int(1)
    dd = L.zxc_b200_dict_device_create(d, len(d), None, C.byref(err), None)
    assert dd and err.value == 0, err.value
    out = {"card": card(), "dict_bytes": len(d), "level": 5}
    legs = args.legs.split(",")
    try:
        if "records" in legs:
            out["records"] = {"workload": f"{args.records} x {REC} B records", **records_leg(L, data, args.records, d,
                                                                                          dd, args.rounds)}
        if "small" in legs:
            out["small"] = {"workload": f"{args.calls} calls of {args.small} x {REC} B records, compress + decompress",
                            **small_leg(L, data, args.small, d, dd, args.calls)}
    finally:
        L.zxc_b200_dict_device_free(dd)
    if "seed" in legs:
        out["seed"] = seed_leg(L, data, d16, d64, args.seed_calls)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
