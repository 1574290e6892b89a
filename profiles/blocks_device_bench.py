"""The block API in HBM on BASELINE.json configs[3]'s shape: 1 Mi records of 4 KiB, a 16 KiB dictionary from the
reference's trainer, level 5.

Two forms of the same records:
  blocks   zxc_b200_compress_blocks_device into one frameless block per record (each in its own slot of one arena),
           and zxc_b200_decompress_blocks_device of those blocks back into the records
  frame    the records as one seekable frame with 4 KiB blocks (this library's zxc_compress), decoded from HBM with
           zxc_b200_decode_blocks and its job table, timed as bench.py's dict leg times it
Per round, each call runs once between CUDA events on one stream, the forms alternating; every shape is warmed
first.  Rates: compress GB/s of input bytes, decompress GB/s of decoded bytes, medians over --rounds.  Also printed:
compressed bytes of both forms, launches per call, scratch bytes, and the card's name, power limit and SM clocks,
read in the same run.
Usage (GPU machine): python profiles/blocks_device_bench.py [--records 1048576] [--rounds 5]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "profiles"))
sys.path.insert(0, ROOT)
import zxc_corpus as zc  # noqa: E402
import zxc_ctypes as z  # noqa: E402
from compress_batch_bench import card  # noqa: E402
from test_blocks_device import bind, dopts  # noqa: E402
from test_compress_device import opts  # noqa: E402

REC = 4096


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1 << 20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    n = args.records
    prod, ref = z.ZxcLib(z.PRODUCT_SO), z.ZxcLib(z.REF_SO)
    L = bind(prod.lib)
    L.zxc_b200_plan_frame.restype = C.c_int64
    L.zxc_b200_plan_frame.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    L.zxc_b200_decode_scratch_size.restype = C.c_size_t
    L.zxc_b200_decode_scratch_size.argtypes = [C.c_uint32]
    L.zxc_b200_decode_blocks.restype = C.c_int
    L.zxc_b200_decode_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                         C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_int,
                                         C.c_void_p]
    L.zxc_b200_reduce_status.restype = C.c_int64
    L.zxc_b200_reduce_status.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    data = zc.records(n, REC)
    d = zc.train_dict_ref(ref, data, REC)
    total = data.size
    d_in = torch.from_numpy(data).cuda()
    stride = (REC + 8 + 68 + 4 + 15) // 16 * 16  # zxc_compress_block_bound, 16-byte aligned slots
    arena = torch.empty(n * stride, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(total, dtype=torch.uint8, device="cuda")
    idx = torch.arange(n, dtype=torch.int64, device="cuda")
    cdesc = torch.stack([d_in.data_ptr() + idx * REC, torch.full_like(idx, REC), arena.data_ptr() + idx * stride,
                         torch.full_like(idx, stride)], 1).contiguous()
    ddesc = torch.stack([arena.data_ptr() + idx * stride, torch.zeros_like(idx), d_out.data_ptr() + idx * REC,
                         torch.full_like(idx, REC)], 1).contiguous()
    co, do = opts(5, d=d), dopts(0, d)
    c_ss = int(L.zxc_b200_compress_blocks_device_scratch_size(n, total, REC, C.byref(co)))
    d_ss = int(L.zxc_b200_decompress_blocks_device_scratch_size(n, REC))
    c_scr = torch.empty(c_ss, dtype=torch.uint8, device="cuda")
    d_scr = torch.empty(d_ss, dtype=torch.uint8, device="cuda")
    cres = torch.empty(n, dtype=torch.int64, device="cuda")
    dres = torch.empty(n, dtype=torch.int64, device="cuda")
    launches = {}

    def compress():
        c0 = L.zxc_b200_launch_count()
        assert L.zxc_b200_compress_blocks_device(cdesc.data_ptr(), n, C.byref(co), c_scr.data_ptr(), c_ss,
                                                 cres.data_ptr(), None) == 0
        launches["compress"] = L.zxc_b200_launch_count() - c0

    def decompress():
        c0 = L.zxc_b200_launch_count()
        assert L.zxc_b200_decompress_blocks_device(ddesc.data_ptr(), n, C.byref(do), 0, d_scr.data_ptr(), d_ss,
                                                   dres.data_ptr(), None) == 0
        launches["decompress"] = L.zxc_b200_launch_count() - c0

    compress()
    torch.cuda.synchronize()
    assert bool((cres > 0).all()), "a record failed to compress"
    ddesc[:, 1] = cres
    decompress()
    torch.cuda.synchronize()
    assert bool((dres == REC).all()) and torch.equal(d_out, d_in), "blocks: decoded records differ"
    block_bytes = int(cres.sum().item())
    # a sample of blocks against this library's host zxc_compress_block
    for i in range(0, n, max(1, n // 16)):
        cc = prod.lib.zxc_create_cctx(None)
        buf = np.zeros(stride, np.uint8)
        src = np.ascontiguousarray(data[i * REC:(i + 1) * REC])
        r = prod.lib.zxc_compress_block(cc, src.ctypes.data, REC, buf.ctypes.data, stride, C.byref(co))
        prod.lib.zxc_free_cctx(cc)
        got = arena[i * stride:i * stride + r].cpu().numpy()
        assert r == int(cres[i].item()) and np.array_equal(got, buf[:r]), ("sampled block", i)

    # the frame form
    frame = prod.compress(data, level=5, block_size=REC, seekable=1, dict=d)
    assert not isinstance(frame, int), frame
    nb = L.zxc_b200_plan_frame(frame.ctypes.data, frame.size, None, 0, None)
    jobs = np.zeros(nb * 24, dtype=np.uint8)
    assert L.zxc_b200_plan_frame(frame.ctypes.data, frame.size, jobs.ctypes.data, nb, None) == nb == n
    f_src = torch.from_numpy(frame).cuda()
    f_jobs = torch.from_numpy(jobs).cuda()
    f_status = torch.empty(nb, dtype=torch.int32, device="cuda")
    f_dict = torch.from_numpy(np.frombuffer(d, np.uint8).copy()).cuda()
    f_ss = int(L.zxc_b200_decode_scratch_size(REC))
    f_scr = torch.empty(f_ss, dtype=torch.uint8, device="cuda")

    def frame_decode():
        c0 = L.zxc_b200_launch_count()
        assert L.zxc_b200_decode_blocks(f_src.data_ptr(), d_out.data_ptr(), f_jobs.data_ptr(), nb, f_status.data_ptr(),
                                        f_dict.data_ptr(), len(d), None, f_scr.data_ptr(), f_ss, REC, 0, None) == 0
        launches["frame_decode"] = L.zxc_b200_launch_count() - c0

    d_out.zero_()
    frame_decode()
    torch.cuda.synchronize()
    assert L.zxc_b200_reduce_status(f_status.data_ptr(), f_jobs.data_ptr(), nb, None) == total
    assert torch.equal(d_out, d_in), "frame: decoded records differ"

    t = {"compress": [], "decompress": [], "frame_decode": []}
    for _ in range(args.rounds):
        t["compress"].append(timed(compress))
        t["decompress"].append(timed(decompress))
        t["frame_decode"].append(timed(frame_decode))
    assert bool((dres == REC).all())
    med = {k: statistics.median(v) for k, v in t.items()}
    print(json.dumps({
        "card": card(),
        "workload": f"{n} x {REC} B records (zxc_corpus.records), {len(d)} B dictionary (reference trainer), level 5",
        "blocks": {"compress_gbps": round(total / med["compress"] / 1e6, 2),
                   "decompress_gbps": round(total / med["decompress"] / 1e6, 2),
                   "compress_ms": [round(x, 3) for x in t["compress"]],
                   "decompress_ms": [round(x, 3) for x in t["decompress"]],
                   "compressed_bytes": block_bytes, "compress_scratch_bytes": c_ss,
                   "decompress_scratch_bytes": d_ss},
        "frame": {"decode_gbps": round(total / med["frame_decode"] / 1e6, 2),
                  "decode_ms": [round(x, 3) for x in t["frame_decode"]], "compressed_bytes": int(frame.size),
                  "decode_scratch_bytes": f_ss},
        "launches_per_call": launches,
    }, indent=1))


if __name__ == "__main__":
    main()
