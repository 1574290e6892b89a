"""Phase trace of the lean decode kernel on the bench-shaped frame.

A library built with -DZXC_TRACE=1 has lane 0 of every warp add clock64() deltas per phase of the sequence-centric
body (zxc_decode.cuh, TR_*) to a per-warp row in device memory.  This script decodes the frame that bench.py
measures (Silesia-shaped, 64 KiB blocks, level 3, seed 1) through each traced library given, and prints the mean SM
cycles a warp spends per batch in each phase, the per-block costs, and where the matches read from.

    python profiles/trace_decode.py                       # builds a traced library into a temporary directory
    python profiles/trace_decode.py --lib A.so --lib B.so # compares prebuilt traced libraries on one frame

Needs oracle/_ref/libzxc_ref.so (to compress the frame) and one GPU.  The numbers are warp-time: a warp shares its
SM sub-partition with six others, so a phase's cycles include the time it waited for issue slots.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

SLOTS = 16
ROWS = 8192
PHASES = ["unpack", "escapes+scans+validation", "literal pass", "free-match pass", "sequence-order tail", "flush"]
PER_BLOCK = [(6, "block start (sections, extras scan)"), (7, "block end (trailing literals)"), (9, "job claim"),
             (8, "giant sequences")]
TR_BATCHES, TR_BLOCKS, TR_M_RING, TR_M_GLOBAL, TR_M_DICT, TR_M_SEQ = 10, 11, 12, 13, 14, 15


def build_traced(out_dir):
    subprocess.run(["make", "-j", str(os.cpu_count() or 4), "NVEXTRA=-DZXC_TRACE=1", f"OUT={out_dir}"],
                   cwd=os.path.join(ROOT, "zxc_b200", "csrc"), check=True, stdout=subprocess.DEVNULL)
    return os.path.join(out_dir, "libzxc.so.4")


def trace_one(path, data, frame, reps):
    import torch
    import bench

    lib = C.CDLL(path)
    lib.zxc_b200_plan_frame.restype = C.c_int64
    lib.zxc_b200_plan_frame.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.zxc_b200_decode_scratch_size.restype = C.c_size_t
    lib.zxc_b200_decode_scratch_size.argtypes = [C.c_uint32]
    lib.zxc_b200_decode_blocks.restype = C.c_int
    lib.zxc_b200_decode_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                           C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_int,
                                           C.c_void_p]
    if not hasattr(lib, "zxc_b200_trace_read"):
        raise SystemExit(f"{path}: not a traced build (make NVEXTRA=-DZXC_TRACE=1 OUT=<dir>)")
    lib.zxc_b200_trace_read.restype = C.c_int
    lib.zxc_b200_trace_read.argtypes = [C.c_void_p]

    dev = torch.device("cuda", 0)
    nb = lib.zxc_b200_plan_frame(frame.ctypes.data, frame.size, None, 0, None)
    jobs = np.zeros(nb * C.sizeof(bench.Job), dtype=np.uint8)
    assert lib.zxc_b200_plan_frame(frame.ctypes.data, frame.size, jobs.ctypes.data, nb, None) == nb
    d_src = torch.from_numpy(frame).to(dev)
    d_dst = torch.empty(data.size, dtype=torch.uint8, device=dev)
    d_jobs = torch.from_numpy(jobs).to(dev)
    d_status = torch.empty(nb, dtype=torch.int32, device=dev)
    scratch_size = lib.zxc_b200_decode_scratch_size(bench.BLOCK)
    d_scratch = torch.empty(scratch_size, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev)
    acc = np.zeros(ROWS * SLOTS, dtype=np.uint64)

    def step():
        rc = lib.zxc_b200_decode_blocks(d_src.data_ptr(), d_dst.data_ptr(), d_jobs.data_ptr(), nb,
                                        d_status.data_ptr(), None, 0, None, d_scratch.data_ptr(), scratch_size,
                                        bench.BLOCK, 0, stream.cuda_stream)
        assert rc == 0, rc

    step()
    assert lib.zxc_b200_trace_read(acc.ctypes.data) > 0  # drop the first launch's counts
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(reps):
        step()
    ev1.record(stream)
    torch.cuda.synchronize(dev)
    ms = ev0.elapsed_time(ev1) / reps
    assert lib.zxc_b200_trace_read(acc.ctypes.data) > 0
    assert np.array_equal(d_dst.cpu().numpy(), data), "traced build decoded different bytes"
    rows = acc.reshape(ROWS, SLOTS)
    active = rows[rows[:, TR_BLOCKS] > 0]
    return active.sum(axis=0).astype(np.float64), len(active), ms


def report(name, tot, warps, ms, n_bytes):
    batches, blocks = tot[TR_BATCHES], tot[TR_BLOCKS]
    per_batch = [tot[k] / batches for k in range(len(PHASES))]
    print(f"\n## {name}")
    print(f"{warps} warps, {int(blocks)} blocks, {int(batches)} batches ({batches / blocks:.1f} per block); "
          f"traced decode {ms:.2f} ms = {n_bytes / ms / 1e6:.1f} GB/s (the trace itself costs time)")
    print("\n| phase | cycles per batch | share |")
    print("|---|---|---|")
    whole = sum(tot[k] for k in range(10))
    for k, p in enumerate(PHASES):
        print(f"| {p} | {per_batch[k]:.0f} | {100 * tot[k] / whole:.1f} % |")
    print(f"| **batch total** | **{sum(per_batch):.0f}** | {100 * sum(tot[:6]) / whole:.1f} % |")
    for k, p in PER_BLOCK:
        print(f"| {p}, per block | {tot[k] / blocks:.0f} | {100 * tot[k] / whole:.1f} % |")
    print(f"\nmatches per batch: ring {tot[TR_M_RING] / batches:.2f}, global {tot[TR_M_GLOBAL] / batches:.2f}, "
          f"dictionary {tot[TR_M_DICT] / batches:.2f}; in the sequence-order tail {tot[TR_M_SEQ] / batches:.2f}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", help="traced libzxc.so.4 (repeatable); default: build one")
    ap.add_argument("--gib", type=float, default=1.0, help="decoded GiB of the bench-shaped frame")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()

    import bench
    import zxc_ctypes as z

    libs = args.lib
    tmp = None
    if not libs:
        tmp = tempfile.TemporaryDirectory(prefix="zxc_trace_")
        libs = [build_traced(tmp.name)]
    ref = z.ZxcLib(z.REF_SO)
    data, frame, _ = bench.build_shard(ref, args.gib, 0)
    for path in libs:
        tot, warps, ms = trace_one(path, data, frame, args.reps)
        report(path, tot, warps, ms, data.size)


if __name__ == "__main__":
    main()
