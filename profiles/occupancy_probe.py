"""Occupancy probe of the lean decode kernel: what the eighth CTA per SM gains, and what the carve-out step costs.

Builds library variants with `make NVEXTRA=... OUT=<dir>` and times each on the frame bench.py measures (Silesia-shaped,
64 KiB blocks, level 3, seed 1), decode-only through zxc_b200_decode_blocks, the variants alternated round by round so
that drift on a shared machine lands on all of them alike.  Prints each variant's ptxas numbers for the lean instance,
its GB/s per round, the spread, and the card's name, power limit and SM clock, read in the same run.

    python profiles/occupancy_probe.py                      # builds every variant into a temporary directory
    python profiles/occupancy_probe.py --out DIR            # builds into DIR (reused when already there)
    python profiles/occupancy_probe.py --only parent,cta7   # a subset

Needs oracle/_ref/libzxc_ref.so (to compress the frame) and one GPU for the timing; `--build-only` needs neither.
"""
import argparse
import ctypes as C
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

# The carve-out steps of H100 are 0/8/16/32/64/100/132/164/196/228 KB; a resident
# CTA costs its dynamic shared memory plus 1 KB.  4 warps x 4 KiB rings = 16 KiB: 7 CTAs need 119 KB (132 KB carve-out),
# 8 need 136 KB (164 KB).  2048 bytes of padding take 7 CTAs to 133 KB, past the 132 KB step.  A 57 % carve-out hint
# (130 KB) rounds up to the 132 KB step, where only 7 CTAs of the 64-register build fit.
# A grid of 7 CTAs per SM (ZXC_B200_DECODE_CTAS=7) of a build that could hold 8 leaves the eighth slot empty: the
# block scheduler spreads a grid over the SMs breadth-first, and the persistent CTAs never end before the frame does.
# Each variant's resident CTAs per SM, as the occupancy calculator gives them, are printed beside its timing.
# name, build (a directory per NVEXTRA), NVEXTRA, environment, what it isolates
VARIANTS = [
    ("parent", "parent", "", {}, "shipped: lean at 8 CTAs, 64 registers without spills, look-ahead slot"),
    ("lookahead0", "lookahead0", "-DZXC_LOOKAHEAD=0", {},
     "the lean instances without the look-ahead slot (tokens, offsets, escapes loaded at the batch top)"),
    ("cta7", "cta7", "-DLEAN_CTAS_PER_SM=7u", {}, "the same source built for 7 CTAs (72 registers)"),
    ("grid7", "parent", "", {"ZXC_B200_DECODE_CTAS": "7"},
     "the shipped build with a 7-CTA grid: the eighth CTA alone, at the 164 KB carve-out"),
    ("pad7", "pad7", "-DLEAN_CTAS_PER_SM=7u -DLEAN_SMEM_PAD=2048u", {},
     "7 CTAs, 164 KB carve-out: the L1 shrink alone"),
    ("ring2k_7", "ring2k_7", "-DRING_BYTES=2048u -DLEAN_CTAS_PER_SM=7u", {}, "7 CTAs, 2 KiB rings"),
    ("ring2k_8", "ring2k_8", "-DRING_BYTES=2048u", {}, "8 CTAs, 2 KiB rings: more warps at a 100 KB carve-out"),
]
LEAN = "_Z17zxc_decode_kernelILb0ELb0ELb0ELb1EEv12DecodeParams"


def build(out_dir, nvextra):
    lib = os.path.join(out_dir, "libzxc.so.4")
    if not os.path.exists(lib):
        subprocess.run(["make", "-j", str(os.cpu_count() or 4), f"NVEXTRA={nvextra}", f"OUT={out_dir}"],
                       cwd=os.path.join(ROOT, "zxc_b200", "csrc"), check=True, stdout=subprocess.DEVNULL)
    return lib


def lean_resources(out_dir):
    """(registers, spill stores, spill loads) of the dictionary-free lean instance, from the build's ptxas log"""
    log = open(os.path.join(out_dir, "obj", "ptxas.log")).read()
    blk = log.split(f"Compiling entry function '{LEAN}'")[1].split("Compiling entry function")[0]
    sp = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", blk)
    return int(re.search(r"Used (\d+) registers", blk).group(1)), int(sp.group(1)), int(sp.group(2))


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


class Runner:
    def __init__(self, path, dev, d_src, d_dst, d_jobs, d_status, nb):
        import bench
        import torch

        lib = C.CDLL(path)
        lib.zxc_b200_decode_scratch_size.restype = C.c_size_t
        lib.zxc_b200_decode_scratch_size.argtypes = [C.c_uint32]
        lib.zxc_b200_decode_blocks.restype = C.c_int
        lib.zxc_b200_decode_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                               C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t,
                                               C.c_uint32, C.c_int, C.c_void_p]
        self.lib, self.nb, self.block = lib, nb, bench.BLOCK
        self.bufs = (d_src, d_dst, d_jobs, d_status)
        self.scratch_size = lib.zxc_b200_decode_scratch_size(bench.BLOCK)
        self.d_scratch = torch.empty(self.scratch_size, dtype=torch.uint8, device=dev)
        self.stream = torch.cuda.current_stream(dev)
        lean, general = C.c_int(0), C.c_int(0)
        assert lib.zxc_b200_decode_occupancy(C.byref(lean), C.byref(general)) == 0
        self.occupancy = (lean.value, general.value)

    def step(self):
        d_src, d_dst, d_jobs, d_status = self.bufs
        rc = self.lib.zxc_b200_decode_blocks(d_src.data_ptr(), d_dst.data_ptr(), d_jobs.data_ptr(), self.nb,
                                             d_status.data_ptr(), None, 0, None, self.d_scratch.data_ptr(),
                                             self.scratch_size, self.block, 0, self.stream.cuda_stream)
        assert rc == 0, rc

    def time(self, steps):
        import torch

        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(self.stream)
        for _ in range(steps):
            self.step()
        e1.record(self.stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="build directory (default: a temporary one)")
    ap.add_argument("--only", help="comma-separated variant names")
    ap.add_argument("--gib", type=float, default=4.0, help="decoded GiB of the bench-shaped frame")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20, help="timed decodes per variant and round")
    ap.add_argument("--build-only", action="store_true")
    args = ap.parse_args()

    variants = [v for v in VARIANTS if not args.only or v[0] in args.only.split(",")]
    tmp = None if args.out else tempfile.TemporaryDirectory(prefix="zxc_occ_")
    top = args.out or tmp.name
    libs = {}
    print("| variant | NVEXTRA, environment | lean registers | lean spills (stores / loads) | isolates |")
    print("|---|---|---|---|---|")
    for name, bdir, extra, env, what in variants:
        d = os.path.join(top, bdir)
        libs[name] = build(d, extra)
        if env:  # a copy of its own: the library reads the environment once per load
            libs[name] = os.path.join(d, f"libzxc_{name}.so")
            shutil.copyfile(os.path.join(d, "libzxc.so.4"), libs[name])
        r, s, l_ = lean_resources(d)
        envs = " ".join(f"{k}={v}" for k, v in env.items())
        print(f"| {name} | `{extra}` {envs} | {r} | {s} / {l_} B | {what} |", flush=True)
    if args.build_only:
        return

    import numpy as np
    import torch
    import bench
    import zxc_ctypes as z

    print(f"\ncard (name, power limit, max SM clock, SM clock now): {card()}", flush=True)
    ref = z.ZxcLib(z.REF_SO)
    data, frame, _ = bench.build_shard(ref, args.gib, 0)
    prod = C.CDLL(libs[variants[0][0]])
    prod.zxc_b200_plan_frame.restype = C.c_int64
    prod.zxc_b200_plan_frame.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    nb = prod.zxc_b200_plan_frame(frame.ctypes.data, frame.size, None, 0, None)
    jobs = np.zeros(nb * C.sizeof(bench.Job), dtype=np.uint8)
    assert prod.zxc_b200_plan_frame(frame.ctypes.data, frame.size, jobs.ctypes.data, nb, None) == nb
    dev = torch.device("cuda", 0)
    d_src = torch.from_numpy(frame).to(dev)
    d_dst = torch.empty(data.size, dtype=torch.uint8, device=dev)
    d_jobs = torch.from_numpy(jobs).to(dev)
    d_status = torch.empty(nb, dtype=torch.int32, device=dev)
    want = torch.from_numpy(data).to(dev)
    runners = {}
    for name, _, _, env, _ in variants:
        r = Runner(libs[name], dev, d_src, d_dst, d_jobs, d_status, nb)
        d_dst.zero_()
        os.environ.update(env)
        for _ in range(3):
            r.step()
        torch.cuda.synchronize(dev)
        for k in env:
            del os.environ[k]
        assert torch.equal(d_dst, want), f"{name}: decoded bytes differ"
        runners[name] = r
        print(f"{name}: resident CTAs per SM, lean / general instance: {r.occupancy[0]} / {r.occupancy[1]}", flush=True)
    del want
    rates = {v[0]: [] for v in variants}
    for k in range(args.rounds):
        for name in rates:
            runners[name].time(2)  # re-warm after the previous variant
            ms = runners[name].time(args.steps)
            rates[name].append(data.size / ms / 1e6)
        print(f"round {k + 1}: " + ", ".join(f"{n} {rates[n][-1]:.1f}" for n in rates), flush=True)
        time.sleep(0.5)
    print(f"\ncard after the runs: {card()}")
    base = np.median(rates[variants[0][0]])
    print(f"\n| variant | GB/s decoded, per round | median | spread | against {variants[0][0]} |")
    print("|---|---|---|---|---|")
    for name in rates:
        v = rates[name]
        med = float(np.median(v))
        print(f"| {name} | {' / '.join(f'{x:.1f}' for x in v)} | {med:.1f} | {100 * (max(v) - min(v)) / med:.2f} % | "
              f"{100 * (med / base - 1):+.1f} % |")


if __name__ == "__main__":
    main()
