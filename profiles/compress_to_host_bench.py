"""zxc_b200_compress_device_to_host against zxc_b200_compress_device + a pinned device-to-host copy of its frame.

Inputs are silesia-shaped (tests/zxc_corpus.py), 1 GiB and 4 GiB, 64 KiB blocks, levels 1 and 3, seekable, with
windows of 64 MiB, 256 MiB and 1 GiB.  Call times are CUDA events around one call (median of --reps after a
warm-up call).  The HBM each path needs comes from the size queries: the scratch for this call, the output plus the
scratch for the device path.  Every frame is checked against the device path's.  A separate torch.profiler run gives
the writer kernel's time per call and the share of the call each kernel takes, and a pinned device-to-host copy of the
same byte count gives the copy engine's rate.  The card's name, power limit and SM clock are read in the same run.
Prints one JSON line per row; --out FILE also writes the whole result there."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import zxc_corpus as zc  # noqa: E402
from zxc_b200 import device as D  # noqa: E402

lib = D.lib
BS = 65536
MiB = 1 << 20


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "not read"


def events_ms(fn, reps):
    fn()  # warm-up
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,4", help="input sizes in GiB")
    ap.add_argument("--levels", default="1,3")
    ap.add_argument("--windows", default="64,256,1024", help="windows in MiB")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    a = ap.parse_args()
    info = {"card": card(), "rows": []}
    print(info["card"], flush=True)
    st = torch.cuda.current_stream()
    for gib in [int(x) for x in a.sizes.split(",")]:
        n = gib << 30
        x = torch.from_numpy(zc.silesia_shaped(n, seed=7)).cuda()
        cap = int(lib.zxc_compress_bound(n))
        pinned = torch.empty(cap, dtype=torch.uint8, pin_memory=True)
        for level in [int(v) for v in a.levels.split(",")]:
            o = D._Opts(level=level, block_size=BS, checksum_enabled=0, seekable=1)
            # the device path: compress into HBM, then one pinned copy of the frame
            ss_dev = int(lib.zxc_b200_encode_scratch_size(n, C.byref(o)))
            dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
            scr = torch.empty(ss_dev, dtype=torch.uint8, device="cuda")
            res = torch.zeros(1, dtype=torch.int64, device="cuda")

            def dev_compress():
                assert lib.zxc_b200_compress_device(x.data_ptr(), n, dst.data_ptr(), cap, C.byref(o), scr.data_ptr(),
                                                    ss_dev, res.data_ptr(), None, st.cuda_stream) == 0

            dev_compress()
            torch.cuda.synchronize()
            size = int(res.item())
            assert size > 0
            want = dst[:size].cpu().numpy()

            def dev_path():
                dev_compress()
                pinned[:size].copy_(dst[:size], non_blocking=True)

            t_dev = events_ms(dev_path, a.reps)
            t_enc = events_ms(dev_compress, a.reps)
            t_d2h = events_ms(lambda: pinned[:size].copy_(dst[:size], non_blocking=True), a.reps)
            del dst, scr
            torch.cuda.empty_cache()
            row = {"gib": gib, "level": level, "frame": size, "dev_path_ms": t_dev, "dev_compress_ms": t_enc,
                   "d2h_copy_ms": t_d2h, "d2h_copy_gbs": size / t_d2h[0] / 1e6,
                   "dev_path_hbm": cap + ss_dev, "windows": []}
            for wm in [int(v) for v in a.windows.split(",")]:
                w = wm * MiB
                ss = int(lib.zxc_b200_compress_device_to_host_scratch_size(n, w, C.byref(o)))
                scr = torch.empty(ss, dtype=torch.uint8, device="cuda")
                out = torch.empty(cap, dtype=torch.uint8, pin_memory=True)

                def c2h():
                    assert lib.zxc_b200_compress_device_to_host(x.data_ptr(), n, out.data_ptr(), cap, C.byref(o), w,
                                                                scr.data_ptr(), ss, res.data_ptr(),
                                                                st.cuda_stream) == 0

                c2h()
                torch.cuda.synchronize()
                ok = int(res.item()) == size and np.array_equal(out[:size].numpy(), want)
                t = events_ms(c2h, a.reps)
                row["windows"].append({"window_mib": wm, "scratch": ss, "call_ms": t, "same_frame": ok})
                print(gib, level, wm, size, t, ok, flush=True)
                del scr, out
                torch.cuda.empty_cache()
            info["rows"].append(row)
            print(json.dumps(row), flush=True)
        del x
        torch.cuda.empty_cache()
    # the kernels of one call, in a separate profiled run (256 MiB window)
    from torch.profiler import ProfilerActivity, profile
    prof_rows = []
    for gib in [int(x) for x in a.sizes.split(",")]:
        n = gib << 30
        x = torch.from_numpy(zc.silesia_shaped(n, seed=7)).cuda()
        cap = int(lib.zxc_compress_bound(n))
        out = torch.empty(cap, dtype=torch.uint8, pin_memory=True)
        for level in [int(v) for v in a.levels.split(",")]:
            o = D._Opts(level=level, block_size=BS, checksum_enabled=0, seekable=1)
            w = 256 * MiB
            ss = int(lib.zxc_b200_compress_device_to_host_scratch_size(n, w, C.byref(o)))
            scr = torch.empty(ss, dtype=torch.uint8, device="cuda")
            res = torch.zeros(1, dtype=torch.int64, device="cuda")

            def c2h():
                assert lib.zxc_b200_compress_device_to_host(x.data_ptr(), n, out.data_ptr(), cap, C.byref(o), w,
                                                            scr.data_ptr(), ss, res.data_ptr(),
                                                            st.cuda_stream) == 0

            c2h()
            torch.cuda.synchronize()
            size = int(res.item())
            calls = 3
            with profile(activities=[ProfilerActivity.CUDA]) as p:
                for _ in range(calls):
                    c2h()
                torch.cuda.synchronize()
            k = {}
            for e in p.key_averages():
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                if t:
                    k[e.key] = k.get(e.key, 0) + t / calls / 1e3
            total = sum(v for kk, v in k.items() if "zxc_" in kk or "Memcpy" in kk or "Memset" in kk)
            wr = sum(v for kk, v in k.items() if "zxc_c2h_write" in kk)
            d2h = torch.empty(size, dtype=torch.uint8, device="cuda")
            t_ce = events_ms(lambda: out[:size].copy_(d2h, non_blocking=True), 5)
            pr = {"gib": gib, "level": level, "frame": size, "kernels_ms": k, "writer_ms": wr,
                  "writer_gbs": size / wr / 1e6 if wr else None, "writer_share": wr / total if total else None,
                  "copy_engine_ms": t_ce, "copy_engine_gbs": size / t_ce[0] / 1e6}
            prof_rows.append(pr)
            print(json.dumps(pr), flush=True)
            del scr, d2h
        del x, out
        torch.cuda.empty_cache()
    info["profile"] = prof_rows
    info["card_after"] = card()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(info, f, indent=1)
        print("wrote", a.out)


if __name__ == "__main__":
    main()
