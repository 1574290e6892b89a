"""The lean block-decode instances run at eight CTAs per SM (CPU only: needs nvcc, no GPU).

Eight CTAs of 128 threads share the SM's 64 K registers only at 64 registers per thread, and the eighth CTA pays off
only without spills (DESIGN.md section 9).  This compiles zxc_gpu.cu for sm_90a with the Makefile's flags and
-Xptxas -v and checks both lean instances at <= 64 registers with no spill stores or loads, and that the source sets
LEAN_CTAS_PER_SM to 8, the launch bound that makes ptxas hold that budget.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "zxc_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
         "-I" + os.path.join(ROOT, "include"), "-I" + CSRC]

LEAN = [
    "_Z17zxc_decode_kernelILb0ELb0ELb0ELb1EEv12DecodeParams",
    "_Z17zxc_decode_kernelILb0ELb0ELb1ELb1EEv12DecodeParams",
]
LEAN_REGS = 64  # 65536 registers / (8 CTAs x 128 threads)


@pytest.fixture(scope="module")
def nvcc():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not found")
    return NVCC


@pytest.fixture(scope="module")
def ptxas(nvcc, tmp_path_factory):
    out = tmp_path_factory.mktemp("ptxas")
    cmd = [nvcc] + FLAGS + ["-Xptxas", "-v", "-cubin", "-o", str(out / "zxc_gpu.cubin"), os.path.join(CSRC, "zxc_gpu.cu")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    per = {}
    for blk in r.stdout.split("Compiling entry function '")[1:]:
        name = blk.split("'")[0]
        regs = re.search(r"Used (\d+) registers", blk)
        sp = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", blk)
        per[name] = (int(regs.group(1)), int(sp.group(1)), int(sp.group(2)))
    return per


@pytest.mark.parametrize("name", LEAN)
def test_lean_fits_eight_ctas_without_spills(ptxas, name):
    regs, st, ld = ptxas[name]
    assert regs <= LEAN_REGS, f"{name}: {regs} registers > {LEAN_REGS}"
    assert (st, ld) == (0, 0), f"{name}: spills {st} / {ld} B"


def test_lean_ctas_per_sm_is_eight(nvcc, tmp_path):
    probe = tmp_path / "probe.cu"
    probe.write_text('#include "zxc_decode.cuh"\nlean_ctas_per_sm = LEAN_CTAS_PER_SM;\n')
    r = subprocess.run([nvcc] + FLAGS + ["-E", "-x", "cu", str(probe)], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    m = re.search(r"lean_ctas_per_sm = (.*?);", r.stdout)
    assert m and m.group(1).strip() == "8u", m.group(1) if m else r.stdout[-2000:]
