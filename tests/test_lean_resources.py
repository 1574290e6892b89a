"""Register and spill budget of the decode kernel instances (CPU only: needs nvcc, no GPU).

The lean block-decode instances run at their own CTAs per SM (DESIGN.md section 9), which holds only while ptxas keeps
them at or below the register count that occupancy allows and their spill traffic at or below what was measured.  This
compiles zxc_gpu.cu for sm_90a with -Xptxas -v and the Makefile's flags and checks both, and that the general instances
keep their 72 registers.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "zxc_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"

# (registers, spill stores, spill loads) at most, per lean instance: <UNITS, DEFERRED, HAS_DICT, LEAN>
LEAN_BUDGET = {
    "_Z17zxc_decode_kernelILb0ELb0ELb0ELb1EEv12DecodeParams": (72, 0, 0),
    "_Z17zxc_decode_kernelILb0ELb0ELb1ELb1EEv12DecodeParams": (72, 0, 0),
}
GENERAL = [
    "_Z17zxc_decode_kernelILb0ELb0ELb0ELb0EEv12DecodeParams",
    "_Z17zxc_decode_kernelILb0ELb0ELb1ELb0EEv12DecodeParams",
    "_Z17zxc_decode_kernelILb0ELb1ELb0ELb0EEv12DecodeParams",
    "_Z17zxc_decode_kernelILb0ELb1ELb1ELb0EEv12DecodeParams",
]
GENERAL_REGS = 72


@pytest.fixture(scope="module")
def ptxas(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("ptxas")
    cmd = [NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-Xptxas", "-v", "-cubin",
           "-o", str(out / "zxc_gpu.cubin"), os.path.join(CSRC, "zxc_gpu.cu")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    per = {}
    for blk in r.stdout.split("Compiling entry function '")[1:]:
        name = blk.split("'")[0]
        regs = re.search(r"Used (\d+) registers", blk)
        sp = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", blk)
        per[name] = (int(regs.group(1)), int(sp.group(1)), int(sp.group(2)))
    return per


@pytest.mark.parametrize("name", sorted(LEAN_BUDGET))
def test_lean_within_budget(ptxas, name):
    regs, st, ld = ptxas[name]
    max_regs, max_st, max_ld = LEAN_BUDGET[name]
    assert regs <= max_regs, f"{name}: {regs} registers > {max_regs}"
    assert st <= max_st and ld <= max_ld, f"{name}: spills {st} / {ld} B > {max_st} / {max_ld} B"


@pytest.mark.parametrize("name", GENERAL)
def test_general_registers(ptxas, name):
    assert ptxas[name][0] == GENERAL_REGS, (name, ptxas[name])
