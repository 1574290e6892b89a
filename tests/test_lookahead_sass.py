"""The look-ahead slot touches the dictionary-free lean block-decode instance only (CPU only: nvcc, cuobjdump, no GPU).

The lean instance without a dictionary stages the next batch's tokens, offsets and escape values into shared memory
with cp.async (zxc_decode.cuh, ZXC_LOOKAHEAD; DESIGN.md section 3a step 8).  This compiles zxc_gpu.cu for sm_90a with the Makefile's
flags twice, as shipped and with -DZXC_LOOKAHEAD=0, and checks with cuobjdump -sass, function by function, that every
kernel other than that one is the same in both (the dictionary lean instance measured slower with the slot and does not
carry it), and that the shipped instance carries the copies (LDGSTS) and their wait while the ZXC_LOOKAHEAD=0 one does
not.
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
LEAN = "_Z17zxc_decode_kernelILb0ELb0ELb0ELb1EEv12DecodeParams"
LEAN_DICT = "_Z17zxc_decode_kernelILb0ELb0ELb1ELb1EEv12DecodeParams"


def sass_per_function(cubin):
    cuobjdump = os.path.join(os.path.dirname(os.path.realpath(NVCC)), "cuobjdump")
    out = subprocess.run([cuobjdump, "-sass", cubin], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout[-2000:]
    per = {}
    for blk in re.split(r"\n\s*Function : ", out.stdout)[1:]:
        name, body = blk.split("\n", 1)
        per[name.strip()] = body
    return per


@pytest.fixture(scope="module")
def builds(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("lookahead")
    procs = {}
    for tag, extra in (("on", []), ("off", ["-DZXC_LOOKAHEAD=0"])):
        cmd = [NVCC] + FLAGS + extra + ["-cubin", "-o", str(out / f"{tag}.cubin"), os.path.join(CSRC, "zxc_gpu.cu")]
        procs[tag] = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    for tag, p in procs.items():
        log = p.communicate()[0]
        assert p.returncode == 0, log[-4000:]
    return {tag: sass_per_function(str(out / f"{tag}.cubin")) for tag in procs}


def test_other_kernels_unchanged(builds):
    on, off = builds["on"], builds["off"]
    assert set(on) == set(off)
    assert {LEAN, LEAN_DICT} <= set(on)
    changed = sorted(n for n in on if n != LEAN and on[n] != off[n])
    assert not changed, changed


def test_lean_instance_stages_with_cp_async(builds):
    on, off = builds["on"][LEAN], builds["off"][LEAN]
    assert "LDGSTS" in on and "LDGDEPBAR" in on
    assert "LDGSTS" not in off
