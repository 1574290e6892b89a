"""TEST INFRASTRUCTURE: ctypes binding of tests/simt/libzxc_simt_decode.so -- the product's decode DEVICE code compiled
for the CPU on the fiber warp emulator (tests/simt/).  decode_frame() plans a frame with the product's host code
(zxc_b200_plan_frame, no device needed) and runs decode_job() once per block on an emulated warp."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import zxc_ctypes as z

HERE = os.path.dirname(os.path.abspath(__file__))
SIMT_DIR = os.path.join(HERE, "simt")
SIMT_SO = os.environ.get("ZXC_SIMT_SO") or os.path.join(SIMT_DIR, "libzxc_simt_decode.so")  # variant builds: make SO=... EXTRA=-D...


class Job(C.Structure):
    _fields_ = [("src_off", C.c_uint64), ("dst_off", C.c_uint64), ("src_len", C.c_uint32), ("dst_cap", C.c_uint32)]


class Info(C.Structure):
    _fields_ = [("decoded_size", C.c_uint64), ("block_size", C.c_uint32), ("n_blocks", C.c_uint32),
                ("dict_id", C.c_uint32), ("has_checksum", C.c_int), ("seekable", C.c_int), ("global_hash", C.c_uint32)]


def build():
    if os.environ.get("ZXC_SIMT_SO"):
        return
    r = subprocess.run(["make", "-s"], cwd=SIMT_DIR, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(SIMT_SO)
        _lib.simt_decode_blocks.restype = C.c_uint64
        _lib.simt_decode_blocks.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p,
                                            C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_uint64,
                                            C.c_void_p]
    return _lib


def decode_frame(prod, frame, dict=None, dict_huf=None, verify=0, units=0, seed=1, max_blocks=None):
    """(per-block status list, decoded bytes ndarray, oob_writes, rendezvous) for the blocks of `frame`."""
    fb = frame.tobytes() if isinstance(frame, np.ndarray) else bytes(frame)
    prod.lib.zxc_b200_plan_frame.restype = C.c_int64
    prod.lib.zxc_b200_plan_frame.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    info = Info()
    nb = prod.lib.zxc_b200_plan_frame(fb, len(fb), None, 0, C.byref(info))
    assert nb >= 0, nb
    jobs = (Job * max(nb, 1))()
    assert prod.lib.zxc_b200_plan_frame(fb, len(fb), jobs, nb, None) == nb
    if max_blocks is not None:
        nb = min(nb, max_blocks)
    total = int(jobs[nb - 1].dst_off + jobs[nb - 1].dst_cap) if nb else 0
    out = np.zeros(max(total, 1), np.uint8)
    status = (C.c_int32 * max(nb, 1))()
    oob = C.c_int(0)
    src = np.frombuffer(fb, np.uint8)
    d = np.frombuffer(dict, np.uint8) if dict else None
    h = np.frombuffer(dict_huf, np.uint8) if dict_huf else None
    rv = lib().simt_decode_blocks(src.ctypes.data, src.size, out.ctypes.data, total, jobs, nb, status,
                                  d.ctypes.data if d is not None else None, d.size if d is not None else 0,
                                  h.ctypes.data if h is not None else None, max(info.block_size, 4096),
                                  1 if (verify and info.has_checksum) else 0, units, seed, C.byref(oob))
    return list(status)[:nb], out[:total], oob.value, rv


@pytest.fixture(scope="session")
def lean_emu(tmp_path_factory):
    """tests/simt/simt_lean.cc -- the two-launch route: lean instance, then the general one for what it deferred --
    built like tests/simt/Makefile builds the emulator, into a temporary directory"""
    so = str(tmp_path_factory.mktemp("simt_lean") / "libzxc_simt_lean.so")
    root = os.path.dirname(HERE)
    extra = os.environ.get("ZXC_SIMT_EXTRA", "").split()  # the flavour of a variant build (ZXC_SIMT_SO)
    r = subprocess.run(["g++", *extra, "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas",
                        "-Wno-unused-function", "-I.", "-I" + os.path.join(root, "include"),
                        "-I" + os.path.join(root, "zxc_b200", "csrc"), "-o", so, "simt_lean.cc", "simt_rt.cc"],
                       cwd=SIMT_DIR, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    lib = C.CDLL(so)
    lib.simt_decode_two_stage.restype = C.c_uint64
    lib.simt_decode_two_stage.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32,
                                          C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint64,
                                          C.c_void_p]
    return lib


def build_encoder(out_dir):
    """tests/simt/simt_encode.cc -- the encode kernels' source on the fiber warp emulator -- compiled into out_dir"""
    so = os.path.join(str(out_dir), "libzxc_simt_encode.so")
    root = os.path.dirname(HERE)
    extra = os.environ.get("ZXC_SIMT_EXTRA", "").split()  # e.g. -I<dir> ahead of zxc_b200/csrc for a variant encoder
    r = subprocess.run(["g++", *extra, "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas",
                        "-Wno-unused-function", "-I.", "-I" + os.path.join(root, "include"),
                        "-I" + os.path.join(root, "zxc_b200", "csrc"), "-o", so, "simt_encode.cc", "simt_rt.cc"],
                       cwd=SIMT_DIR, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0 and "warning" not in r.stdout, r.stdout[-3000:]
    lib = C.CDLL(so)
    lib.simt_encode.restype = C.c_uint64
    lib.simt_encode.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.c_uint32, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
    lib.simt_enc_staging_stride.restype = C.c_uint32
    lib.simt_enc_staging_stride.argtypes = [C.c_uint32]
    lib.simt_enc_guard_pages.argtypes = [C.c_int]
    return lib


@pytest.fixture(scope="session")
def enc_emu(tmp_path_factory):
    return build_encoder(tmp_path_factory.mktemp("simt_encode"))


def encode_stats(lib):
    """the encode harness's ZXC_STAT / ZXC_LANE_STAT counters (zxc_encode.cuh, zxc_encode_opt.cuh: 64 and up)"""
    return (C.c_uint64 * 128).in_dll(lib, "simt_stat")


class Encoded:
    def __init__(self, blocks, body, rendezvous, stray_slot, stray_scratch):
        self.blocks, self.body, self.rendezvous = blocks, body, rendezvous
        self.stray_slot, self.stray_scratch = stray_slot, stray_scratch


def encode_frame(lib, data, level, block_size, checksum=0, dict=None, dict_huf=None, seed=1):
    """the frame body zxg_encode_body would emit for `data` (one emulated warp per block): an Encoded with the per-block
    bytes, the compacted body, the rendezvous count and the stores found outside the slots / outside the scratch.
    dict_huf is the dictionary's packed 128-byte literal table, unpacked here as zxc_compress does."""
    src = np.ascontiguousarray(np.frombuffer(bytes(data), np.uint8) if not isinstance(data, np.ndarray) else data)
    nb = (src.size + block_size - 1) // block_size
    stride = lib.simt_enc_staging_stride(block_size)
    slots = np.zeros(max(nb * stride, 1), np.uint8)
    sizes = (C.c_uint32 * max(nb, 1))()
    body = np.zeros(max(nb * stride, 1), np.uint8)
    stray = (C.c_uint64 * 2)()
    d = np.frombuffer(bytes(dict), np.uint8) if dict else None
    lens = None
    if dict_huf is not None and any(dict_huf):
        h = np.frombuffer(bytes(dict_huf), np.uint8)
        lens = np.empty(256, np.uint8)
        lens[0::2], lens[1::2] = h & 15, h >> 4
    rv = lib.simt_encode(src.ctypes.data if src.size else None, src.size, block_size, level, checksum,
                         d.ctypes.data if d is not None else None, d.size if d is not None else 0,
                         lens.ctypes.data if lens is not None else None, slots.ctypes.data, sizes, body.ctypes.data, seed,
                         stray)
    blocks = [slots[j * stride:j * stride + sizes[j]].tobytes() for j in range(nb)]
    total = sum(sizes[j] for j in range(nb))
    return Encoded(blocks, body[:total].tobytes(), rv, stray[0], stray[1])


def frame_blocks(frame, checksum):
    """the data blocks of a frame (16-byte file header, then blocks of an 8-byte header -- type in byte 0, payload size
    in bytes 3..6 -- the payload and, with checksums, 4 more bytes) up to the EOF block"""
    fb = bytes(frame)
    cks = checksum
    out, p = [], 16
    while p + 8 <= len(fb) and fb[p] != 255:
        n = 8 + int.from_bytes(fb[p + 3:p + 7], "little") + (4 if cks else 0)
        out.append(fb[p:p + n])
        p += n
    return out
