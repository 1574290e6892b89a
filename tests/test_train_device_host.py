"""Dictionary trainers on samples in HBM (zxc_b200_train_dict_device, zxc_b200_train_dict_huf_device,
zxc_b200_dict_train_device): the verdicts that need no device.

Every argument case of test_train_gpu's verdict table gives the device twins the code the host trainers give, and the
reference's where it is built: all of them come before any sample byte is read, so the table's host pointers stand in
for device pointers.  Without a device, a valid call gives ZXC_B200_ERROR_NO_DEVICE."""
import ctypes as C

import numpy as np
import pytest

import test_train_gpu as T
import zxc_corpus as zc
import zxc_ctypes as z
from conftest import has_cuda


def bind_device(lib):
    L = lib.lib
    L.zxc_b200_train_dict_device.restype = C.c_int64
    L.zxc_b200_train_dict_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    L.zxc_b200_train_dict_huf_device.restype = C.c_int
    L.zxc_b200_train_dict_huf_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                                 C.c_void_p, C.c_void_p]
    L.zxc_b200_dict_train_device.restype = C.c_int64
    L.zxc_b200_dict_train_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    return L


class Twins:
    """the device twins under the host trainers' names, on the legacy default stream (or `stream`), so that calls
    written for the host trainers run unchanged against them"""

    def __init__(self, lib, stream=None):
        L = bind_device(lib)
        self.zxc_train_dict = lambda *a: L.zxc_b200_train_dict_device(*a, stream)
        self.zxc_train_dict_huf = lambda *a: L.zxc_b200_train_dict_huf_device(*a, stream)
        self.zxc_dict_train = lambda *a: L.zxc_b200_dict_train_device(*a, stream)


@pytest.fixture(scope="module")
def twins(prod):
    return Twins(prod)


@pytest.mark.parametrize("name", [n for n, _ in T.VERDICTS])
def test_verdicts_match_host_trainers(prod, twins, name):
    call = dict(T.VERDICTS)[name]
    want = call(T.bind(prod))
    assert want < 0, (name, want)
    assert call(twins) == want, (name, z.ERR.get(want))


@pytest.mark.parametrize("name", [n for n, _ in T.VERDICTS])
def test_verdicts_match_reference(ref, twins, name):
    call = dict(T.VERDICTS)[name]
    want = call(T.bind(ref))
    assert call(twins) == want, (name, z.ERR.get(want))


def test_valid_call_without_device_reports_no_device(twins):
    if has_cuda():
        pytest.skip("a CUDA device is present")
    s = T.Samples.one(zc.gen_text(20000))
    assert T.train_content(twins, s, 4096)[0] == -100
    assert T.train_table(twins, s, b"some dictionary bytes")[0] == -100
    assert T.train_zxd(twins, s)[0] == -100
    # NULL samples of non-zero size pass the checks too (the content trainer reads them as zeros)
    n = T.Samples(np.zeros(1, np.uint8), [None, None])
    n.sizes[0] = n.sizes[1] = 1000
    assert T.train_content(twins, n, 64)[0] == -100
