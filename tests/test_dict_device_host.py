"""Prepared device dictionaries without a device: zxc_b200_dict_device_create's verdicts and the _using_dict
variants' host verdicts, which come in their base calls' order (opts' own dictionary fields are ignored)."""
import ctypes as C

import pytest

from conftest import has_cuda
from test_compress_device import opts

NULL_INPUT, DICT_BIG, NO_DEVICE = -12, -17, -100
FAKE = 1 << 40  # never dereferenced


def bind(L):
    L.zxc_b200_dict_device_create.restype = C.c_void_p
    L.zxc_b200_dict_device_create.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int), C.c_void_p]
    L.zxc_b200_dict_device_id.restype = C.c_uint32
    L.zxc_b200_dict_device_id.argtypes = [C.c_void_p]
    L.zxc_b200_dict_device_size.restype = C.c_size_t
    L.zxc_b200_dict_device_size.argtypes = [C.c_void_p]
    L.zxc_b200_dict_device_free.restype = None
    L.zxc_b200_dict_device_free.argtypes = [C.c_void_p]
    v, p, u32, u64, sz, i = C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_size_t, C.c_int
    sigs = {
        "compress_device": ([p, u64, p, u64, v], [p, sz, p, p, p]),
        "compress_device_batch": ([p, u32, v], [p, sz, p, p]),
        "compress_blocks_device": ([p, u32, v], [p, sz, p, p]),
        "decompress_device": ([p, u64, p, u64, v], [p, sz, p, p]),
        "decompress_inplace_device": ([p, u64, u64, v], [p, sz, p, p]),
        "decompress_device_batch": ([p, u32, v], [p, sz, p, p]),
        "decompress_blocks_device": ([p, u32, v], [i, p, sz, p, p]),
    }
    for name, (head, tail) in sigs.items():
        base, var = getattr(L, "zxc_b200_" + name), getattr(L, f"zxc_b200_{name}_using_dict")
        base.restype = var.restype = C.c_int
        base.argtypes = head + tail
        var.argtypes = head + [p] + tail
    return L


def dopts(d=None):
    import zxc_ctypes as z
    o = z.DecompressOpts(checksum_enabled=1)
    o._keep = None
    if d is not None:
        o._keep = bytes(d)
        o.dict, o.dict_size = C.cast(C.c_char_p(o._keep), C.c_void_p), len(o._keep)
    return o


# every call's argument lists (head, tail) around opts, for a NULL-input case and for one that passes the arguments
CASES = {
    "compress_device": (((FAKE, 100, None, 1000), (FAKE, 1 << 20, FAKE, None, None)),
                        ((FAKE, 100, FAKE, 1000), (FAKE, 1 << 20, FAKE, None, None))),
    "compress_device_batch": (((None, 1), (FAKE, 1 << 20, FAKE, None)), ((FAKE, 1), (FAKE, 1 << 20, FAKE, None))),
    "compress_blocks_device": (((FAKE, 1), (None, 1 << 20, FAKE, None)), ((FAKE, 1), (FAKE, 1 << 20, FAKE, None))),
    "decompress_device": (((None, 100, FAKE, 1000), (FAKE, 1 << 20, FAKE, None)),
                          ((FAKE, 100, FAKE, 1000), (FAKE, 1 << 20, FAKE, None))),
    "decompress_inplace_device": (((FAKE, 100, 10), (FAKE, 1 << 20, FAKE, None)),
                                  ((FAKE, 1000, 100), (FAKE, 1 << 20, FAKE, None))),
    "decompress_device_batch": (((FAKE, 1), (None, 1 << 20, FAKE, None)), ((FAKE, 1), (FAKE, 1 << 20, FAKE, None))),
    "decompress_blocks_device": (((FAKE, 1), (0, FAKE, 1 << 20, None, None)),
                                 ((FAKE, 1), (0, FAKE, 1 << 20, FAKE, None))),
}


@pytest.fixture(scope="module")
def L(prod):
    if has_cuda():
        pytest.skip("only meaningful without a GPU")
    return bind(prod.lib)


def test_create_verdicts_without_a_device(L):
    err = C.c_int(1)
    d = b"0123456789" * 10
    assert L.zxc_b200_dict_device_create(None, 10, None, C.byref(err), None) is None and err.value == NULL_INPUT
    assert L.zxc_b200_dict_device_create(d, 0, None, C.byref(err), None) is None and err.value == NULL_INPUT
    big = b"x" * (65536 + 1)
    assert L.zxc_b200_dict_device_create(big, len(big), None, C.byref(err), None) is None and err.value == DICT_BIG
    assert L.zxc_b200_dict_device_create(None, len(big), None, C.byref(err), None) is None and err.value == NULL_INPUT
    assert L.zxc_b200_dict_device_create(d, len(d), bytes(128), C.byref(err), None) is None and err.value == NO_DEVICE
    assert L.zxc_b200_dict_device_create(d, len(d), None, None, None) is None  # err may be NULL
    assert L.zxc_b200_dict_device_id(None) == 0 and L.zxc_b200_dict_device_size(None) == 0
    L.zxc_b200_dict_device_free(None)


@pytest.mark.parametrize("name", sorted(CASES))
def test_variants_give_the_base_calls_host_verdicts(L, name):
    """dd == NULL: the base call's verdicts without a dictionary, in its order; a dictionary in opts is ignored, so
    where the base call gives DICT_TOO_LARGE the variant goes on to the device check"""
    base, var = getattr(L, "zxc_b200_" + name), getattr(L, f"zxc_b200_{name}_using_dict")
    comp = name.startswith("compress")
    plain = opts(3, 65536) if comp else dopts()
    big = opts(3, 65536, d=b"x" * 70000, h=bytes(128)) if comp else dopts(b"x" * 70000)
    (nh, nt), (ah, at) = CASES[name]
    for o in (None, plain, big):
        ob = C.byref(o) if o is not None else None
        assert var(*nh, ob, None, *nt) == base(*nh, ob, *nt) == NULL_INPUT
    assert base(*ah, C.byref(big), *at) == DICT_BIG
    assert var(*ah, C.byref(big), None, *at) == NO_DEVICE
    for o in (None, plain):
        ob = C.byref(o) if o is not None else None
        assert var(*ah, ob, None, *at) == base(*ah, ob, *at) == NO_DEVICE
