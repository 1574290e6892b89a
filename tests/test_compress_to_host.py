"""zxc_b200_compress_device_to_host: a device buffer compressed into a frame in page-locked host memory, one window
of input per round.

Every frame is compared byte for byte with zxc_compress of a host copy (and with the reference where it is built),
whatever the window; host memory around the room is checked against canaries; the frames are decoded back with
zxc_b200_seekable_device_open_host and with load_frame."""
import ctypes as C

import numpy as np
import pytest

import zxc_corpus as zc
import zxc_ctypes as z
from conftest import has_cuda
from test_compress_device import MEMORY, NO_DEVICE, NULL_INPUT, DST_TOO_SMALL, CORRUPT, BAD_BS, DICT_BIG, opts
from test_oracle import golden_dicts, make_case

UNSUPPORTED = -102
HDR, EOF, FOOT, SEK_HDR = 16, 8, 12, 8


def bind(L):
    L.zxc_compress_bound.restype = C.c_uint64
    L.zxc_compress_bound.argtypes = [C.c_size_t]
    L.zxc_b200_compress_device_to_host_scratch_size.restype = C.c_size_t
    L.zxc_b200_compress_device_to_host_scratch_size.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p]
    L.zxc_b200_compress_device_to_host.restype = C.c_int
    L.zxc_b200_compress_device_to_host.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p,
                                                   C.c_uint64, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.zxc_b200_compress_device_to_host_using_dict.restype = C.c_int
    L.zxc_b200_compress_device_to_host_using_dict.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64,
                                                              C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                                              C.c_size_t, C.c_void_p, C.c_void_p]
    L.zxc_b200_launch_count.restype = C.c_uint64
    return L


def test_without_a_device(prod):
    """Without a device: the argument verdicts in their order, then NO_DEVICE; the size query gives 0"""
    if has_cuda():
        pytest.skip("only meaningful without a GPU")
    L = bind(prod.lib)
    fake = 1 << 40  # never dereferenced: every verdict here is decided before memory is touched
    c = L.zxc_b200_compress_device_to_host
    assert c(fake, 100, None, 1000, None, 0, fake, 1 << 20, fake, None) == NULL_INPUT
    assert c(fake, 100, fake, 0, None, 0, fake, 1 << 20, fake, None) == NULL_INPUT
    assert c(None, 100, fake, 1000, None, 0, fake, 1 << 20, fake, None) == NULL_INPUT
    assert c(fake, 100, fake, 1000, None, 0, None, 1 << 20, fake, None) == NULL_INPUT
    assert c(fake, 100, fake, 1000, None, 0, fake, 1 << 20, None, None) == NULL_INPUT
    big = opts(3, 3000, d=b"x" * 70000)
    assert c(fake, 100, fake, 1000, C.byref(big), 0, fake, 1 << 20, fake, None) == DICT_BIG
    assert c(fake, 100, fake, 1000, C.byref(opts(3, 3000)), 0, fake, 1 << 20, fake, None) == BAD_BS
    assert c(fake, 100, fake, 1000, C.byref(opts(3, 65536)), 0, fake, 1 << 20, fake, None) == NO_DEVICE
    assert L.zxc_b200_compress_device_to_host_using_dict(fake, 100, fake, 1000, None, None, 0, fake, 1 << 20, fake,
                                                         None) == NO_DEVICE
    assert L.zxc_b200_compress_device_to_host_scratch_size(1 << 20, 1 << 18, None) == 0
    assert L.zxc_b200_compress_device_to_host_scratch_size(1 << 20, 1 << 18, C.byref(opts(6, 65536, seek=1))) == 0


def test_python_argument_checks():
    """compress_to_host takes a CUDA src only, and `out` only as a pinned contiguous uint8 CPU tensor"""
    import torch
    from zxc_b200 import device
    with pytest.raises(ValueError, match="CUDA"):
        device.compress_to_host(torch.zeros(100, dtype=torch.uint8))
    if torch.cuda.is_available():
        src = torch.zeros(100, dtype=torch.uint8, device="cuda")
        for bad in (torch.zeros(1000, dtype=torch.uint8), torch.zeros(1000, dtype=torch.int32).pin_memory(),
                    torch.zeros((100, 20), dtype=torch.uint8).pin_memory()[:, 0],
                    torch.zeros(1000, dtype=torch.uint8, device="cuda")):
            with pytest.raises(ValueError, match="pinned"):
                device.compress_to_host(src, out=bad)


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
def _cudart():
    rt = C.CDLL("libcudart.so.12")
    rt.cudaHostAlloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t, C.c_uint]
    rt.cudaFreeHost.argtypes = [C.c_void_p]
    rt.cudaHostRegister.argtypes = [C.c_void_p, C.c_size_t, C.c_uint]
    rt.cudaHostUnregister.argtypes = [C.c_void_p]
    return rt


class HostAlloc:
    """an exact-size cudaHostAlloc allocation, seen as a numpy array"""

    def __init__(self, rt, size):
        self.rt, self.p = rt, C.c_void_p()
        assert rt.cudaHostAlloc(C.byref(self.p), size, 0) == 0
        self.a = np.ctypeslib.as_array((C.c_uint8 * size).from_address(self.p.value))

    def free(self):
        assert self.rt.cudaFreeHost(self.p) == 0


class C2H:
    def __init__(self, prod):
        import torch
        self.t = torch
        self.L = bind(prod.lib)
        self.rt = _cudart()

    def scratch_size(self, n, o, window):
        return int(self.L.zxc_b200_compress_device_to_host_scratch_size(n, window, C.byref(o)))

    def src(self, data, src_off=0):
        t = self.t
        s = t.empty(src_off + data.size, dtype=t.uint8, device="cuda")  # the input ends at the end of its tensor
        if data.size:
            s[src_off:].copy_(t.from_numpy(data))
        return s

    def enqueue(self, d_src, n, h_dst, cap, o, window, scratch, ss, result, dd=None, stream=None):
        st = stream.cuda_stream if stream is not None else None
        if dd is None:
            return self.L.zxc_b200_compress_device_to_host(d_src, n, h_dst, cap, C.byref(o), window, scratch.data_ptr(),
                                                           ss, result.data_ptr(), st)
        return self.L.zxc_b200_compress_device_to_host_using_dict(d_src, n, h_dst, cap, C.byref(o), dd, window,
                                                                  scratch.data_ptr(), ss, result.data_ptr(), st)

    def compress(self, data, o, window, src_off=0, scratch_size=None, dd=None):
        """-> (result, frame ndarray or None), into a pinned tensor of the bound's size"""
        t = self.t
        n = data.size
        src = self.src(data, src_off)
        cap = int(self.L.zxc_compress_bound(n))
        out = t.empty(cap, dtype=t.uint8, pin_memory=True)
        ss = scratch_size if scratch_size is not None else self.scratch_size(n, o, window)
        scratch = t.empty(max(ss, 1), dtype=t.uint8, device="cuda")
        result = t.zeros(1, dtype=t.int64, device="cuda")
        rc = self.enqueue(src.data_ptr() + src_off if n else None, n, out.data_ptr(), cap, o, window, scratch, ss,
                          result, dd)
        if rc != 0:
            return rc, None
        t.cuda.synchronize()
        r = int(result.item())
        return r, (out.numpy()[:r].copy() if r > 0 else None)


@pytest.fixture(scope="module")
def c2h(prod):
    return C2H(prod)


def _ref():
    return z.ZxcLib(z.REF_SO) if z.have_ref() else None


def check(c2h, prod, ref, data, level, bs, cks, seek, windows, d=None, h=None, dd=None, **kw):
    want = prod.compress(data, level=level, block_size=bs, checksum=cks, seekable=seek, dict=d, dict_huf=h)
    assert not isinstance(want, int)
    if ref is not None:
        rf = ref.compress(data, level=level, block_size=bs, checksum=cks, seekable=seek, dict=d, dict_huf=h)
        assert np.array_equal(want, rf), ("reference", data.size, level, bs)
    o = opts(level, bs, cks, seek, None if dd is not None else d, None if dd is not None else h)
    for w in windows:
        r, fr = c2h.compress(data, o, w, dd=dd, **kw)
        assert r == want.size, (data.size, level, bs, cks, seek, w, z.ERR.get(r, r))
        assert np.array_equal(fr, want), (data.size, level, bs, cks, seek, w)
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, 3, 5, 6, 7])
def test_parity_levels_and_block_sizes(c2h, prod, level):
    ref = _ref()
    for bs in (4096, 65536, 2 << 20):
        data = make_case("silesia", 3 * bs + 1234)
        for cks in (0, 1):
            for seek in (0, 1):
                check(c2h, prod, ref, data, level, bs, cks, seek, (bs, 3 * bs, 1 << 30))


@pytest.mark.gpu
def test_windows(c2h, prod):
    """one block, three blocks, a window that is not a whole number of blocks, 0, and more than the input: one frame"""
    ref = _ref()
    bs = 4096
    data = zc.silesia_shaped(1 << 20, seed=5)[: 77 * bs + 999]
    check(c2h, prod, ref, data, 3, bs, 1, 1, (0, 1, bs, 3 * bs, 5 * bs + 17, 64 * bs, data.size, 1 << 40))
    check(c2h, prod, ref, data, 1, bs, 0, 0, (bs, 7 * bs + 1))


@pytest.mark.gpu
def test_edge_sizes(c2h, prod):
    ref = _ref()
    bs = 65536
    for n in (0, 1, bs - 1, bs, bs + 1, 9 * bs + 77):
        data = make_case("text", n)
        for seek in (0, 1):
            check(c2h, prod, ref, data, 3, bs, 1, seek, (bs, 2 * bs, 1 << 30))


@pytest.mark.gpu
def test_odd_source_offsets(c2h, prod):
    data = make_case("silesia", 5 * 4096 + 3)
    for off in (1, 3, 7, 13):
        check(c2h, prod, None, data, 2, 4096, 1, 1, (4096, 2 * 4096), src_off=off)


@pytest.mark.gpu
@pytest.mark.parametrize("level", [3, 6, 7])
def test_dictionaries(c2h, prod, level):
    from zxc_b200 import device
    d, h = next(iter(golden_dicts().values()))
    data = make_case("text", 300001)
    ref = _ref()
    check(c2h, prod, ref, data, level, 65536, 1, 1, (65536, 3 * 65536), d=d)
    if level >= 6:
        check(c2h, prod, ref, data, level, 65536, 1, 1, (65536, 1 << 30), d=d, h=h)
    with device.DeviceDict(d, h if level >= 6 else None) as dd:
        check(c2h, prod, ref, data, level, 65536, 1, 1, (65536, 1 << 30), d=d, h=h if level >= 6 else None,
              dd=dd.handle)


@pytest.mark.gpu
def test_host_memory_edges(c2h, prod):
    """frames at offsets 0-15 in exact-size cudaHostAlloc buffers with canaries on both sides, and flush against the
    allocation's end; a room of exactly the frame's size succeeds; one byte less gives DST_TOO_SMALL and nothing
    outside the room is written"""
    t = c2h.t
    G = 64
    for level, bs, n, seek in ((1, 4096, 9 * 4096 + 5, 1), (3, 65536, 3 * 65536 + 100, 0), (3, 4096, 40, 1)):
        data = make_case("silesia", n)
        want = prod.compress(data, level=level, block_size=bs, checksum=1, seekable=seek)
        o = opts(level, bs, 1, seek)
        src = c2h.src(data)
        for w in (bs, 1 << 30):
            ss = c2h.scratch_size(n, o, w)
            scratch = t.empty(ss, dtype=t.uint8, device="cuda")
            result = t.zeros(1, dtype=t.int64, device="cuda")
            for off in range(16):
                for cap, tail in ((want.size, G), (want.size, 0), (want.size - 1, G)):
                    buf = HostAlloc(c2h.rt, G + off + cap + tail)
                    try:
                        buf.a[:] = 0xA5
                        assert c2h.enqueue(src.data_ptr(), n, buf.p.value + G + off, cap, o, w, scratch, ss,
                                           result) == 0
                        t.cuda.synchronize()
                        r = int(result.item())
                        a = buf.a.copy()
                    finally:
                        buf.free()
                    assert (a[:G + off] == 0xA5).all() and (a[G + off + cap:] == 0xA5).all(), (level, w, off, cap)
                    if cap == want.size:
                        assert r == want.size and np.array_equal(a[G + off:G + off + cap], want), (level, w, off)
                    else:
                        assert r == DST_TOO_SMALL, (level, w, off, r)
            # a room below header + trailer: the host's verdict
            fixed = HDR + EOF + FOOT + ((SEK_HDR + 4 * ((n + bs - 1) // bs)) if seek else 0)
            buf = HostAlloc(c2h.rt, fixed)
            try:
                assert c2h.enqueue(src.data_ptr(), n, buf.p.value, fixed - 1, o, w, scratch, ss, result) == \
                    DST_TOO_SMALL
            finally:
                buf.free()


@pytest.mark.gpu
def test_registered_and_pageable_memory(c2h, prod):
    """cudaHostRegister memory is accepted; pageable memory gives UNSUPPORTED and stays untouched"""
    t = c2h.t
    data = make_case("silesia", 200001)
    o = opts(3, 65536, 1, 1)
    want = prod.compress(data, level=3, block_size=65536, checksum=1, seekable=1)
    src = c2h.src(data)
    ss = c2h.scratch_size(data.size, o, 65536)
    scratch = t.empty(ss, dtype=t.uint8, device="cuda")
    result = t.zeros(1, dtype=t.int64, device="cuda")
    cap = int(c2h.L.zxc_compress_bound(data.size))
    pageable = np.full(cap + 64, 0xA5, np.uint8)
    assert c2h.enqueue(src.data_ptr(), data.size, pageable.ctypes.data + 3, cap, o, 65536, scratch, ss,
                       result) == UNSUPPORTED
    assert (pageable == 0xA5).all()
    assert c2h.rt.cudaHostRegister(pageable.ctypes.data, pageable.nbytes, 0) == 0
    try:
        assert c2h.enqueue(src.data_ptr(), data.size, pageable.ctypes.data + 3, cap, o, 65536, scratch, ss,
                           result) == 0
        t.cuda.synchronize()
        assert int(result.item()) == want.size
        assert np.array_equal(pageable[3:3 + want.size], want)
        # a room that runs past the registered range is not one mapping
        assert c2h.enqueue(src.data_ptr(), data.size, pageable.ctypes.data + 3, cap + 64, o, 65536, scratch, ss,
                           result) == UNSUPPORTED
    finally:
        assert c2h.rt.cudaHostUnregister(pageable.ctypes.data) == 0


@pytest.mark.gpu
def test_verdict_order(c2h, prod):
    """zxc_b200_compress_device's host verdicts in its order, UNSUPPORTED just before MEMORY"""
    t = c2h.t
    data = make_case("text", 10000)
    src = c2h.src(data)
    cap = int(c2h.L.zxc_compress_bound(data.size))
    out = t.empty(cap, dtype=t.uint8, pin_memory=True)
    pageable = np.zeros(cap, np.uint8)
    o = opts(6, 4096)
    ss = c2h.scratch_size(data.size, o, 4096)
    scratch = t.empty(ss, dtype=t.uint8, device="cuda")
    result = t.zeros(1, dtype=t.int64, device="cuda")
    d, h = next(iter(golden_dicts().values()))
    bad = bytes([0x11]) * 128  # 256 codes of length 1: not a prefix code
    p, q = src.data_ptr(), pageable.ctypes.data
    e = c2h.enqueue
    assert e(p, data.size, q, cap, opts(6, 5000, d=b"x" * 70000), 0, scratch, 1, result) == DICT_BIG
    assert e(p, data.size, q, cap, opts(6, 5000), 0, scratch, 1, result) == BAD_BS
    assert e(p, data.size, q, 20, o, 0, scratch, 1, result) == DST_TOO_SMALL
    assert e(p, data.size, q, cap, opts(6, 4096, d=d, h=bad), 0, scratch, 1, result) == CORRUPT
    assert e(p, data.size, q, cap, o, 0, scratch, 1, result) == UNSUPPORTED
    assert e(p, data.size, out.data_ptr(), cap, o, 0, scratch, 1, result) == MEMORY
    assert e(None, data.size, out.data_ptr(), cap, o, 0, scratch, ss, result) == NULL_INPUT
    assert c2h.scratch_size(data.size, opts(6, 5000), 4096) == 0


@pytest.mark.gpu
def test_scratch_for_one_warp(c2h, prod):
    """one warp's scratch gives the same bytes; a byte less gives MEMORY"""
    ref = _ref()
    for level, bs in ((3, 65536), (6, 65536), (7, 4096)):
        w = 4 * bs
        n = 10 * bs + 3
        s4 = c2h.scratch_size(n, opts(level, bs, 1, 1), w)  # four blocks per window: one CTA of four warps
        s8 = c2h.scratch_size(n, opts(level, bs, 1, 1), 8 * bs)  # eight: two CTAs, four more slots and staging
        sstride = (bs + 80 + 255) & ~255
        assert (s8 - s4 - 4 * bs - 4 * sstride) % 4 == 0
        per = (s8 - s4 - 4 * bs - 4 * sstride) // 4
        one = s4 - 3 * per
        data = make_case("silesia", n)
        want = check(c2h, prod, ref, data, level, bs, 1, 1, (w,), scratch_size=one)
        r, _ = c2h.compress(data, opts(level, bs, 1, 1), w, scratch_size=one - 1)
        assert r == MEMORY, (level, bs, per)
        assert want is not None


@pytest.mark.gpu
def test_graph_capture_and_replay(c2h, prod):
    """captured once, replayed over new input contents: the frame is rewritten correctly each time"""
    t = c2h.t
    n, bs, w = 700001, 65536, 3 * 65536
    o = opts(3, bs, 1, 1)
    src = t.empty(n, dtype=t.uint8, device="cuda")
    cap = int(c2h.L.zxc_compress_bound(n))
    out = t.empty(cap + 7, dtype=t.uint8, pin_memory=True)
    ss = c2h.scratch_size(n, o, w)
    scratch = t.empty(ss, dtype=t.uint8, device="cuda")
    result = t.zeros(1, dtype=t.int64, device="cuda")
    s = t.cuda.Stream()
    s.wait_stream(t.cuda.current_stream())
    with t.cuda.stream(s):  # warm-up outside capture
        assert c2h.enqueue(src.data_ptr(), n, out.data_ptr() + 7, cap, o, w, scratch, ss, result, stream=s) == 0
    t.cuda.current_stream().wait_stream(s)
    t.cuda.synchronize()
    g = t.cuda.CUDAGraph()
    with t.cuda.graph(g):
        assert c2h.enqueue(src.data_ptr(), n, out.data_ptr() + 7, cap, o, w, scratch, ss, result,
                           stream=t.cuda.current_stream()) == 0
    for seed in (1, 2, 3):
        data = zc.silesia_shaped(1 << 20, seed=seed)[:n]
        src.copy_(t.from_numpy(data))
        out.zero_()
        g.replay()
        t.cuda.synchronize()
        want = prod.compress(data, level=3, block_size=bs, checksum=1, seekable=1)
        assert int(result.item()) == want.size
        assert np.array_equal(out.numpy()[7:7 + want.size], want), seed


@pytest.mark.gpu
def test_two_streams(c2h, prod):
    t = c2h.t
    bs, w = 65536, 2 * 65536
    datas = [zc.silesia_shaped(3 << 20, seed=61 + i)[: (3 << 20) - 5 * i] for i in range(2)]
    o = opts(3, bs, 1, 1)
    streams = [t.cuda.Stream(), t.cuda.Stream()]
    state = []
    for data, s in zip(datas, streams):
        src = c2h.src(data)
        cap = int(c2h.L.zxc_compress_bound(data.size))
        out = t.empty(cap, dtype=t.uint8, pin_memory=True)
        ss = c2h.scratch_size(data.size, o, w)
        scratch = t.empty(ss, dtype=t.uint8, device="cuda")
        result = t.zeros(1, dtype=t.int64, device="cuda")
        state.append((src, out, cap, scratch, ss, result))
    for s in streams:
        s.wait_stream(t.cuda.current_stream())
    for _ in range(2):
        for (src, out, cap, scratch, ss, result), data, s in zip(state, datas, streams):
            assert c2h.enqueue(src.data_ptr(), data.size, out.data_ptr(), cap, o, w, scratch, ss, result,
                               stream=s) == 0
    t.cuda.synchronize()
    for (src, out, cap, scratch, ss, result), data in zip(state, datas):
        want = prod.compress(data, level=3, block_size=bs, checksum=1, seekable=1)
        assert int(result.item()) == want.size
        assert np.array_equal(out.numpy()[:want.size], want)


@pytest.mark.gpu
def test_launch_count(c2h, prod):
    from zxc_b200 import device
    d, h = next(iter(golden_dicts().values()))
    L = c2h.L
    bs = 65536
    for n, w, dct, dd, want in ((300000, bs, None, False, 1 + 5 * 5), (300000, 1 << 30, None, False, 1 + 5),
                                (0, bs, None, False, 1), (300000, 2 * bs, d, False, 1 + 5 * 3 + 1),
                                (300000, 2 * bs, d, True, 1 + 5 * 3)):
        data = make_case("text", n)
        if dd:
            with device.DeviceDict(d) as dev_dict:
                n0 = L.zxc_b200_launch_count()
                r, _ = c2h.compress(data, opts(3, bs, 1, 1), w, dd=dev_dict.handle)
                got = L.zxc_b200_launch_count() - n0
        else:
            n0 = L.zxc_b200_launch_count()
            r, _ = c2h.compress(data, opts(3, bs, 1, 1, d=dct), w)
            got = L.zxc_b200_launch_count() - n0
        assert r > 0
        assert got == want, (n, w, dct is not None, dd, got)


@pytest.mark.gpu
def test_round_trips(c2h, prod):
    """a seekable output opens with zxc_b200_seekable_device_open_host and decodes back, whole and over random ranges;
    any output decodes back with load_frame"""
    import torch
    from zxc_b200 import device
    data = zc.silesia_shaped(6 << 20, seed=17)[: (6 << 20) - 333]
    x = torch.from_numpy(data).cuda()
    frame = device.compress_to_host(x, level=3, block_size=65536, checksum=True, seekable=True, window=1 << 20)
    assert frame.is_pinned()
    sf = device.SeekableFrame(frame)
    assert sf.decompressed_size == data.size
    assert np.array_equal(sf.read(0, data.size).cpu().numpy(), data)
    rng = np.random.default_rng(3)
    offs = rng.integers(0, data.size - 5000, 200)
    lens = rng.integers(1, 5000, 200)
    got, res = sf.gather(torch.from_numpy(offs), torch.from_numpy(lens))
    assert res.tolist() == lens.tolist()
    want = np.concatenate([data[o:o + k] for o, k in zip(offs, lens)])
    assert np.array_equal(got.cpu().numpy(), want)
    sf.close()
    for kw in (dict(level=1), dict(level=5, block_size=4096, checksum=True), dict(level=6, seekable=True)):
        fr = device.compress_to_host(x, window=3 << 20, **kw)
        assert np.array_equal(device.load_frame(fr, checksum=True).cpu().numpy(), data), kw


@pytest.mark.gpu
def test_python_helper(prod):
    """compress_to_host: the frame of zxc_compress, into `out` or a fresh pinned tensor, with host or device
    dictionaries, on a side stream; ZxcError with the code"""
    import torch
    from zxc_b200 import device
    data = zc.silesia_shaped(2 << 20, seed=23)
    x = torch.from_numpy(data).cuda()
    want = prod.compress(data, level=3, block_size=65536, checksum=1, seekable=1)
    fr = device.compress_to_host(x, level=3, block_size=65536, checksum=True, seekable=True, window=300000)
    assert np.array_equal(fr.numpy(), want)
    out = torch.empty(want.size + 100, dtype=torch.uint8, pin_memory=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    fr2 = device.compress_to_host(x, level=3, block_size=65536, checksum=True, seekable=True, out=out, stream=s)
    assert fr2.data_ptr() == out.data_ptr() and np.array_equal(fr2.numpy(), want)
    d, h = next(iter(golden_dicts().values()))
    wd = prod.compress(data, level=6, block_size=65536, dict=d, dict_huf=h)
    assert np.array_equal(device.compress_to_host(x, level=6, block_size=65536, dict=d, dict_huf=h).numpy(), wd)
    with device.DeviceDict(d, h) as dd:
        assert np.array_equal(device.compress_to_host(x, level=6, block_size=65536, dict=dd).numpy(), wd)
    small = torch.empty(100, dtype=torch.uint8, pin_memory=True)
    with pytest.raises(device.ZxcError) as e:
        device.compress_to_host(x, level=3, out=small)
    assert e.value.code == DST_TOO_SMALL
    with pytest.raises(device.ZxcError) as e:
        device.compress_to_host(x, level=3, out=torch.empty(want.size - 1, dtype=torch.uint8, pin_memory=True),
                                block_size=65536, checksum=True, seekable=True)
    assert e.value.code == DST_TOO_SMALL
    empty = device.compress_to_host(torch.empty(0, dtype=torch.uint8, device="cuda"), level=3)
    assert np.array_equal(empty.numpy(), prod.compress(np.empty(0, np.uint8), level=3))
