"""zxc_b200_compress_device: a frame compressed from HBM into HBM on a stream, assembled on the device.

Frames are read back and compared byte for byte with zxc_compress (host to host, pinned to the reference by
test_encode_gpu.py) and with the reference itself; the decode plan it emits is compared with zxc_b200_plan_frame."""
import ctypes as C

import numpy as np
import pytest

import zxc_corpus as zc
import zxc_ctypes as z
from conftest import has_cuda
from test_oracle import CASES, golden_dicts, make_case

HDR, EOF, FOOT, SEK_HDR = 16, 8, 12, 8
NULL_INPUT, DST_TOO_SMALL, CORRUPT, BAD_BS, DICT_BIG, MEMORY, NO_DEVICE = -12, -2, -8, -14, -17, -1, -100


class Job(C.Structure):
    _fields_ = [("src_off", C.c_uint64), ("dst_off", C.c_uint64), ("src_len", C.c_uint32), ("dst_cap", C.c_uint32)]


def bind(L):
    L.zxc_b200_encode_scratch_size.restype = C.c_size_t
    L.zxc_b200_encode_scratch_size.argtypes = [C.c_uint64, C.c_void_p]
    L.zxc_b200_compress_device.restype = C.c_int
    L.zxc_b200_compress_device.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                           C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    L.zxc_b200_plan_frame.restype = C.c_int64
    L.zxc_b200_plan_frame.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    L.zxc_b200_launch_count.restype = C.c_uint64
    return L


def opts(level=0, bs=0, cks=0, seek=0, d=None, h=None):
    o = z.CompressOpts(level=level, block_size=bs, checksum_enabled=cks, seekable=seek)
    keep = []
    if d is not None:
        d = bytes(d)
        keep.append(d)
        o.dict, o.dict_size = C.cast(C.c_char_p(d), C.c_void_p), len(d)
        if h is not None:
            h = bytes(h)
            keep.append(h)
            o.dict_huf = C.cast(C.c_char_p(h), C.c_void_p)
    o._keep = keep
    return o


def test_host_verdicts_without_a_device(prod):
    """Argument verdicts come in zxc_compress's order and need no device; without one the call then fails loudly and
    the scratch query returns 0."""
    if has_cuda():
        pytest.skip("only meaningful without a GPU")
    L = bind(prod.lib)
    fake = 1 << 40  # never dereferenced: every verdict here is decided before the device is touched
    cd = L.zxc_b200_compress_device
    assert cd(fake, 100, None, 1000, None, fake, 1 << 20, fake, None, None) == NULL_INPUT
    assert cd(fake, 100, fake, 0, None, fake, 1 << 20, fake, None, None) == NULL_INPUT
    assert cd(None, 100, fake, 1000, None, fake, 1 << 20, fake, None, None) == NULL_INPUT
    assert cd(fake, 100, fake, 1000, None, None, 1 << 20, fake, None, None) == NULL_INPUT
    assert cd(fake, 100, fake, 1000, None, fake, 1 << 20, None, None, None) == NULL_INPUT
    big = opts(3, 3000, d=b"x" * 70000)  # dictionary first, then block size
    assert cd(fake, 100, fake, 1000, C.byref(big), fake, 1 << 20, fake, None, None) == DICT_BIG
    assert cd(fake, 100, fake, 1000, C.byref(opts(3, 3000)), fake, 1 << 20, fake, None, None) == BAD_BS
    assert cd(fake, 100, fake, 1000, C.byref(opts(3, 1 << 22)), fake, 1 << 20, fake, None, None) == BAD_BS
    assert cd(fake, 100, fake, 1000, C.byref(opts(3, 65536)), fake, 1 << 20, fake, None, None) == NO_DEVICE
    assert cd(None, 0, fake, 1, None, fake, 1, fake, None, None) == NO_DEVICE  # empty input: no source needed
    assert L.zxc_b200_encode_scratch_size(1 << 20, None) == 0
    assert L.zxc_b200_encode_scratch_size(1 << 20, C.byref(opts(6, 65536))) == 0


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
class Dev:
    """compress_device through the C ABI with torch buffers"""

    def __init__(self, prod):
        import torch
        self.torch = torch
        self.L = bind(prod.lib)

    def scratch_size(self, n, o):
        return int(self.L.zxc_b200_encode_scratch_size(n, C.byref(o)))

    def enqueue(self, d_src, n, d_dst, cap, o, scratch, result, jobs=None, stream=None, scratch_size=None):
        return self.L.zxc_b200_compress_device(
            d_src, n, d_dst, cap, C.byref(o), scratch.data_ptr(),
            scratch.numel() if scratch_size is None else scratch_size, result.data_ptr(),
            jobs.data_ptr() if jobs is not None else None, stream.cuda_stream if stream is not None else None)

    def compress(self, data, o, src_off=0, dst_off=0, jobs=False, scratch_size=None):
        """-> (result, frame bytes or None, jobs ndarray or None)"""
        t = self.torch
        n = data.size
        src = t.empty(src_off + n, dtype=t.uint8, device="cuda")  # the input ends at the end of its tensor
        if n:
            src[src_off:].copy_(t.from_numpy(data))
        cap = int(self.L.zxc_compress_bound(n))
        dst = t.empty(dst_off + cap, dtype=t.uint8, device="cuda")
        ss = scratch_size if scratch_size is not None else self.scratch_size(n, o)
        scratch = t.empty(ss, dtype=t.uint8, device="cuda")
        result = t.zeros(1, dtype=t.int64, device="cuda")
        bs = o.block_size or 512 * 1024
        nb = (n + bs - 1) // bs
        d_jobs = t.empty(max(nb, 1) * 24, dtype=t.uint8, device="cuda") if jobs else None
        rc = self.enqueue(src.data_ptr() + src_off if n else None, n, dst.data_ptr() + dst_off, cap, o, scratch,
                          result, d_jobs)
        if rc != 0:
            return rc, None, None
        t.cuda.synchronize()
        r = int(result.item())
        if r < 0:
            return r, None, None
        frame = dst[dst_off:dst_off + r].cpu().numpy()
        return r, frame, (d_jobs[:nb * 24].cpu().numpy() if jobs else None)


def plan(L, frame):
    nb = L.zxc_b200_plan_frame(frame.ctypes.data, frame.size, None, 0, None)
    assert nb >= 0
    jobs = (Job * max(nb, 1))()
    assert L.zxc_b200_plan_frame(frame.ctypes.data, frame.size, jobs, nb, None) == nb
    return np.frombuffer(bytes(jobs), np.uint8)[:nb * 24]


@pytest.fixture(scope="module")
def dev(prod):
    return Dev(prod)


def check(dev, prod, ref, data, level, bs, cks, seek, d=None, h=None, **kw):
    o = opts(level, bs, cks, seek, d, h)
    r, fr, jobs = dev.compress(data, o, jobs=True, **kw)
    assert r > 0, (level, bs, cks, seek, z.ERR.get(r, r))
    want = prod.compress(data, level=level, block_size=bs, checksum=cks, seekable=seek, dict=d, dict_huf=h)
    assert not isinstance(want, int)
    assert fr.size == want.size and np.array_equal(fr, want), (data.size, level, bs, cks, seek)
    if ref is not None:
        rf = ref.compress(data, level=level, block_size=bs, checksum=cks, seekable=seek, dict=d, dict_huf=h)
        assert np.array_equal(fr, rf), ("reference", data.size, level, bs, cks, seek)
    assert np.array_equal(jobs, plan(dev.L, fr)), ("decode plan", data.size, level, bs)
    return fr


def _ref():
    return z.ZxcLib(z.REF_SO) if z.have_ref() else None


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, 2, 3, 4, 5, 6, 7])
def test_parity_with_host_path_and_reference(dev, prod, level):
    ref = _ref()
    for kind, n in CASES:
        if level >= 6 and n > 1 << 20:
            n = 1 << 20  # a single warp parses each block at levels 6-7: keep the big case to seconds
        data = make_case(kind, n)
        for bs in (4096, 65536, 0):
            if bs == 0 and level >= 6 and n > 200000:
                continue
            for cks in (0, 1):
                for seek in (0, 1):
                    check(dev, prod, ref, data, level, bs, cks, seek)


@pytest.mark.gpu
@pytest.mark.parametrize("level", [5, 6, 7])
def test_parity_with_dictionaries(dev, prod, level):
    ref = _ref()
    data = make_case("text", 150000)
    for d, h in golden_dicts().values():
        for huf in (None, h):
            for bs, cks, seek in ((4096, 1, 1), (65536, 0, 0)):
                check(dev, prod, ref, data, level, bs, cks, seek, d=d, h=huf)


@pytest.mark.gpu
def test_edge_sizes_and_hash_wrap(dev, prod):
    ref = _ref()
    bs = 4096
    base = zc.silesia_shaped(1100 * bs, seed=31)
    for n in (0, 1, bs - 1, bs, bs + 1):
        for cks, seek in ((0, 0), (1, 1)):
            check(dev, prod, ref, base[:n], 3, bs, cks, seek)
    for nb in (31, 32, 33, 1023, 1024, 1025):  # the global hash's rotation wraps every 32 blocks
        check(dev, prod, ref, base[:nb * bs - 7], 1, bs, 1, 1)
        check(dev, prod, ref, base[:nb * bs], 2, bs, 1, 0)


@pytest.mark.gpu
def test_half_a_million_blocks(dev, prod):
    """2^19 blocks (2 GiB at 4 KiB, level 1): the multi-CTA scan and the hash reduction at scale."""
    ref = _ref()
    bs = 4096
    data = zc.silesia_shaped(bs << 19, seed=41)
    o = opts(1, bs, 1, 1)
    r, fr, jobs = dev.compress(data, o, jobs=True)
    assert r > 0, z.ERR.get(r, r)
    want = prod.compress(data, level=1, block_size=bs, checksum=1, seekable=1)
    assert fr.size == want.size and np.array_equal(fr, want)
    assert np.array_equal(jobs, plan(dev.L, fr))
    del want, jobs
    if ref is not None:  # the reference on a prefix of whole blocks: the same block bytes
        k = 4096
        rp = ref.compress(data[:k * bs], level=1, block_size=bs, checksum=1)
        body = rp[HDR:rp.size - EOF - FOOT]
        assert np.array_equal(fr[HDR:HDR + body.size], body)


@pytest.mark.gpu
@pytest.mark.parametrize("src_off,dst_off", [(1, 3), (3, 15), (15, 1)])
def test_unaligned_buffers(dev, prod, src_off, dst_off):
    ref = _ref()
    data = make_case("silesia", 300001)
    for level, bs in ((1, 4096), (3, 65536), (6, 65536)):
        check(dev, prod, ref, data, level, bs, 1, 1, src_off=src_off, dst_off=dst_off)


@pytest.mark.gpu
def test_capacity(dev, prod):
    t = dev.torch
    data = make_case("text", 200000)
    o = opts(3, 65536, 1, 1)
    want = prod.compress(data, level=3, block_size=65536, checksum=1, seekable=1)
    src = t.from_numpy(data).cuda()
    scratch = t.empty(dev.scratch_size(data.size, o), dtype=t.uint8, device="cuda")
    result = t.zeros(1, dtype=t.int64, device="cuda")
    guard = 4096
    for cap, expect in ((want.size, want.size), (want.size - 1, DST_TOO_SMALL)):
        dst = t.full((cap + guard,), 0xA5, dtype=t.uint8, device="cuda")
        assert dev.enqueue(src.data_ptr(), data.size, dst.data_ptr(), cap, o, scratch, result) == 0
        t.cuda.synchronize()
        assert int(result.item()) == expect
        h = dst.cpu().numpy()
        assert (h[cap:] == 0xA5).all(), "written past dst_capacity"
        if expect > 0:
            assert np.array_equal(h[:cap], want)
    nb = (data.size + 65535) // 65536
    fixed = HDR + EOF + SEK_HDR + 4 * nb + FOOT
    dst = t.empty(fixed, dtype=t.uint8, device="cuda")
    assert dev.enqueue(src.data_ptr(), data.size, dst.data_ptr(), fixed - 1, o, scratch, result) == DST_TOO_SMALL
    # header + trailer fit: the host accepts, the device finds the body does not fit
    result.fill_(7)
    assert dev.enqueue(src.data_ptr(), data.size, dst.data_ptr(), fixed, o, scratch, result) == 0
    t.cuda.synchronize()
    assert int(result.item()) == DST_TOO_SMALL


@pytest.mark.gpu
def test_host_verdicts_with_a_device(dev, prod):
    t = dev.torch
    data = make_case("text", 10000)
    src = t.from_numpy(data).cuda()
    dst = t.empty(int(dev.L.zxc_compress_bound(data.size)), dtype=t.uint8, device="cuda")
    o = opts(6, 4096)
    scratch = t.empty(dev.scratch_size(data.size, o), dtype=t.uint8, device="cuda")
    result = t.zeros(1, dtype=t.int64, device="cuda")
    d, h = next(iter(golden_dicts().values()))
    bad = bytes([0x11]) * 128  # 256 codes of length 1: not a prefix code
    assert dev.enqueue(src.data_ptr(), data.size, dst.data_ptr(), dst.numel(), opts(6, 4096, d=d, h=bad),
                       scratch, result) == CORRUPT
    assert dev.enqueue(src.data_ptr(), data.size, dst.data_ptr(), 20, o, scratch, result) == DST_TOO_SMALL
    assert dev.enqueue(src.data_ptr(), data.size, dst.data_ptr(), dst.numel(), opts(6, 5000), scratch,
                       result) == BAD_BS
    assert dev.scratch_size(data.size, opts(6, 5000)) == 0
    t.cuda.synchronize()


@pytest.mark.gpu
def test_round_trip_on_a_stream_without_host_sync(dev, prod):
    t = dev.torch
    L = dev.L
    L.zxc_b200_decode_scratch_size.restype = C.c_size_t
    L.zxc_b200_decode_scratch_size.argtypes = [C.c_uint32]
    L.zxc_b200_decode_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                         C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_int,
                                         C.c_void_p]
    L.zxc_b200_reduce_status.restype = C.c_int64
    L.zxc_b200_reduce_status.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    data = zc.silesia_shaped(24 << 20, seed=17)
    bs = 65536
    nb = (data.size + bs - 1) // bs
    o = opts(3, bs, 1, 1)
    s = t.cuda.Stream()
    with t.cuda.stream(s):
        src = t.from_numpy(data).cuda(non_blocking=False)
        cap = int(L.zxc_compress_bound(data.size))
        dst = t.empty(cap, dtype=t.uint8, device="cuda")
        scratch = t.empty(dev.scratch_size(data.size, o), dtype=t.uint8, device="cuda")
        result = t.zeros(1, dtype=t.int64, device="cuda")
        jobs = t.empty(nb * 24, dtype=t.uint8, device="cuda")
        out = t.empty(data.size, dtype=t.uint8, device="cuda")
        status = t.empty(nb, dtype=t.int32, device="cuda")
        dss = int(L.zxc_b200_decode_scratch_size(bs))
        dscr = t.empty(dss, dtype=t.uint8, device="cuda")
    s.synchronize()
    assert dev.enqueue(src.data_ptr(), data.size, dst.data_ptr(), cap, o, scratch, result, jobs, stream=s) == 0
    assert L.zxc_b200_decode_blocks(dst.data_ptr(), out.data_ptr(), jobs.data_ptr(), nb, status.data_ptr(), None, 0,
                                    None, dscr.data_ptr(), dss, bs, 1, s.cuda_stream) == 0
    assert L.zxc_b200_reduce_status(status.data_ptr(), jobs.data_ptr(), nb, s.cuda_stream) == data.size
    assert t.equal(out, src)
    r = int(result.item())
    fr = dst[:r].cpu().numpy()
    assert np.array_equal(fr, prod.compress(data, level=3, block_size=bs, checksum=1, seekable=1))
    assert np.array_equal(jobs.cpu().numpy(), plan(L, fr))


@pytest.mark.gpu
def test_two_streams_interleaved(dev, prod):
    t = dev.torch
    L = dev.L
    inputs = [zc.silesia_shaped(6 << 20, seed=51), make_case("text", 5 << 20)]
    o = [opts(3, 65536, 1, 1), opts(6, 65536, 0, 1)]
    streams = [t.cuda.Stream(), t.cuda.Stream()]
    bufs = []
    for i in range(2):
        src = t.from_numpy(inputs[i]).cuda()
        cap = int(L.zxc_compress_bound(inputs[i].size))
        bufs.append((src, t.empty(cap, dtype=t.uint8, device="cuda"), cap,
                     t.empty(dev.scratch_size(inputs[i].size, o[i]), dtype=t.uint8, device="cuda"),
                     t.zeros(1, dtype=t.int64, device="cuda")))
    t.cuda.synchronize()
    frames = [[], []]
    for rep in range(3):
        for i in (0, 1):
            src, dst, cap, scr, res = bufs[i]
            assert dev.enqueue(src.data_ptr(), inputs[i].size, dst.data_ptr(), cap, o[i], scr, res,
                               stream=streams[i]) == 0
        for i in (0, 1):
            streams[i].synchronize()
            src, dst, cap, scr, res = bufs[i]
            frames[i].append(dst[:int(res.item())].cpu().numpy())
    want = [prod.compress(inputs[0], level=3, block_size=65536, checksum=1, seekable=1),
            prod.compress(inputs[1], level=6, block_size=65536, seekable=1)]
    for i in (0, 1):
        for f in frames[i]:
            assert np.array_equal(f, want[i])


@pytest.mark.gpu
def test_graph_capture_and_replay(dev, prod):
    t = dev.torch
    L = dev.L
    n = 3 << 20
    o = opts(2, 65536, 1, 1)
    src = t.empty(n, dtype=t.uint8, device="cuda")
    cap = int(L.zxc_compress_bound(n))
    dst = t.empty(cap, dtype=t.uint8, device="cuda")
    scratch = t.empty(dev.scratch_size(n, o), dtype=t.uint8, device="cuda")
    result = t.zeros(1, dtype=t.int64, device="cuda")
    src.copy_(t.from_numpy(zc.silesia_shaped(n, seed=61)))
    s = t.cuda.Stream()
    s.wait_stream(t.cuda.current_stream())
    with t.cuda.stream(s):  # warm-up outside the capture
        assert dev.enqueue(src.data_ptr(), n, dst.data_ptr(), cap, o, scratch, result,
                           stream=t.cuda.current_stream()) == 0
    t.cuda.current_stream().wait_stream(s)
    t.cuda.synchronize()
    g = t.cuda.CUDAGraph()
    with t.cuda.graph(g):
        assert dev.enqueue(src.data_ptr(), n, dst.data_ptr(), cap, o, scratch, result,
                           stream=t.cuda.current_stream()) == 0
    for seed in (62, 63):
        data = zc.silesia_shaped(n, seed=seed)
        src.copy_(t.from_numpy(data))
        result.fill_(0)
        g.replay()
        t.cuda.synchronize()
        fr = dst[:int(result.item())].cpu().numpy()
        assert np.array_equal(fr, prod.compress(data, level=2, block_size=65536, checksum=1, seekable=1)), seed


@pytest.mark.gpu
def test_scratch_for_one_warp(dev, prod):
    """The per-warp slot w follows from the scratch query: 4 blocks take one CTA of 4 warps, 5 blocks two CTAs
    (8 warps) and one more staging slot.  One warp's scratch gives the same frame; a byte less is refused."""
    ref = _ref()
    for level, bs in ((3, 65536), (6, 65536), (7, 4096)):
        sstride = (bs + 80 + 255) & ~255
        s4 = dev.scratch_size(4 * bs, opts(level, bs))
        s5 = dev.scratch_size(4 * bs + 1, opts(level, bs))
        w = (s5 - s4 - sstride) // 4
        assert w > 0 and s5 - s4 - sstride == 4 * w
        one = s4 - 3 * w
        data = make_case("silesia", 4 * bs)
        check(dev, prod, ref, data, level, bs, 1, 1, scratch_size=one)
        r, _, _ = dev.compress(data, opts(level, bs), scratch_size=one - 1)
        assert r == MEMORY


@pytest.mark.gpu
def test_launch_count(dev, prod):
    t = dev.torch
    L = dev.L
    d, h = next(iter(golden_dicts().values()))
    for data, o, want in ((make_case("text", 300000), opts(3, 65536, 1, 1), 6), (make_case("text", 0), opts(3), 1),
                          (make_case("text", 100000), opts(6, 65536, d=d, h=h), 7)):
        n0 = L.zxc_b200_launch_count()
        r, _, _ = dev.compress(data, o)
        assert r > 0
        assert L.zxc_b200_launch_count() - n0 == want
    t.cuda.synchronize()


@pytest.mark.gpu
def test_python_device_helper(prod):
    import torch
    from zxc_b200 import device
    data = zc.silesia_shaped(9 << 20, seed=71)
    src = torch.from_numpy(data).cuda()
    s = torch.cuda.Stream()
    for kw in (dict(level=3, block_size=65536, checksum=True, seekable=True), dict(level=1),
               dict(level=6, block_size=4096)):
        f = device.compress(src, stream=s, **kw)
        want = prod.compress(data, level=kw["level"], block_size=kw.get("block_size", 0),
                             checksum=int(kw.get("checksum", False)), seekable=int(kw.get("seekable", False)))
        assert np.array_equal(f.frame.cpu().numpy(), want)
        assert f.decoded_size == data.size and f.n_blocks == (data.size + f.block_size - 1) // f.block_size
        out = device.decompress(f, verify=True, stream=s)
        assert torch.equal(out, src)
    floats = torch.linspace(0, 1, 100003, device="cuda")  # any dtype, viewed as bytes
    f = device.compress(floats, level=2)
    assert torch.equal(device.decompress(f).view(torch.float32), floats)
    d, h = next(iter(golden_dicts().values()))
    f = device.compress(src[:300000], level=6, block_size=4096, dict=d, dict_huf=h)
    assert torch.equal(device.decompress(f), src[:300000])
    e = device.compress(torch.empty(0, dtype=torch.uint8, device="cuda"))
    assert e.frame.numel() == HDR + EOF + FOOT and device.decompress(e).numel() == 0
