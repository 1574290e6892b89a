"""zxc_b200_decompress_device: a frame in HBM planned, decoded and checked on the device, on a stream.

The oracle for every result is zxc_decompress through the C ABI (pinned to the reference by test_decode_gpu.py);
where the reference library is built it is compared as well.  Vectors come from tests/golden."""
import ctypes as C
import glob
import os
import struct

import numpy as np
import pytest

import zxc_corpus as zc
import zxc_ctypes as z
from conftest import has_cuda
from test_oracle import CASES, G, GC_DICT, INVALID, VALID, golden_dicts, make_case

HDR, EOF, FOOT = 16, 8, 12
NULL_INPUT, SRC_SMALL, DST_TOO_SMALL, DICT_BIG, MEMORY, NO_DEVICE = -12, -3, -2, -17, -1, -100


def bind(L):
    L.zxc_b200_decompress_device_scratch_size.restype = C.c_size_t
    L.zxc_b200_decompress_device_scratch_size.argtypes = [C.c_uint64, C.c_uint32]
    L.zxc_b200_decompress_device.restype = C.c_int
    L.zxc_b200_decompress_device.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                             C.c_size_t, C.c_void_p, C.c_void_p]
    L.zxc_b200_encode_scratch_size.restype = C.c_size_t
    L.zxc_b200_encode_scratch_size.argtypes = [C.c_uint64, C.c_void_p]
    L.zxc_b200_compress_device.restype = C.c_int
    L.zxc_b200_compress_device.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                           C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    L.zxc_b200_launch_count.restype = C.c_uint64
    return L


def dopts(cks=0, d=None, h=None):
    o = z.DecompressOpts(checksum_enabled=cks)
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
    """The verdicts that need no frame bytes come in zxc_decompress's order without a device; the size query is 0."""
    if has_cuda():
        pytest.skip("only meaningful without a GPU")
    L = bind(prod.lib)
    fake = 1 << 40  # never dereferenced
    dd = L.zxc_b200_decompress_device
    assert dd(None, 100, fake, 1000, None, fake, 1 << 20, fake, None) == NULL_INPUT
    assert dd(fake, 100, None, 1000, None, fake, 1 << 20, fake, None) == NULL_INPUT
    assert dd(fake, 100, fake, 1000, None, None, 1 << 20, fake, None) == NULL_INPUT
    assert dd(fake, 100, fake, 1000, None, fake, 1 << 20, None, None) == NULL_INPUT
    assert dd(fake, 27, fake, 1000, None, fake, 1 << 20, fake, None) == SRC_SMALL
    assert dd(fake, 27, None, 0, C.byref(dopts(d=b"x" * 70000)), fake, 1 << 20, fake, None) == SRC_SMALL
    assert dd(fake, 28, fake, 1000, C.byref(dopts(d=b"x" * 70000)), fake, 1 << 20, fake, None) == DICT_BIG
    assert dd(fake, 28, fake, 1000, C.byref(dopts(1)), fake, 1 << 20, fake, None) == NO_DEVICE
    assert dd(fake, 28, None, 0, None, fake, 0, fake, None) == NO_DEVICE  # capacity 0: no output needed
    assert L.zxc_b200_decompress_device_scratch_size(1 << 20, 65536) == 0
    assert L.zxc_b200_decompress_device_scratch_size(1 << 20, 5000) == 0


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
class Dev:
    """decompress_device through the C ABI with torch buffers"""

    def __init__(self, prod):
        import torch
        self.torch = torch
        self.L = bind(prod.lib)

    def scratch_size(self, cap, bs):
        return int(self.L.zxc_b200_decompress_device_scratch_size(cap, bs))

    def enqueue(self, d_src, n, d_dst, cap, o, scratch, result, stream=None, scratch_size=None):
        return self.L.zxc_b200_decompress_device(
            d_src, n, d_dst, cap, C.byref(o) if o is not None else None, scratch.data_ptr(),
            scratch.numel() if scratch_size is None else scratch_size, result.data_ptr(),
            stream.cuda_stream if stream is not None else None)

    def run(self, frame, cap, cks=0, d=None, h=None, src_off=0, bs=None):
        """-> (result, output bytes); the frame ends at the end of its tensor (an empty one gets a one-byte tensor)"""
        t = self.torch
        frame = np.asarray(frame, np.uint8)
        src = t.empty(src_off + max(frame.size, 1), dtype=t.uint8, device="cuda")
        if frame.size:
            src[src_off:src_off + frame.size].copy_(t.from_numpy(frame.copy()))
        if bs is None:
            bs = 1 << int(frame[5]) if frame.size > 5 and 12 <= frame[5] <= 21 else 4096
        scratch = t.empty(self.scratch_size(cap, bs), dtype=t.uint8, device="cuda")
        dst = t.empty(max(cap, 1), dtype=t.uint8, device="cuda")
        result = t.full((1,), 12345, dtype=t.int64, device="cuda")
        rc = self.enqueue(src.data_ptr() + src_off, frame.size, dst.data_ptr() if cap else None,
                          cap, dopts(cks, d, h), scratch, result)
        if rc != 0:
            return rc, np.zeros(0, np.uint8)
        t.cuda.synchronize()
        r = int(result.item())
        return r, (dst[:r].cpu().numpy() if r > 0 else np.zeros(0, np.uint8))


@pytest.fixture(scope="module")
def dev(prod):
    return Dev(prod)


def _ref():
    return z.ZxcLib(z.REF_SO) if z.have_ref() else None


def same(dev, prod, frame, cap, cks=0, d=None, h=None, ref=None, what=None, **kw):
    """the device's result and bytes equal zxc_decompress's (and the reference's, when given)"""
    r1, o1 = dev.run(frame, cap, cks, d, h, **kw)
    r0, o0 = prod.decompress(frame, cap, checksum=cks, dict=d, dict_huf=h)
    assert r1 == r0, (what, z.ERR.get(r1, r1), z.ERR.get(r0, r0))
    if r0 > 0:
        assert np.array_equal(o1, o0), what
    if ref is not None:
        rr, orr = ref.decompress(frame, cap, checksum=cks, dict=d, dict_huf=h)
        assert rr == r0, (what, "reference", rr, r0)
        if rr > 0:
            assert np.array_equal(orr, o0), what
    return r1


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, 2, 3, 4, 5, 6, 7])
def test_valid_frames(dev, prod, level):
    ref = _ref()
    for kind, n in CASES:
        if level >= 6 and n > 1 << 20:
            n = 1 << 20
        data = make_case(kind, n)
        for bs in (4096, 65536, 0) + ((2 << 20,) if kind == "silesia" else ()):
            for cks, seek in ((0, 0), (1, 1), (1, 0), (0, 1)):
                frame = prod.compress(data, level=level, block_size=bs, checksum=cks, seekable=seek)
                for opt in (0, 1):
                    r = same(dev, prod, frame, data.size, opt, ref=ref, what=(kind, level, bs, cks, seek, opt))
                    assert r == data.size


@pytest.mark.gpu
@pytest.mark.parametrize("level", [5, 6])
def test_dictionaries(dev, prod, level):
    ref = _ref()
    data = make_case("text", 150000)
    for d, h in golden_dicts().values():
        for huf in (None, h):
            for bs, cks, seek in ((4096, 1, 1), (65536, 0, 0)):
                frame = prod.compress(data, level=level, block_size=bs, checksum=cks, seekable=seek, dict=d,
                                      dict_huf=huf)
                assert same(dev, prod, frame, data.size, 1, d, huf, ref=ref) == data.size
                same(dev, prod, frame, data.size, 1)  # DICT_REQUIRED
                same(dev, prod, frame, data.size, 1, d[:-1], huf)  # DICT_MISMATCH
                same(dev, prod, frame, data.size, 1, d, bytes([0x11]) * 128)  # malformed table


@pytest.mark.gpu
def test_golden_vectors(dev, prod):
    dicts = golden_dicts()
    for name in VALID:
        frame = np.fromfile(os.path.join(G, "valid", name + ".zxc"), np.uint8)
        exp = open(os.path.join(G, "valid", name + ".expected"), "rb").read()
        did = int.from_bytes(frame[7:11].tobytes(), "little") if frame[6] & 0x40 else 0
        d, h = dicts.get(did, (None, None))
        for cks in (0, 1):
            r, out = dev.run(frame, len(exp), cks, d, h)
            assert r == len(exp) and out.tobytes() == exp, (name, cks, z.ERR.get(r, r))
            same(dev, prod, frame, len(exp), cks, d, h, what=name)
    for p in sorted(glob.glob(os.path.join(G, "format", "*.zxc"))):
        if os.path.basename(p).startswith("12_"):
            continue  # its shared table is trained first: test_golden_12_with_trained_table
        frame = np.fromfile(p, np.uint8)
        n = int(prod.lib.zxc_get_decompressed_size(frame.ctypes.data, frame.size))
        d = GC_DICT if frame[6] & 0x40 else None
        assert same(dev, prod, frame, n, 1, d, what=p) == n
    for name in sorted(INVALID):
        frame = np.fromfile(os.path.join(G, "invalid", name + ".zxc"), np.uint8)
        cap = 1 << 20
        r, _ = dev.run(frame, cap, 1)
        assert r == INVALID[name], (name, z.ERR.get(r, r))
        if frame.size:
            assert r == prod.decompress(frame, cap, checksum=1)[0], name


@pytest.mark.gpu
def test_golden_12_with_trained_table(dev, prod):
    """format archive 12 needs the shared literal table the trainer builds from the case's payload and GC_DICT
    (zxc_train_dict_huf on the GPU, as in test_train_gpu.py)"""
    from test_train_gpu import Samples, bind as bind_train, train_table

    def lcg(seed):
        s = seed
        while True:
            s = (s * 1103515245 + 12345) & 0xFFFFFFFF
            yield s

    g = lcg(0x5EEDCAFE)
    buf = b""
    while len(buf) + 160 < 4096:
        uid, sess, page = next(g) % 100000, next(g), next(g) % 64
        buf += (b"GET /api/v1/users/%d/profile?session=%08x&page=%d HTTP/1.1\r\nHost: api.example.com\r\n"
                b"Accept: application/json\r\nUser-Agent: zxc-client\r\n\r\n" % (uid, sess, page))
    payload = np.frombuffer(buf, np.uint8).copy()
    rc, huf = train_table(bind_train(prod), Samples.one(payload), GC_DICT)
    assert rc == 0
    golden = np.fromfile(os.path.join(G, "format", "12_glo_huffman_dict.zxc"), np.uint8)
    for cks in (0, 1):
        r, out = dev.run(golden, payload.size, cks, GC_DICT, huf)
        assert r == payload.size and np.array_equal(out, payload), (cks, z.ERR.get(r, r))
        same(dev, prod, golden, payload.size, cks, GC_DICT, huf)
    same(dev, prod, golden, payload.size, 1, GC_DICT)  # without the table the Huffman literals need one


@pytest.mark.gpu
def test_pinned_dictionary_may_be_reused_at_once(dev, prod):
    """The call has read the dictionary when it returns, even from page-locked memory: the stream is held back by a
    sleeping kernel, the caller's pinned copy is overwritten right after the call, and the output is still right."""
    t = dev.torch
    d, h = next(iter(golden_dicts().values()))
    data = make_case("text", 200000)
    frame = prod.compress(data, level=5, block_size=4096, dict=d)
    pinned = t.empty(len(d), dtype=t.uint8).pin_memory()
    pinned.copy_(t.frombuffer(bytearray(d), dtype=t.uint8))
    o = z.DecompressOpts(checksum_enabled=0)
    o.dict, o.dict_size = pinned.data_ptr(), len(d)
    src = t.from_numpy(frame).cuda()
    out = t.zeros(data.size, dtype=t.uint8, device="cuda")
    scr = t.empty(dev.scratch_size(data.size, 4096), dtype=t.uint8, device="cuda")
    res = t.zeros(1, dtype=t.int64, device="cuda")
    s = t.cuda.Stream()
    t.cuda.synchronize()
    with t.cuda.stream(s):
        t.cuda._sleep(200_000_000)  # about 0.1 s at 2 GHz: the copies below wait behind it
    assert dev.enqueue(src.data_ptr(), frame.size, out.data_ptr(), data.size, o, scr, res, stream=s) == 0
    pinned.fill_(0x77)
    s.synchronize()
    assert int(res.item()) == data.size and np.array_equal(out.cpu().numpy(), data)


@pytest.mark.gpu
def test_empty_frame_and_zero_capacity(dev, prod):
    e = prod.compress(np.zeros(0, np.uint8), level=3, checksum=1)
    assert same(dev, prod, e, 0, 1) == 0
    assert same(dev, prod, e, 100, 1) == 0
    f = prod.compress(make_case("text", 5000), level=3)
    assert same(dev, prod, f, 0) == DST_TOO_SMALL
    g = f.copy()
    g[0] ^= 1
    assert same(dev, prod, g, 0) == -4  # BAD_MAGIC
    h = f.copy()
    h[1 + HDR] ^= 0x40  # a damaged block header: the capacity-0 shortcut does not look at it
    assert same(dev, prod, h, 0) == DST_TOO_SMALL


def _mutants(frame, count, seed):
    rng = np.random.default_rng(seed)
    for _ in range(count):
        m = frame.copy()
        k = int(rng.integers(0, m.size))
        m[k] ^= np.uint8(int(rng.integers(1, 256)))
        yield k, m


@pytest.mark.gpu
def test_mutations(dev, prod):
    d, h = next(iter(golden_dicts().values()))
    data = zc.silesia_shaped(1 << 20, seed=5)[:90000]
    frames = [
        ("lz", prod.compress(data, level=3, block_size=4096, checksum=1), None, None),
        ("huffman", prod.compress(make_case("text", 60000), level=6, block_size=4096, checksum=1), None, None),
        ("seekable", prod.compress(data, level=2, block_size=4096, checksum=1, seekable=1), None, None),
        ("dict", prod.compress(make_case("text", 40000), level=6, block_size=4096, checksum=1, seekable=1, dict=d,
                               dict_huf=h), d, h),
    ]
    for name, frame, dd, hh in frames:
        n = int(prod.lib.zxc_get_decompressed_size(frame.ctypes.data, frame.size))
        for k, m in _mutants(frame, 80, seed=len(name)):
            for cks in (1, 0) if k % 7 == 0 else (1,):
                same(dev, prod, m, n, cks, dd, hh, what=(name, k, cks))


@pytest.mark.gpu
def test_forged_seek_tables(dev, prod):
    """SEK tables whose predictions are wrong: the sequential walk takes over and gives zxc_decompress's verdict."""
    data = zc.silesia_shaped(1 << 20, seed=7)[:200000]
    frame = prod.compress(data, level=1, block_size=4096, checksum=1, seekable=1)
    nb = (data.size + 4095) // 4096
    ent = frame.size - FOOT - 4 * nb
    sizes = np.frombuffer(frame[ent:ent + 4 * nb].tobytes(), "<u4").copy()
    cases = []
    sw = sizes.copy()
    sw[[3, 4]] = sw[[4, 3]]  # same sum, wrong offsets in between
    cases.append(sw)
    mv = sizes.copy()
    mv[0] += 1
    mv[1] -= 1  # same sum, every later offset right but one
    cases.append(mv)
    sh = sizes.copy()
    sh[-1] += 4  # the chain no longer closes at the EOF block
    cases.append(sh)
    for forged in cases:
        f = frame.copy()
        f[ent:ent + 4 * nb] = np.frombuffer(forged.astype("<u4").tobytes(), np.uint8)
        assert same(dev, prod, f, data.size, 1) == data.size
    # a damaged data header behind a valid table: the walk reports it exactly as zxc_decompress does
    f = frame.copy()
    f[HDR + int(sizes[:5].sum()) + 3] ^= 0x10
    same(dev, prod, f, data.size, 1)
    # an EOF block with a length and a table that points at it
    for cks in (0, 1):
        same(dev, prod, frame[:frame.size - 1], data.size, cks)


def _stitched(prod, data, bs, level, seed):
    rng = np.random.default_rng(seed)
    cuts, p = [], 0
    while p < data.size:
        n = int(rng.integers(1, bs + 1)) if len(cuts) % 3 else bs
        cuts.append((p, min(data.size, p + n)))
        p += n
    head, eof, blocks = None, None, []
    for a, b in cuts:
        fr = prod.compress(data[a:b], level=level, block_size=bs).tobytes()
        head, eof = fr[:16], fr[-20:-12]
        blocks.append(fr[16:-20])
    return np.frombuffer(head + b"".join(blocks) + eof + struct.pack("<QI", data.size, 0), np.uint8), len(cuts)


@pytest.mark.gpu
def test_frames_with_short_non_final_blocks(dev, prod):
    """Any split into blocks of at most block_size decodes (the general split on the device); one byte short of
    the size gives zxc_decompress's verdict."""
    data = zc.silesia_shaped(1 << 20, seed=21)[:400000]
    for level in (1, 3, 6):
        frame, _ = _stitched(prod, data, 65536, level, 4)
        assert same(dev, prod, frame, data.size, what=level) == data.size
        same(dev, prod, frame, data.size - 1, what=(level, "short"))
        same(dev, prod, frame, data.size + 70000, what=(level, "roomy"))


@pytest.mark.gpu
def test_capacity_and_guard_regions(dev, prod):
    t = dev.torch
    data = make_case("text", 300000)
    for seek in (0, 1):
        frame = prod.compress(data, level=3, block_size=65536, checksum=1, seekable=seek)
        for cap in (data.size, data.size - 1, data.size - 65536, 65536, 1, 0, data.size + 1):
            same(dev, prod, frame, cap, 1, what=(seek, cap))
        # guard bytes behind dst_capacity and around the scratch stay as they were
        src = t.from_numpy(frame).cuda()
        guard = 4096
        ss = dev.scratch_size(data.size, 65536)
        for cap in (data.size, data.size - 1):
            dst = t.full((cap + guard,), 0xA5, dtype=t.uint8, device="cuda")
            scr = t.full((ss + 2 * guard,), 0x5A, dtype=t.uint8, device="cuda")
            res = t.zeros(1, dtype=t.int64, device="cuda")
            assert dev.L.zxc_b200_decompress_device(src.data_ptr(), frame.size, dst.data_ptr(), cap,
                                                    C.byref(dopts(1)), scr.data_ptr() + guard, ss, res.data_ptr(),
                                                    None) == 0
            t.cuda.synchronize()
            r = int(res.item())
            assert r == (data.size if cap == data.size else DST_TOO_SMALL)
            h = dst.cpu().numpy()
            assert (h[cap:] == 0xA5).all(), "written past dst_capacity"
            if r > 0:
                assert np.array_equal(h[:r], data)
            g = scr.cpu().numpy()
            assert (g[:guard] == 0x5A).all() and (g[guard + ss:] == 0x5A).all(), "written outside the scratch"


@pytest.mark.gpu
def test_guard_regions_with_short_non_final_blocks(dev, prod):
    """the general split writes d_dst at offsets it computes on the device: nothing lands past dst_capacity, with the
    exact capacity and one byte short, and nothing outside the scratch"""
    t = dev.torch
    data = zc.silesia_shaped(1 << 20, seed=21)[:400000]
    guard = 4096
    for level in (1, 6):
        frame, _ = _stitched(prod, data, 65536, level, 4)
        src = t.from_numpy(frame.copy()).cuda()
        ss = dev.scratch_size(data.size, 65536)
        for cap in (data.size, data.size - 1):
            want = prod.decompress(frame, cap)[0]
            assert want == (data.size if cap == data.size else DST_TOO_SMALL)
            dst = t.full((cap + guard,), 0xA5, dtype=t.uint8, device="cuda")
            scr = t.full((ss + 2 * guard,), 0x5A, dtype=t.uint8, device="cuda")
            res = t.zeros(1, dtype=t.int64, device="cuda")
            assert dev.L.zxc_b200_decompress_device(src.data_ptr(), frame.size, dst.data_ptr(), cap, C.byref(dopts()),
                                                    scr.data_ptr() + guard, ss, res.data_ptr(), None) == 0
            t.cuda.synchronize()
            assert int(res.item()) == want, (level, cap)
            h = dst.cpu().numpy()
            assert (h[cap:] == 0xA5).all(), ("written past dst_capacity", level, cap)
            if want > 0:
                assert np.array_equal(h[:want], data)
            g = scr.cpu().numpy()
            assert (g[:guard] == 0x5A).all() and (g[guard + ss:] == 0x5A).all(), ("outside the scratch", level, cap)


@pytest.mark.gpu
@pytest.mark.parametrize("src_off", [1, 3, 7])
def test_unaligned_source(dev, prod, src_off):
    data = make_case("silesia", 300001)
    for level, bs, cks, seek in ((1, 4096, 1, 1), (3, 65536, 0, 0), (6, 65536, 1, 0)):
        frame = prod.compress(data, level=level, block_size=bs, checksum=cks, seekable=seek)
        assert same(dev, prod, frame, data.size, cks, src_off=src_off) == data.size


@pytest.mark.gpu
def test_half_a_million_blocks(dev, prod):
    """2^19 blocks of 4 KiB: the SEK-guided plan and, without a table, the sequential walk at scale."""
    data = zc.silesia_shaped(4096 << 19, seed=41)
    for seek in (1, 0):
        frame = prod.compress(data, level=1, block_size=4096, checksum=1, seekable=seek)
        r, out = dev.run(frame, data.size, 1)
        assert r == data.size, (seek, z.ERR.get(r, r))
        assert np.array_equal(out, data), seek
        del out


def _compress_device(dev, t, src, n, o, s):
    L = dev.L
    cap = int(L.zxc_compress_bound(n))
    dst = t.empty(cap, dtype=t.uint8, device="cuda")
    scr = t.empty(int(L.zxc_b200_encode_scratch_size(n, C.byref(o))), dtype=t.uint8, device="cuda")
    res = t.zeros(1, dtype=t.int64, device="cuda")
    assert L.zxc_b200_compress_device(src.data_ptr(), n, dst.data_ptr(), cap, C.byref(o), scr.data_ptr(), scr.numel(),
                                      res.data_ptr(), None, s.cuda_stream) == 0
    return dst, cap, scr, res


@pytest.mark.gpu
def test_compress_then_decompress_on_one_stream(dev, prod):
    """compress_device then decompress_device on one stream with no host synchronisation in between.  The decode
    needs the frame's size; the encoder is deterministic, so a first round learns it and the later rounds enqueue
    both calls back to back and synchronise only at the end."""
    t = dev.torch
    data = zc.silesia_shaped(24 << 20, seed=17)
    n = data.size
    s = t.cuda.Stream()
    with t.cuda.stream(s):
        src = t.from_numpy(data).cuda()
        out = t.empty(n, dtype=t.uint8, device="cuda")
        res = t.zeros(1, dtype=t.int64, device="cuda")
        dscr = t.empty(dev.scratch_size(n, 65536), dtype=t.uint8, device="cuda")
    s.synchronize()
    o = z.CompressOpts(level=3, block_size=65536, checksum_enabled=1, seekable=1)
    dst, cap, scr, cres = _compress_device(dev, t, src, n, o, s)
    s.synchronize()
    size = int(cres.item())
    for rep in range(2):
        with t.cuda.stream(s):
            out.fill_(0)
            res.fill_(0)
        dst, cap, scr, cres = _compress_device(dev, t, src, n, o, s)
        assert dev.enqueue(dst.data_ptr(), size, out.data_ptr(), n, dopts(1), dscr, res, stream=s) == 0
        s.synchronize()
        assert int(cres.item()) == size
        assert int(res.item()) == n and t.equal(out, src), rep


@pytest.mark.gpu
def test_two_streams(dev, prod):
    t = dev.torch
    inputs = [zc.silesia_shaped(6 << 20, seed=51), make_case("text", 5 << 20)]
    frames = [prod.compress(inputs[0], level=3, block_size=65536, checksum=1, seekable=1),
              prod.compress(inputs[1], level=6, block_size=4096, seekable=0)]
    streams = [t.cuda.Stream(), t.cuda.Stream()]
    bufs = []
    for i in range(2):
        n = inputs[i].size
        bufs.append((t.from_numpy(frames[i]).cuda(), t.empty(n, dtype=t.uint8, device="cuda"),
                     t.empty(dev.scratch_size(n, 65536), dtype=t.uint8, device="cuda"),
                     t.zeros(1, dtype=t.int64, device="cuda")))
    t.cuda.synchronize()
    for rep in range(3):
        for i in (0, 1):
            src, out, scr, res = bufs[i]
            out.fill_(0)
        t.cuda.synchronize()
        for i in (0, 1):
            src, out, scr, res = bufs[i]
            assert dev.enqueue(src.data_ptr(), frames[i].size, out.data_ptr(), inputs[i].size, dopts(1), scr, res,
                               stream=streams[i]) == 0
        for i in (0, 1):
            streams[i].synchronize()
            src, out, scr, res = bufs[i]
            assert int(res.item()) == inputs[i].size
            assert np.array_equal(out.cpu().numpy(), inputs[i]), (rep, i)


@pytest.mark.gpu
def test_graph_capture_and_replay(dev, prod):
    """Captured once without a dictionary, replayed on new frames of the same size (random bytes make RAW blocks,
    so the frame size depends on the length only) and on a damaged one."""
    t = dev.torch
    n = 3 << 20 | 12345
    frames = [(d, prod.compress(d, level=2, block_size=65536, checksum=1, seekable=1))
              for d in (np.random.default_rng(s).integers(0, 256, n, dtype=np.uint8) for s in (61, 62, 63))]
    m = frames[0][1].size
    assert all(f.size == m for _, f in frames)
    src = t.empty(m, dtype=t.uint8, device="cuda")
    out = t.empty(n, dtype=t.uint8, device="cuda")
    scr = t.empty(dev.scratch_size(n, 65536), dtype=t.uint8, device="cuda")
    res = t.zeros(1, dtype=t.int64, device="cuda")
    src.copy_(t.from_numpy(frames[0][1]))
    s = t.cuda.Stream()
    s.wait_stream(t.cuda.current_stream())
    with t.cuda.stream(s):  # warm-up outside the capture
        assert dev.enqueue(src.data_ptr(), m, out.data_ptr(), n, dopts(1), scr, res,
                           stream=t.cuda.current_stream()) == 0
    t.cuda.current_stream().wait_stream(s)
    t.cuda.synchronize()
    assert int(res.item()) == n
    g = t.cuda.CUDAGraph()
    with t.cuda.graph(g):
        assert dev.enqueue(src.data_ptr(), m, out.data_ptr(), n, dopts(1), scr, res,
                           stream=t.cuda.current_stream()) == 0
    for data, f in frames[1:]:
        src.copy_(t.from_numpy(f))
        res.fill_(0)
        out.fill_(0)
        g.replay()
        t.cuda.synchronize()
        assert int(res.item()) == n and np.array_equal(out.cpu().numpy(), data)
    bad = frames[0][1].copy()
    bad[HDR + 5000] ^= 0xFF  # a RAW payload byte: the block checksum fails
    src.copy_(t.from_numpy(bad))
    g.replay()
    t.cuda.synchronize()
    assert int(res.item()) == prod.decompress(bad, n, checksum=1)[0] == -7


@pytest.mark.gpu
def test_launch_count(dev, prod):
    d, h = next(iter(golden_dicts().values()))
    data = make_case("text", 300000)
    frame = prod.compress(data, level=3, block_size=65536, checksum=1, seekable=1)
    L = dev.L
    for bs, cks, want in ((65536, 0, 12 + 5 * 2), (65536, 1, 12 + 5 * 3), (4096, 0, 12 + 2), (2 << 20, 1, 12 + 30)):
        n0 = L.zxc_b200_launch_count()
        r, _ = dev.run(frame, data.size, cks, bs=bs)
        assert r == (data.size if bs >= 65536 else MEMORY)
        assert L.zxc_b200_launch_count() - n0 == want, (bs, cks)
    fd = prod.compress(data, level=6, block_size=4096, dict=d, dict_huf=h)
    n0 = L.zxc_b200_launch_count()
    assert dev.run(fd, data.size, 0, d, h)[0] == data.size
    assert L.zxc_b200_launch_count() - n0 == 12 + 2


@pytest.mark.gpu
def test_limits(dev, prod):
    """The call's own limits give ZXC_ERROR_MEMORY: blocks larger than the scratch was sized for, more blocks than the
    job table holds, and a scratch below the minimum (decided on the host)."""
    t = dev.torch
    data = make_case("text", 200000)
    frame = prod.compress(data, level=3, block_size=65536)
    assert dev.run(frame, data.size, bs=32768)[0] == MEMORY
    assert dev.run(frame, data.size, bs=65536)[0] == data.size
    # 40 one-byte blocks into 40 bytes: the table holds ceil(40 / 4096) + 2 = 3 entries
    tiny = np.frombuffer(b"abcdefghij" * 4, np.uint8)
    blocks = [prod.compress(tiny[i:i + 1], level=1, block_size=4096).tobytes() for i in range(tiny.size)]
    fr = np.frombuffer(blocks[0][:16] + b"".join(b[16:-20] for b in blocks) + blocks[0][-20:-12] +
                       struct.pack("<QI", tiny.size, 0), np.uint8)
    assert prod.decompress(fr, tiny.size)[0] == tiny.size
    assert dev.run(fr, tiny.size)[0] == MEMORY
    r, out = dev.run(fr, tiny.size * 4096)  # a larger capacity gives a larger table
    assert r == tiny.size and out.tobytes() == tiny.tobytes()
    src = t.from_numpy(frame).cuda()
    need = dev.scratch_size(data.size, 4096)
    scr = t.empty(need, dtype=t.uint8, device="cuda")
    out = t.empty(data.size, dtype=t.uint8, device="cuda")
    res = t.zeros(1, dtype=t.int64, device="cuda")
    assert dev.enqueue(src.data_ptr(), frame.size, out.data_ptr(), data.size, None, scr, res,
                       scratch_size=need - 1) == MEMORY
    assert dev.scratch_size(data.size, 5000) == 0


@pytest.mark.gpu
def test_python_decompress_frame(prod):
    import torch
    from zxc_b200 import device
    data = zc.silesia_shaped(9 << 20, seed=71)
    src = torch.from_numpy(data).cuda()
    s = torch.cuda.Stream()
    f = device.compress(src, level=3, block_size=65536, checksum=True, seekable=True, stream=s)
    out = device.decompress_frame(f.frame, checksum=True, stream=s)
    assert torch.equal(out, src)
    host = prod.compress(data[:500000], level=6, block_size=4096, checksum=1)
    t = torch.from_numpy(host).cuda()
    assert np.array_equal(device.decompress_frame(t).cpu().numpy(), data[:500000])
    assert device.decompress_frame(t, capacity=600000, checksum=True).numel() == 500000
    with pytest.raises(device.ZxcError) as e:
        device.decompress_frame(t, capacity=499999)
    assert e.value.code == DST_TOO_SMALL
    bad = t.clone()
    bad[0] ^= 1
    with pytest.raises(device.ZxcError) as e:
        device.decompress_frame(bad, capacity=500000)
    assert e.value.code == -4
    d, h = next(iter(golden_dicts().values()))
    fd = torch.from_numpy(prod.compress(data[:100000], level=6, block_size=4096, dict=d, dict_huf=h)).cuda()
    assert np.array_equal(device.decompress_frame(fd, dict=d, dict_huf=h).cpu().numpy(), data[:100000])
    with pytest.raises(device.ZxcError) as e:
        device.decompress_frame(fd)
    assert e.value.code == -15  # DICT_REQUIRED
    huge = t.clone()
    huge[-12:-4] = torch.tensor(list((1 << 40).to_bytes(8, "little")), dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):  # a footer past what the frame can hold is not trusted for the allocation
        device.decompress_frame(huge)
    with pytest.raises(device.ZxcError) as e:  # with a capacity, the call decides as zxc_decompress does
        device.decompress_frame(huge, capacity=500000)
    assert e.value.code == prod.decompress(huge.cpu().numpy(), 500000)[0]
    e0 = device.compress(torch.empty(0, dtype=torch.uint8, device="cuda"))
    assert device.decompress_frame(e0.frame).numel() == 0
