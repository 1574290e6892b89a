"""zxc_b200_seekable_device_*: byte ranges of a seekable frame in HBM, planned, decoded and judged on the device.

The oracle for every result and byte is this library's zxc_seekable_decompress_range on a handle opened on the same
bytes with the same dictionary (pinned to the reference by test_decode_gpu.py); where the reference library is built
and the frame is valid, it is compared as well."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

import zxc_corpus as zc
import zxc_ctypes as z
from conftest import has_cuda
from test_oracle import G, INVALID, VALID, golden_dicts, make_case

NULL_INPUT, SRC_SMALL, DST_TOO_SMALL, MEMORY, NO_DEVICE = -12, -3, -2, -1, -100
DICT_REQUIRED, DICT_MISMATCH, DICT_BIG = -15, -16, -17
LAUNCHES = 8
U64 = 1 << 64


def bind(L):
    L.zxc_b200_seekable_device_open.restype = C.c_void_p
    L.zxc_b200_seekable_device_open.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
    L.zxc_b200_seekable_device_set_dict.restype = C.c_int
    L.zxc_b200_seekable_device_set_dict.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.zxc_b200_seekable_device_num_blocks.restype = C.c_uint32
    L.zxc_b200_seekable_device_num_blocks.argtypes = [C.c_void_p]
    L.zxc_b200_seekable_device_decompressed_size.restype = C.c_uint64
    L.zxc_b200_seekable_device_decompressed_size.argtypes = [C.c_void_p]
    L.zxc_b200_seekable_device_block_size.restype = C.c_uint32
    L.zxc_b200_seekable_device_block_size.argtypes = [C.c_void_p]
    L.zxc_b200_seekable_device_scratch_size.restype = C.c_size_t
    L.zxc_b200_seekable_device_scratch_size.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64]
    L.zxc_b200_seekable_device_decompress_ranges.restype = C.c_int
    L.zxc_b200_seekable_device_decompress_ranges.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                                             C.c_uint64, C.c_void_p, C.c_size_t, C.c_void_p,
                                                             C.c_void_p]
    L.zxc_b200_seekable_device_free.restype = None
    L.zxc_b200_seekable_device_free.argtypes = [C.c_void_p]
    L.zxc_b200_launch_count.restype = C.c_uint64
    return L


def test_host_verdicts_without_a_device(prod):
    """Without a device: open gives NULL, the size query 0, and the codes that need no device come first."""
    if has_cuda():
        pytest.skip("only meaningful without a GPU")
    L = bind(prod.lib)
    frame = np.fromfile(os.path.join(G, "valid", "seekable_4blocks.zxc"), np.uint8)
    assert not L.zxc_b200_seekable_device_open(frame.ctypes.data, frame.size, None)
    assert not L.zxc_b200_seekable_device_open(None, 100, None)
    assert L.zxc_b200_seekable_device_scratch_size(None, 10, 1 << 20) == 0
    fake = 1 << 40  # never dereferenced
    dr = L.zxc_b200_seekable_device_decompress_ranges
    assert dr(None, fake, 1, fake, 100, fake, 1 << 20, fake, None) == NULL_INPUT
    assert dr(None, None, 0, None, 0, None, 0, None, None) == NULL_INPUT
    assert L.zxc_b200_seekable_device_set_dict(None, b"abc", 3, None) == NULL_INPUT
    assert L.zxc_b200_seekable_device_num_blocks(None) == 0
    assert L.zxc_b200_seekable_device_decompressed_size(None) == 0
    assert L.zxc_b200_seekable_device_block_size(None) == 0
    L.zxc_b200_seekable_device_free(None)


def test_python_argument_checks():
    """SeekableFrame rejects what the range call cannot write into, before anything is enqueued (no device needed)"""
    import gc
    import sys
    import torch
    from zxc_b200 import device
    cuda0 = torch.device("cuda", 0)
    with pytest.raises(ValueError, match="uint8"):
        device._check_out(torch.zeros(8, dtype=torch.float32), cuda0)
    with pytest.raises(ValueError, match="contiguous"):
        device._check_out(torch.zeros((4, 4), dtype=torch.uint8)[:, 0], cuda0)
    with pytest.raises(ValueError, match="device"):
        device._check_out(torch.zeros(8, dtype=torch.uint8), cuda0)
    # a rejected frame leaves an object whose finaliser runs cleanly
    seen = []
    old, sys.unraisablehook = sys.unraisablehook, seen.append
    try:
        with pytest.raises(ValueError, match="frame"):
            device.SeekableFrame(torch.zeros(64, dtype=torch.uint8))
        gc.collect()
    finally:
        sys.unraisablehook = old
    assert not seen, [str(u.exc_value) for u in seen]


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
class Dev:
    def __init__(self, prod):
        import torch
        self.t = torch
        self.L = bind(prod.lib)

    def open(self, frame, src_off=0):
        """-> (handle or None, the source tensor); the frame ends at the end of its tensor"""
        t = self.t
        frame = np.asarray(frame, np.uint8)
        src = t.empty(src_off + max(frame.size, 1), dtype=t.uint8, device="cuda")
        if frame.size:
            src[src_off:].copy_(t.from_numpy(frame.copy()))
        h = self.L.zxc_b200_seekable_device_open(src.data_ptr() + src_off, frame.size, None)
        return h, src

    def set_dict(self, h, d, huf=None):
        return self.L.zxc_b200_seekable_device_set_dict(h, d, len(d), huf)

    def ranges(self, rs):
        a = np.array([[o % U64, n % U64, d % U64] for o, n, d in rs], np.uint64).reshape(-1, 3)
        return self.t.from_numpy(a.view(np.int64)).cuda()

    def scratch(self, h, n, max_bytes, guard=0, fill=0):
        ss = int(self.L.zxc_b200_seekable_device_scratch_size(h, n, max_bytes))
        assert ss > 0
        return self.t.full((ss + 2 * guard,), fill, dtype=self.t.uint8, device="cuda"), ss

    def call(self, h, d_ranges, n, dst_ptr, cap, scr_ptr, ss, res, stream=None):
        return self.L.zxc_b200_seekable_device_decompress_ranges(
            h, d_ranges.data_ptr(), n, dst_ptr, cap, scr_ptr, ss, res.data_ptr(),
            stream.cuda_stream if stream is not None else None)

    def run(self, h, rs, cap, null_dst=False, max_bytes=None):
        """-> (results, dst bytes as numpy)"""
        t = self.t
        n = len(rs)
        if max_bytes is None:
            max_bytes = sum(min(r[1], cap) for r in rs)
        scr, ss = self.scratch(h, n, max_bytes)
        dst = t.zeros(max(cap, 1), dtype=t.uint8, device="cuda")
        res = t.full((n,), 12345, dtype=t.int64, device="cuda")
        d_ranges = self.ranges(rs)
        assert self.call(h, d_ranges, n, None if null_dst else dst.data_ptr(), cap, scr.data_ptr(), ss, res) == 0
        t.cuda.synchronize()
        return res.cpu().tolist(), dst.cpu().numpy()


@pytest.fixture(scope="module")
def dev(prod):
    return Dev(prod)


def _ref():
    return z.ZxcLib(z.REF_SO) if z.have_ref() else None


def host_ranges(lib, frame, rs, cap, d=None, huf=None, null_dst=False):
    """zxc_seekable_decompress_range per range, with the capacity the device call gives it -> [(result, bytes)]"""
    fb = bytes(np.asarray(frame, np.uint8).tobytes())
    h = lib.zxc_seekable_open(fb, len(fb))
    assert h
    if d is not None:
        assert lib.zxc_seekable_set_dict(h, d, len(d), huf) == 0
    total = int(lib.zxc_seekable_get_decompressed_size(h))
    out = []
    for off, n, doff in rs:
        cap_i = 0 if doff > cap else cap - doff
        buf = np.zeros(max(n if n <= total else 1, 1), np.uint8)
        r = lib.zxc_seekable_decompress_range(h, None if null_dst else buf.ctypes.data, cap_i, off % U64, n % U64)
        out.append((r, buf[:r].copy() if r > 0 else None))
    lib.zxc_seekable_free(h)
    return out


def same(dev, prod, frame, rs, cap, d=None, huf=None, ref=None, what=None, null_dst=False, h=None):
    """the device's results and bytes equal zxc_seekable_decompress_range's (and the reference's, when given)"""
    own = h is None
    if own:
        h, src = dev.open(frame)
        assert h, what
        if d is not None:
            assert dev.set_dict(h, d, huf) == 0
    res, dst = dev.run(h, rs, cap, null_dst=null_dst)
    if own:
        dev.L.zxc_b200_seekable_device_free(h)
    want = host_ranges(prod.lib, frame, rs, cap, d, huf, null_dst)
    rw = host_ranges(ref.lib, frame, rs, cap, d, huf, null_dst) if ref is not None else None
    for i, ((off, n, doff), r, (r0, o0)) in enumerate(zip(rs, res, want)):
        assert r == r0, (what, i, off, n, doff, z.ERR.get(r, r), z.ERR.get(r0, r0))
        if r0 > 0:
            assert np.array_equal(dst[doff:doff + n], o0), (what, i, off, n, doff)
        if rw is not None:
            assert rw[i][0] == r0, (what, i, "reference", rw[i][0], r0)
            if r0 > 0:
                assert np.array_equal(rw[i][1], o0), (what, i, "reference bytes")
    return res


def packed(rs):
    """lay ranges (offset, len) out back to back, dst_off 1..15 apart"""
    out, p = [], 0
    for k, (o, n) in enumerate(rs):
        p += k % 16
        out.append((o, n, p))
        p += n
    return out, p


def standard_ranges(total, bs, seed):
    rng = np.random.default_rng(seed)
    nb = (total + bs - 1) // bs
    rs = [(5, 100), (bs - 50, 100), (bs, bs), (0, bs * min(2, nb - 1) or total), (0, total),
          ((nb - 1) * bs - 7, total - (nb - 1) * bs + 7), (total - 1, 1), (3, 0), (bs + 1, bs - 2)]
    rs += [(bs + int(x), 300) for x in rng.integers(0, bs - 300, 12)]  # many on one block
    for _ in range(20):
        o = int(rng.integers(0, total))
        rs.append((o, int(rng.integers(0, min(total - o, 3 * bs) + 1))))
    return packed([(o, n) for o, n in rs if 0 <= o and n >= 0 and o + n <= total])


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, 2, 3, 4, 5, 6, 7])
def test_valid_frames(dev, prod, level):
    ref = _ref()
    for bs in (4096, 65536, 2 << 20):
        data = make_case("silesia", 3 * bs + 12345)
        for cks in (0, 1):
            frame = prod.compress(data, level=level, block_size=bs, checksum=cks, seekable=1)
            rs, cap = standard_ranges(data.size, bs, level * 10 + cks)
            res = same(dev, prod, frame, rs, cap, ref=ref, what=(level, bs, cks))
            assert res == [n for _, n, _ in rs]


@pytest.mark.gpu
def test_argument_verdicts(dev, prod):
    data = make_case("text", 300000)
    frame = prod.compress(data, level=3, block_size=65536, checksum=1, seekable=1)
    n = data.size
    cap = 200000
    rs = [(n - 10, 11, 0), (n, 1, 0), (U64 - 10, 100, 0), (U64 - 1, 2, 0), (1, U64 - 1, 0),  # SRC_TOO_SMALL
          (0, 100, cap - 100), (0, 101, cap - 100), (0, 1, cap), (0, 0, cap + 5), (0, 1, cap + 5),  # near cap
          (70000, 65536, 1000), (0, 0, 0)]
    res = same(dev, prod, frame, rs, cap)  # the reference does not check offset + len for wrapping
    assert res == [SRC_SMALL] * 4 + [DST_TOO_SMALL, 100, DST_TOO_SMALL, DST_TOO_SMALL, 0, DST_TOO_SMALL, 65536, 0]
    # a NULL d_dst, with zero and non-zero lengths
    res = same(dev, prod, frame, [(0, 0, 0), (5, 10, 0), (n, 5, 0)], cap, null_dst=True)
    assert res == [0, NULL_INPUT, NULL_INPUT]


@pytest.mark.gpu
def test_host_decided_codes(dev, prod):
    t = dev.t
    L = dev.L
    data = make_case("text", 100000)
    frame = prod.compress(data, level=3, block_size=4096, seekable=1)
    h, src = dev.open(frame)
    assert h
    assert L.zxc_b200_seekable_device_num_blocks(h) == 25
    assert L.zxc_b200_seekable_device_decompressed_size(h) == data.size
    assert L.zxc_b200_seekable_device_block_size(h) == 4096
    scr, ss = dev.scratch(h, 4, 0)
    res = t.zeros(4, dtype=t.int64, device="cuda")
    rr = dev.ranges([(0, 10, 0)] * 4)
    dst = t.zeros(100, dtype=t.uint8, device="cuda")
    dr = L.zxc_b200_seekable_device_decompress_ranges
    assert dr(None, rr.data_ptr(), 4, dst.data_ptr(), 100, scr.data_ptr(), ss, res.data_ptr(), None) == NULL_INPUT
    assert dr(h, None, 4, dst.data_ptr(), 100, scr.data_ptr(), ss, res.data_ptr(), None) == NULL_INPUT
    assert dr(h, rr.data_ptr(), 4, dst.data_ptr(), 100, None, ss, res.data_ptr(), None) == NULL_INPUT
    assert dr(h, rr.data_ptr(), 4, dst.data_ptr(), 100, scr.data_ptr(), ss, None, None) == NULL_INPUT
    assert dr(h, rr.data_ptr(), 4, dst.data_ptr(), 100, scr.data_ptr(), ss - 1, res.data_ptr(), None) == MEMORY
    n0 = L.zxc_b200_launch_count()
    assert dr(h, None, 0, None, 0, None, 0, None, None) == 0
    assert L.zxc_b200_launch_count() == n0
    assert dr(h, rr.data_ptr(), 4, dst.data_ptr(), 100, scr.data_ptr(), ss, res.data_ptr(), None) == 0
    t.cuda.synchronize()
    assert res.tolist() == [10] * 4 and dst[:10].cpu().numpy().tobytes() == data[:10].tobytes()
    L.zxc_b200_seekable_device_free(h)


@pytest.mark.gpu
def test_dictionaries(dev, prod):
    ref = _ref()
    # the golden seekable dictionary frame
    frame = np.fromfile(os.path.join(G, "valid", "dict_seekable_l7.zxc"), np.uint8)
    exp = np.frombuffer(open(os.path.join(G, "valid", "dict_seekable_l7.expected"), "rb").read(), np.uint8)
    did = int.from_bytes(frame[7:11].tobytes(), "little")
    d, huf = golden_dicts()[did]
    bs = 1 << int(frame[5])
    rs, cap = standard_ranges(exp.size, bs, 3)
    assert same(dev, prod, frame, rs, cap, d, huf, ref=ref) == [n for _, n, _ in rs]
    h, src = dev.open(frame)
    res, _ = dev.run(h, rs, cap)
    assert all(r == (0 if n == 0 else DICT_REQUIRED) for r, (_, n, _) in zip(res, rs))
    dev.L.zxc_b200_seekable_device_free(h)
    # trained and plain dictionaries, with and without a table
    data = make_case("text", 150000)
    for dd, hh in golden_dicts().values():
        for table in (None, hh):
            for bs in (4096, 65536):
                frame = prod.compress(data, level=6, block_size=bs, checksum=1, seekable=1, dict=dd, dict_huf=table)
                rs, cap = standard_ranges(data.size, bs, 5)
                assert same(dev, prod, frame, rs, cap, dd, table, ref=ref) == [n for _, n, _ in rs]
    # a frame with no dictionary id decodes with or without one set
    plain = prod.compress(data, level=3, block_size=4096, seekable=1)
    same(dev, prod, plain, rs, cap, dd)


@pytest.mark.gpu
def test_set_dict_verdicts(dev, prod):
    """zxc_seekable_set_dict's verdicts, in its order; a rejected call changes nothing"""
    d, huf = next(iter(golden_dicts().values()))
    data = make_case("text", 50000)
    frame = prod.compress(data, level=5, block_size=4096, seekable=1, dict=d, dict_huf=huf)
    fb = frame.tobytes()
    hs = prod.lib.zxc_seekable_open(fb, len(fb))
    h, src = dev.open(frame)
    big = b"x" * 70000
    cases = [(None, 5, None), (d, 0, None), (big, len(big), None), (d[:-1], len(d) - 1, huf), (d, len(d), None),
             (d, len(d), huf)]
    for dd, n, hh in cases:
        want = prod.lib.zxc_seekable_set_dict(hs, dd, n, hh)
        assert dev.L.zxc_b200_seekable_device_set_dict(h, dd, n, hh) == want, (n, hh is None)
    assert dev.L.zxc_b200_seekable_device_set_dict(None, d, len(d), huf) == NULL_INPUT
    rs = [(100, 20000, 0)]
    assert dev.run(h, rs, 20000)[0] == [20000]
    for dd, n, hh in cases[:4]:  # rejected: the dictionary set before stays
        dev.L.zxc_b200_seekable_device_set_dict(h, dd, n, hh)
        res, out = dev.run(h, rs, 20000)
        assert res == [20000] and np.array_equal(out[:20000], data[100:20100])
    prod.lib.zxc_seekable_free(hs)
    dev.L.zxc_b200_seekable_device_free(h)


@pytest.mark.gpu
def test_open_parity(dev, prod):
    """open gives NULL exactly where zxc_seekable_open does: golden vectors, and forged SEK tables"""
    L = dev.L
    paths = [os.path.join(G, "valid", v + ".zxc") for v in VALID] + \
            [os.path.join(G, "invalid", v + ".zxc") for v in INVALID] + \
            sorted(glob.glob(os.path.join(G, "format", "*.zxc")))
    opened = 0
    for p in paths:
        frame = np.fromfile(p, np.uint8)
        hs = prod.lib.zxc_seekable_open(frame.ctypes.data, frame.size) if frame.size else None
        h, src = dev.open(frame)
        assert bool(h) == bool(hs), p
        if hs:
            assert L.zxc_b200_seekable_device_num_blocks(h) == prod.lib.zxc_seekable_get_num_blocks(hs)
            assert L.zxc_b200_seekable_device_decompressed_size(h) == prod.lib.zxc_seekable_get_decompressed_size(hs)
            total = int(prod.lib.zxc_seekable_get_decompressed_size(hs))
            did = int.from_bytes(frame[7:11].tobytes(), "little") if frame[6] & 0x40 else 0
            d, huf = golden_dicts().get(did, (None, None))
            if did == 0 or d is not None:
                same(dev, prod, frame, [(0, total, 0), (total // 3, total - total // 3, total)], 2 * total, d, huf,
                     what=p)
            prod.lib.zxc_seekable_free(hs)
            L.zxc_b200_seekable_device_free(h)
            opened += 1
    assert opened >= 3
    # forged SEK tables, as in test_decompress_device.py: the ranges decode at the table's offsets, like the host's
    data = zc.silesia_shaped(1 << 20, seed=7)[:200000]
    frame = prod.compress(data, level=1, block_size=4096, checksum=1, seekable=1)
    nb = (data.size + 4095) // 4096
    ent = frame.size - 12 - 4 * nb
    sizes = np.frombuffer(frame[ent:ent + 4 * nb].tobytes(), "<u4").copy()
    sw, mv, sh = sizes.copy(), sizes.copy(), sizes.copy()
    sw[[3, 4]] = sw[[4, 3]]
    mv[0] += 1
    mv[1] -= 1
    sh[-1] += 4
    rs, cap = standard_ranges(data.size, 4096, 9)
    for forged in (sw, mv, sh):
        f = frame.copy()
        f[ent:ent + 4 * nb] = np.frombuffer(forged.astype("<u4").tobytes(), np.uint8)
        hs = prod.lib.zxc_seekable_open(f.ctypes.data, f.size)
        h, src = dev.open(f)
        assert bool(h) == bool(hs)
        if hs:
            prod.lib.zxc_seekable_free(hs)
            same(dev, prod, f, rs, cap, h=h)
            L.zxc_b200_seekable_device_free(h)


def _mutants(frame, count, seed, lo, hi):
    rng = np.random.default_rng(seed)
    for _ in range(count):
        m = frame.copy()
        k = int(rng.integers(lo, hi))
        m[k] ^= np.uint8(int(rng.integers(1, 256)))
        yield k, m


@pytest.mark.gpu
def test_mutations(dev, prod):
    """seeded payload damage under an intact SEK table: every range's result equals the host call's"""
    d, huf = next(iter(golden_dicts().values()))
    data = zc.silesia_shaped(1 << 20, seed=5)[:90000]
    frames = [("lz", prod.compress(data, level=3, block_size=4096, checksum=1, seekable=1), None, None),
              ("huffman", prod.compress(make_case("text", 60000), level=6, block_size=4096, seekable=1), None, None),
              ("dict", prod.compress(make_case("text", 40000), level=6, block_size=4096, checksum=1, seekable=1,
                                     dict=d, dict_huf=huf), d, huf)]
    for name, frame, dd, hh in frames:
        total = int(prod.lib.zxc_get_decompressed_size(frame.ctypes.data, frame.size))
        nb = (total + 4095) // 4096
        rs, cap = standard_ranges(total, 4096, len(name))
        sek = frame.size - 12 - 4 * nb - 8 - 8  # the EOF block header
        for k, m in _mutants(frame, 40, len(name), 16, sek):
            same(dev, prod, m, rs, cap, dd, hh, what=(name, k))


@pytest.mark.gpu
def test_guard_regions(dev, prod):
    """nothing lands outside the ranges' spans (canaries before, between, behind) or the scratch, for every result"""
    t = dev.t
    data = make_case("silesia", 400001)
    for bs in (4096, 65536):
        frame = prod.compress(data, level=2, block_size=bs, checksum=1, seekable=1)
        good = frame
        bad = frame.copy()
        bad[16 + 3 * bs // 4] ^= 0x5A  # damage inside the first block's payload region
        for f in (good, bad):
            rs, p = standard_ranges(data.size, bs, 77)
            rs = [(o, n, dd + 7 * i) for i, (o, n, dd) in enumerate(rs)]  # gaps between the spans
            rs.append((data.size - 3, 5, 0))  # SRC_TOO_SMALL
            cap = p + 7 * len(rs)
            guard = 4096
            h, src = dev.open(f)
            scr, ss = dev.scratch(h, len(rs), cap, guard, 0x5A)
            dst = t.full((cap + 2 * guard,), 0xA5, dtype=t.uint8, device="cuda")
            res = t.zeros(len(rs), dtype=t.int64, device="cuda")
            assert dev.call(h, dev.ranges(rs), len(rs), dst.data_ptr() + guard, cap, scr.data_ptr() + guard, ss,
                            res) == 0
            t.cuda.synchronize()
            out = dst.cpu().numpy()
            mask = np.zeros(out.size, bool)
            for o, n, dd in rs:
                mask[guard + dd:guard + dd + n] = True
            assert (out[~mask] == 0xA5).all(), (bs, "written outside the spans")
            g = scr.cpu().numpy()
            assert (g[:guard] == 0x5A).all() and (g[guard + ss:] == 0x5A).all(), "written outside the scratch"
            want = host_ranges(prod.lib, f, rs, cap)
            assert res.tolist() == [r for r, _ in want]
            for (o, n, dd), (r0, o0) in zip(rs, want):
                if r0 > 0:
                    assert np.array_equal(out[guard + dd:guard + dd + n], o0)
            dev.L.zxc_b200_seekable_device_free(h)


@pytest.mark.gpu
def test_call_limit(dev, prod):
    """ranges past the job table the scratch holds get MEMORY in index order; the ones in front are right"""
    data = make_case("silesia", 40 * 4096)
    frame = prod.compress(data, level=1, block_size=4096, seekable=1)
    h, src = dev.open(frame)
    rs = packed([(0, 4 * 4096), (100, 10), (4096, 3 * 4096), (5, 0), (2 * 4096, 4 * 4096), (7, 100), (0, 4096)])[0]
    cap = rs[-1][2] + 4096
    # sized for 8 blocks' worth: ranges 0 and 2 take 4 + 3 whole blocks, range 4 needs 4 more
    res, out = dev.run(h, rs, cap, max_bytes=8 * 4096)
    assert res == [4 * 4096, 10, 3 * 4096, 0, MEMORY, MEMORY, MEMORY]
    for (o, n, dd), r in zip(rs, res):
        if r > 0:
            assert np.array_equal(out[dd:dd + n], data[o:o + n])
    res, out = dev.run(h, rs, cap, max_bytes=12 * 4096)
    assert res == [n for _, n, _ in rs]
    dev.L.zxc_b200_seekable_device_free(h)


@pytest.mark.gpu
def test_many_blocks_many_ranges(dev, prod):
    """about 250 000 blocks of 4 KiB and 100 000 random ranges in one call"""
    t = dev.t
    data = zc.silesia_shaped(4096 * 250000 + 777, seed=41)
    frame = prod.compress(data, level=1, block_size=4096, seekable=1)
    rng = np.random.default_rng(5)
    n = 100000
    lens = rng.integers(0, 3 * 4096, n)
    offs = (rng.random(n) * (data.size - lens)).astype(np.int64)
    dst_off = np.cumsum(lens) - lens
    cap = int(lens.sum())
    h, src = dev.open(frame)
    assert dev.L.zxc_b200_seekable_device_num_blocks(h) == 250001
    scr, ss = dev.scratch(h, n, cap)
    ranges = t.from_numpy(np.stack([offs, lens, dst_off], 1).astype(np.int64)).cuda()
    dst = t.empty(cap, dtype=t.uint8, device="cuda")
    res = t.zeros(n, dtype=t.int64, device="cuda")
    assert dev.call(h, ranges, n, dst.data_ptr(), cap, scr.data_ptr(), ss, res) == 0
    t.cuda.synchronize()
    assert np.array_equal(res.cpu().numpy(), lens)
    want = t.from_numpy(data).cuda()
    idx = t.from_numpy(np.repeat(offs - dst_off, lens) + np.arange(cap)).cuda()
    assert t.equal(dst, want[idx])
    dev.L.zxc_b200_seekable_device_free(h)


@pytest.mark.gpu
def test_two_handles_on_two_streams(dev, prod):
    t = dev.t
    inputs = [zc.silesia_shaped(6 << 20, seed=51), make_case("text", 5 << 20)]
    frames = [prod.compress(inputs[0], level=3, block_size=65536, checksum=1, seekable=1),
              prod.compress(inputs[1], level=6, block_size=4096, seekable=1)]
    streams = [t.cuda.Stream(), t.cuda.Stream()]
    state = []
    for i in range(2):
        h, src = dev.open(frames[i])
        rng = np.random.default_rng(i)
        rs = packed([(int(o), 20000) for o in rng.integers(0, inputs[i].size - 20000, 300)])[0]
        cap = rs[-1][2] + 20000
        scr, ss = dev.scratch(h, len(rs), cap)
        state.append((h, src, rs, dev.ranges(rs), scr, ss, t.zeros(cap, dtype=t.uint8, device="cuda"),
                      t.zeros(len(rs), dtype=t.int64, device="cuda"), cap))
    t.cuda.synchronize()
    for rep in range(3):
        for i in (0, 1):
            h, src, rs, rr, scr, ss, dst, res, cap = state[i]
            assert dev.call(h, rr, len(rs), dst.data_ptr(), cap, scr.data_ptr(), ss, res, stream=streams[i]) == 0
        for i in (0, 1):
            streams[i].synchronize()
            h, src, rs, rr, scr, ss, dst, res, cap = state[i]
            assert res.tolist() == [20000] * len(rs)
            out = dst.cpu().numpy()
            for o, n, dd in rs:
                assert np.array_equal(out[dd:dd + n], inputs[i][o:o + n]), (rep, i)
    for s in state:
        dev.L.zxc_b200_seekable_device_free(s[0])


@pytest.mark.gpu
def test_graph_capture_with_a_dictionary(dev, prod):
    """captured once with a dictionary set, replayed after rewriting d_ranges in place: equal to fresh calls"""
    t = dev.t
    d, huf = next(iter(golden_dicts().values()))
    data = make_case("text", 2 << 20)
    frame = prod.compress(data, level=6, block_size=65536, checksum=1, seekable=1, dict=d, dict_huf=huf)
    h, src = dev.open(frame)
    assert dev.set_dict(h, d, huf) == 0
    n, ln = 64, 10000
    cap = n * ln
    scr, ss = dev.scratch(h, n, cap)
    dst = t.zeros(cap, dtype=t.uint8, device="cuda")
    res = t.zeros(n, dtype=t.int64, device="cuda")

    def draw(seed):
        rng = np.random.default_rng(seed)
        return [(int(o), ln, k * ln) for k, o in enumerate(rng.integers(0, data.size - ln, n))]

    rr = dev.ranges(draw(1))
    s = t.cuda.Stream()
    s.wait_stream(t.cuda.current_stream())
    with t.cuda.stream(s):  # warm-up outside the capture
        assert dev.call(h, rr, n, dst.data_ptr(), cap, scr.data_ptr(), ss, res, stream=s) == 0
    t.cuda.current_stream().wait_stream(s)
    t.cuda.synchronize()
    g = t.cuda.CUDAGraph()
    with t.cuda.graph(g):
        assert dev.call(h, rr, n, dst.data_ptr(), cap, scr.data_ptr(), ss, res,
                        stream=t.cuda.current_stream()) == 0
    for seed in (2, 3, 4):
        rs = draw(seed)
        if seed == 4:
            rs[5] = (data.size - 5, ln, 5 * ln)  # SRC_TOO_SMALL
        rr.copy_(dev.ranges(rs))
        dst.zero_()
        res.zero_()
        g.replay()
        t.cuda.synchronize()
        got, out = res.tolist(), dst.cpu().numpy()
        fresh, fout = dev.run(h, rs, cap)
        assert got == fresh
        for (o, k, dd), r in zip(rs, got):
            if r > 0:
                assert np.array_equal(out[dd:dd + k], data[o:o + k]) and np.array_equal(fout[dd:dd + k], out[dd:dd + k])
    dev.L.zxc_b200_seekable_device_free(h)


@pytest.mark.gpu
def test_launch_count(dev, prod):
    d, huf = next(iter(golden_dicts().values()))
    data = make_case("text", 300000)
    L = dev.L
    for frame, dd in ((prod.compress(data, level=3, block_size=65536, checksum=1, seekable=1), None),
                      (prod.compress(data, level=6, block_size=4096, seekable=1, dict=d, dict_huf=huf), d)):
        h, src = dev.open(frame)
        if dd is not None:
            assert dev.set_dict(h, d, huf) == 0
        for rs in ([(0, 0, 0)], [(5, 10, 0)], [(0, data.size, 0)], packed([(k * 999, 5000) for k in range(200)])[0]):
            cap = max(dd + n for _, n, dd in rs) + 1
            n0 = L.zxc_b200_launch_count()
            dev.run(h, rs, cap)
            assert L.zxc_b200_launch_count() - n0 == LAUNCHES, len(rs)
        L.zxc_b200_seekable_device_free(h)


@pytest.mark.gpu
def test_python_seekable_frame(prod):
    import torch
    from zxc_b200 import device
    data = zc.silesia_shaped(3 << 20, seed=71)
    src = torch.from_numpy(data).cuda()
    f = device.compress(src, level=3, block_size=65536, checksum=True, seekable=True)
    whole = device.decompress_frame(f.frame)
    with device.SeekableFrame(f.frame) as sf:
        assert (sf.decompressed_size, sf.block_size, sf.n_blocks) == (data.size, 65536, 48)
        assert torch.equal(sf.read(12345, 200000), whole[12345:212345])
        assert sf.read(7, 0).numel() == 0
        offs = torch.tensor([0, 70000, 5, data.size - 9], dtype=torch.int64, device="cuda")
        lens = torch.tensor([100, 65536 * 2, 0, 9], dtype=torch.int64, device="cuda")
        out, res = sf.gather(offs, lens)
        torch.cuda.synchronize()
        assert res.tolist() == [100, 131072, 0, 9]
        assert torch.equal(out, torch.cat([whole[0:100], whole[70000:201072], whole[data.size - 9:]]))
        out2 = torch.empty(out.numel(), dtype=torch.uint8, device="cuda")
        s = torch.cuda.Stream()
        o2, res2 = sf.gather(offs, lens, out=out2, stream=s)
        s.synchronize()
        assert o2 is out2 and torch.equal(out2, out) and res2.tolist() == res.tolist()
        with pytest.raises(device.ZxcError) as e:
            sf.read(data.size - 5, 10)
        assert e.value.code == SRC_SMALL
        # an out the call cannot write into: rejected before anything is enqueued
        buf = torch.zeros((out.numel(), 2), dtype=torch.uint8, device="cuda")
        for bad in (buf[:, 0], torch.zeros(out.numel(), dtype=torch.int32, device="cuda"),
                    torch.zeros(out.numel(), dtype=torch.uint8)):
            with pytest.raises(ValueError):
                sf.gather(offs, lens, out=bad)
        assert (buf == 0).all()
        # inputs written on the current stream, gathered on another one
        s2 = torch.cuda.Stream()
        torch.cuda._sleep(50_000_000)
        offs2 = offs.clone().fill_(0)
        offs2.copy_(offs)
        o3, res3 = sf.gather(offs2, lens, stream=s2)
        del offs2
        s2.synchronize()
        assert torch.equal(o3, out) and res3.tolist() == res.tolist()
    with pytest.raises(ValueError):
        sf.n_blocks
    d, huf = next(iter(golden_dicts().values()))
    fd = torch.from_numpy(prod.compress(data[:100000], level=6, block_size=4096, seekable=1, dict=d, dict_huf=huf))
    fd = fd.cuda()
    with device.SeekableFrame(fd) as sf:
        with pytest.raises(device.ZxcError) as e:
            sf.read(0, 10)
        assert e.value.code == DICT_REQUIRED
    with device.SeekableFrame(fd, dict=d, dict_huf=huf) as sf:
        assert np.array_equal(sf.read(4000, 50000).cpu().numpy(), data[4000:54000])
    with pytest.raises(device.ZxcError) as e:
        device.SeekableFrame(fd, dict=d[:-1])
    assert e.value.code == DICT_MISMATCH
    plain = torch.from_numpy(prod.compress(data[:100000], level=3, block_size=4096)).cuda()
    with pytest.raises(ValueError):
        device.SeekableFrame(plain)
