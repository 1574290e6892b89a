"""zxc_b200_seekable_device_open_host: byte ranges of a seekable frame in page-locked host memory, decoded into HBM.

Every result and byte is checked against two oracles: this library's zxc_seekable_decompress_range, and the device
handle opened on an HBM copy of the same frame and called with the same d_ranges (each handle with a scratch from its
own size query).  Where the reference library is built and the frame is valid, it is compared as well."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

import zxc_corpus as zc
from conftest import has_cuda
from test_oracle import G, INVALID, VALID, golden_dicts, make_case
from test_seekable_device import Dev, _mutants, _ref, bind, host_ranges, packed, standard_ranges

NULL_INPUT, SRC_SMALL, MEMORY = -12, -3, -1
DICT_REQUIRED = -15
LAUNCHES = 9
U64 = 1 << 64


def bind_host(L):
    bind(L)
    L.zxc_b200_seekable_device_open_host.restype = C.c_void_p
    L.zxc_b200_seekable_device_open_host.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
    return L


def test_host_verdicts_without_a_device(prod):
    """Without a device: open_host gives NULL and the size query 0"""
    if has_cuda():
        pytest.skip("only meaningful without a GPU")
    L = bind_host(prod.lib)
    frame = np.fromfile(os.path.join(G, "valid", "seekable_4blocks.zxc"), np.uint8)
    assert not L.zxc_b200_seekable_device_open_host(frame.ctypes.data, frame.size, None)
    assert not L.zxc_b200_seekable_device_open_host(None, 100, None)
    assert not L.zxc_b200_seekable_device_open_host(frame.ctypes.data, 0, None)
    assert L.zxc_b200_seekable_device_scratch_size(None, 10, 1 << 20) == 0


def test_python_rejects_pageable_and_non_uint8():
    """SeekableFrame takes a CPU frame only in page-locked memory, and only uint8 (no device needed)"""
    import torch
    from zxc_b200 import device
    frame = torch.from_numpy(np.fromfile(os.path.join(G, "valid", "seekable_4blocks.zxc"), np.uint8))
    with pytest.raises(ValueError, match="pin_memory"):
        device.SeekableFrame(frame)
    with pytest.raises(ValueError, match="uint8"):
        device.SeekableFrame(frame.to(torch.int32))
    with pytest.raises(ValueError, match="uint8"):
        device.SeekableFrame(torch.zeros((8, 8), dtype=torch.uint8)[:, 0])


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
class Host(Dev):
    def __init__(self, prod):
        super().__init__(prod)
        bind_host(self.L)

    def open_host(self, frame, src_off=0):
        """-> (handle or None, the pinned buffer); the frame starts src_off bytes into its buffer and ends at its end"""
        t = self.t
        frame = np.asarray(frame, np.uint8)
        buf = t.zeros(src_off + max(frame.size, 1), dtype=t.uint8).pin_memory()
        buf.numpy()[src_off:src_off + frame.size] = frame
        h = self.L.zxc_b200_seekable_device_open_host(buf.data_ptr() + src_off, frame.size, None)
        return h, buf

    def run_on(self, h, d_ranges, n, cap, max_bytes):
        t = self.t
        scr, ss = self.scratch(h, n, max_bytes)
        dst = t.zeros(max(cap, 1), dtype=t.uint8, device="cuda")
        res = t.full((n,), 12345, dtype=t.int64, device="cuda")
        assert self.call(h, d_ranges, n, dst.data_ptr(), cap, scr.data_ptr(), ss, res) == 0
        t.cuda.synchronize()
        return res.cpu().tolist(), dst.cpu().numpy()


@pytest.fixture(scope="module")
def host(prod):
    return Host(prod)


def both(host, prod, frame, rs, cap, d=None, huf=None, ref=None, what=None, src_off=0, max_bytes=None):
    """the host handle's results and bytes equal zxc_seekable_decompress_range's, the device handle's on an HBM copy
    (same d_ranges), and the reference's when given -> results.  A scratch sized below the ranges' lengths (max_bytes)
    may give both handles MEMORY, which the host call has no twin of; those ranges are compared between the handles."""
    hh, buf = host.open_host(frame, src_off)
    hd, src = host.open(frame)
    assert hh and hd, what
    if d is not None:
        assert host.set_dict(hh, d, huf) == 0 and host.set_dict(hd, d, huf) == 0
    if max_bytes is None:
        max_bytes = sum(min(r[1], cap) for r in rs)
    rr = host.ranges(rs)
    res, dst = host.run_on(hh, rr, len(rs), cap, max_bytes)
    res_d, dst_d = host.run_on(hd, rr, len(rs), cap, max_bytes)
    host.L.zxc_b200_seekable_device_free(hh)
    host.L.zxc_b200_seekable_device_free(hd)
    assert np.array_equal(buf.numpy()[src_off:src_off + len(frame)], np.asarray(frame, np.uint8)), what
    want = host_ranges(prod.lib, frame, rs, cap, d, huf)
    rw = host_ranges(ref.lib, frame, rs, cap, d, huf) if ref is not None else None
    assert res == res_d, (what, res, res_d)
    for i, ((off, n, doff), r, (r0, o0)) in enumerate(zip(rs, res, want)):
        if r == MEMORY and max_bytes < sum(k for _, k, _ in rs):
            continue
        assert r == r0, (what, i, off, n, doff, r, r0)
        if r0 > 0:
            assert np.array_equal(dst[doff:doff + n], o0), (what, i, off, n, doff)
            assert np.array_equal(dst_d[doff:doff + n], o0), (what, i, "device handle")
        if rw is not None:
            assert rw[i][0] == r0, (what, i, "reference", rw[i][0], r0)
            if r0 > 0:
                assert np.array_equal(rw[i][1], o0), (what, i, "reference bytes")
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, 3, 5, 7])
def test_valid_frames(host, prod, level):
    ref = _ref()
    for bs in (4096, 65536, 2 << 20):
        data = make_case("silesia", 3 * bs + 12345)
        for cks in (0, 1):
            frame = prod.compress(data, level=level, block_size=bs, checksum=cks, seekable=1)
            rs, cap = standard_ranges(data.size, bs, level * 10 + cks)
            res = both(host, prod, frame, rs, cap, ref=ref, what=(level, bs, cks), src_off=(level + bs + cks) % 16)
            assert res == [n for _, n, _ in rs]


@pytest.mark.gpu
def test_open_parity(host, prod):
    """open_host gives NULL exactly where zxc_seekable_open does: golden vectors, and forged SEK tables"""
    L = host.L
    paths = [os.path.join(G, "valid", v + ".zxc") for v in VALID] + \
            [os.path.join(G, "invalid", v + ".zxc") for v in INVALID] + \
            sorted(glob.glob(os.path.join(G, "format", "*.zxc")))
    opened = 0
    for p in paths:
        frame = np.fromfile(p, np.uint8)
        hs = prod.lib.zxc_seekable_open(frame.ctypes.data, frame.size) if frame.size else None
        h, buf = host.open_host(frame, 3)
        assert bool(h) == bool(hs), p
        if hs:
            assert L.zxc_b200_seekable_device_num_blocks(h) == prod.lib.zxc_seekable_get_num_blocks(hs)
            assert L.zxc_b200_seekable_device_decompressed_size(h) == prod.lib.zxc_seekable_get_decompressed_size(hs)
            total = int(prod.lib.zxc_seekable_get_decompressed_size(hs))
            L.zxc_b200_seekable_device_free(h)
            did = int.from_bytes(frame[7:11].tobytes(), "little") if frame[6] & 0x40 else 0
            d, huf = golden_dicts().get(did, (None, None))
            if did == 0 or d is not None:
                both(host, prod, frame, [(0, total, 0), (total // 3, total - total // 3, total)], 2 * total, d, huf,
                     what=p)
            prod.lib.zxc_seekable_free(hs)
            opened += 1
    assert opened >= 3
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
        h, buf = host.open_host(f, 7)
        assert bool(h) == bool(hs)
        if h:
            L.zxc_b200_seekable_device_free(h)
        if hs:
            prod.lib.zxc_seekable_free(hs)
            both(host, prod, f, rs, cap, what="forged")


@pytest.mark.gpu
def test_dictionaries(host, prod):
    ref = _ref()
    frame = np.fromfile(os.path.join(G, "valid", "dict_seekable_l7.zxc"), np.uint8)
    exp = np.frombuffer(open(os.path.join(G, "valid", "dict_seekable_l7.expected"), "rb").read(), np.uint8)
    did = int.from_bytes(frame[7:11].tobytes(), "little")
    d, huf = golden_dicts()[did]
    bs = 1 << int(frame[5])
    rs, cap = standard_ranges(exp.size, bs, 3)
    assert both(host, prod, frame, rs, cap, d, huf, ref=ref) == [n for _, n, _ in rs]
    # DICT_REQUIRED before set_dict
    assert both(host, prod, frame, rs, cap) == [0 if n == 0 else DICT_REQUIRED for _, n, _ in rs]
    data = make_case("text", 150000)
    for dd, hh in golden_dicts().values():
        for table in (None, hh):
            for bs in (4096, 65536):
                frame = prod.compress(data, level=6, block_size=bs, checksum=1, seekable=1, dict=dd, dict_huf=table)
                rs, cap = standard_ranges(data.size, bs, 5)
                assert both(host, prod, frame, rs, cap, dd, table, ref=ref, src_off=bs % 13) == [n for _, n, _ in rs]


@pytest.mark.gpu
def test_mutations(host, prod):
    """seeded payload damage under an intact SEK table: the same verdicts as the host call and the device handle"""
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
        sek = frame.size - 12 - 4 * nb - 8 - 8
        for k, m in _mutants(frame, 25, len(name) + 100, 16, sek):
            both(host, prod, m, rs, cap, dd, hh, what=(name, k), src_off=k % 16)


@pytest.mark.gpu
def test_call_limit(host, prod):
    """a scratch sized for fewer bytes: MEMORY for a suffix of ranges only, and the admitted prefix exact"""
    data = make_case("silesia", 40 * 4096)
    frame = prod.compress(data, level=1, block_size=4096, seekable=1)
    rs = packed([(0, 4 * 4096), (100, 10), (4096, 3 * 4096), (5, 0), (2 * 4096, 4 * 4096), (7, 100), (0, 4096)])[0]
    cap = rs[-1][2] + 4096
    res = both(host, prod, frame, rs, cap, max_bytes=8 * 4096)  # the device handle gives the same MEMORY
    assert res == [4 * 4096, 10, 3 * 4096, 0, MEMORY, MEMORY, MEMORY]
    assert both(host, prod, frame, rs, cap, max_bytes=12 * 4096) == [n for _, n, _ in rs]
    # a scratch sized for (n, B) admits every call within it, whatever the frame's block sizes: ranges that each
    # touch three blocks for few bytes, on a frame of incompressible blocks
    rnd = np.random.default_rng(3).integers(0, 256, 64 * 4096, dtype=np.uint8)
    frame = prod.compress(rnd, level=1, block_size=4096, seekable=1)
    rs = packed([(k * 4096 - 1, 4098) for k in range(1, 60, 2)])[0]
    cap = rs[-1][2] + 4098
    assert both(host, prod, frame, rs, cap) == [4098] * len(rs)
    # ranges that each cover the short last block whole: one job per range for fewer than block_size bytes
    data = make_case("silesia", 10 * 4096 + 100)
    frame = prod.compress(data, level=1, block_size=4096, seekable=1)
    hh, buf = host.open_host(frame, 1)
    rs = packed([(10 * 4096, 100)] * 40 + [(0, 4096)])[0]
    cap = rs[-1][2] + 4096
    res, dst = host.run_on(hh, host.ranges(rs), len(rs), cap, sum(n for _, n, _ in rs))
    host.L.zxc_b200_seekable_device_free(hh)
    assert res == [n for _, n, _ in rs]
    for o, n, dd in rs:
        assert np.array_equal(dst[dd:dd + n], data[o:o + n])


@pytest.mark.gpu
def test_pinned_sources(host, prod):
    """pin_memory() and cudaHostRegister memory open, at any offset; pageable numpy memory gives NULL"""
    t = host.t
    data = make_case("silesia", 300001)
    frame = prod.compress(data, level=3, block_size=65536, checksum=1, seekable=1)
    rs, cap = standard_ranges(data.size, 65536, 11)
    for off in (0, 1, 7, 15):
        both(host, prod, frame, rs, cap, what=("pin_memory", off), src_off=off)
    pageable = np.zeros(frame.size + 64, np.uint8)
    pageable[5:5 + frame.size] = frame
    assert not host.L.zxc_b200_seekable_device_open_host(pageable.ctypes.data + 5, frame.size, None)
    # cudaHostRegister of the numpy buffer, through torch's runtime binding
    cudart = t.cuda.cudart()
    assert int(cudart.cudaHostRegister(pageable.ctypes.data, pageable.nbytes, 0)) == 0
    try:
        h = host.L.zxc_b200_seekable_device_open_host(pageable.ctypes.data + 5, frame.size, None)
        assert h
        res, dst = host.run_on(h, host.ranges(rs), len(rs), cap, sum(n for _, n, _ in rs))
        host.L.zxc_b200_seekable_device_free(h)
        assert res == [n for _, n, _ in rs]
        for o, n, dd in rs:
            assert np.array_equal(dst[dd:dd + n], data[o:o + n])
    finally:
        assert int(cudart.cudaHostUnregister(pageable.ctypes.data)) == 0
    assert not host.L.zxc_b200_seekable_device_open_host(pageable.ctypes.data + 5, frame.size, None)


@pytest.mark.gpu
def test_guard_regions(host, prod):
    """nothing lands outside the ranges' spans or the scratch, and the host frame is unchanged, for every result"""
    t = host.t
    data = make_case("silesia", 400001)
    for bs in (4096, 65536):
        frame = prod.compress(data, level=2, block_size=bs, checksum=1, seekable=1)
        bad = frame.copy()
        bad[16 + 3 * bs // 4] ^= 0x5A
        for f in (frame, bad):
            rs, p = standard_ranges(data.size, bs, 77)
            rs = [(o, n, dd + 7 * i) for i, (o, n, dd) in enumerate(rs)]
            rs.append((data.size - 3, 5, 0))
            cap = p + 7 * len(rs)
            guard = 4096
            h, buf = host.open_host(f, 9)
            before = buf.numpy().copy()
            scr, ss = host.scratch(h, len(rs), cap, guard, 0x5A)
            dst = t.full((cap + 2 * guard,), 0xA5, dtype=t.uint8, device="cuda")
            res = t.zeros(len(rs), dtype=t.int64, device="cuda")
            assert host.call(h, host.ranges(rs), len(rs), dst.data_ptr() + guard, cap, scr.data_ptr() + guard, ss,
                             res) == 0
            t.cuda.synchronize()
            out = dst.cpu().numpy()
            mask = np.zeros(out.size, bool)
            for o, n, dd in rs:
                mask[guard + dd:guard + dd + n] = True
            assert (out[~mask] == 0xA5).all(), (bs, "written outside the spans")
            g = scr.cpu().numpy()
            assert (g[:guard] == 0x5A).all() and (g[guard + ss:] == 0x5A).all(), "written outside the scratch"
            assert np.array_equal(buf.numpy(), before), "the host frame changed"
            want = host_ranges(prod.lib, f, rs, cap)
            assert res.tolist() == [r for r, _ in want]
            for (o, n, dd), (r0, o0) in zip(rs, want):
                if r0 > 0:
                    assert np.array_equal(out[guard + dd:guard + dd + n], o0)
            host.L.zxc_b200_seekable_device_free(h)


@pytest.mark.gpu
def test_two_handles_on_one_host_frame(host, prod):
    """two handles on one pinned frame, called on two streams at once"""
    t = host.t
    data = zc.silesia_shaped(6 << 20, seed=51)
    frame = prod.compress(data, level=3, block_size=65536, checksum=1, seekable=1)
    buf = t.from_numpy(frame.copy()).pin_memory()
    streams = [t.cuda.Stream(), t.cuda.Stream()]
    state = []
    for i in range(2):
        h = host.L.zxc_b200_seekable_device_open_host(buf.data_ptr(), frame.size, None)
        assert h
        rng = np.random.default_rng(i)
        rs = packed([(int(o), 20000) for o in rng.integers(0, data.size - 20000, 300)])[0]
        cap = rs[-1][2] + 20000
        scr, ss = host.scratch(h, len(rs), cap)
        state.append((h, rs, host.ranges(rs), scr, ss, t.zeros(cap, dtype=t.uint8, device="cuda"),
                      t.zeros(len(rs), dtype=t.int64, device="cuda"), cap))
    t.cuda.synchronize()
    for rep in range(3):
        for i in (0, 1):
            h, rs, rr, scr, ss, dst, res, cap = state[i]
            assert host.call(h, rr, len(rs), dst.data_ptr(), cap, scr.data_ptr(), ss, res, stream=streams[i]) == 0
        for i in (0, 1):
            streams[i].synchronize()
            h, rs, rr, scr, ss, dst, res, cap = state[i]
            assert res.tolist() == [20000] * len(rs)
            out = dst.cpu().numpy()
            for o, n, dd in rs:
                assert np.array_equal(out[dd:dd + n], data[o:o + n]), (rep, i)
    for s in state:
        host.L.zxc_b200_seekable_device_free(s[0])
    assert np.array_equal(buf.numpy(), frame)


@pytest.mark.gpu
def test_graph_capture_with_a_dictionary(host, prod):
    """captured once with a dictionary set, replayed after rewriting d_ranges in place: equal to fresh calls"""
    t = host.t
    d, huf = next(iter(golden_dicts().values()))
    data = make_case("text", 2 << 20)
    frame = prod.compress(data, level=6, block_size=65536, checksum=1, seekable=1, dict=d, dict_huf=huf)
    h, buf = host.open_host(frame, 5)
    assert host.set_dict(h, d, huf) == 0
    n, ln = 64, 10000
    cap = n * ln
    scr, ss = host.scratch(h, n, cap)
    dst = t.zeros(cap, dtype=t.uint8, device="cuda")
    res = t.zeros(n, dtype=t.int64, device="cuda")

    def draw(seed):
        rng = np.random.default_rng(seed)
        return [(int(o), ln, k * ln) for k, o in enumerate(rng.integers(0, data.size - ln, n))]

    rr = host.ranges(draw(1))
    s = t.cuda.Stream()
    s.wait_stream(t.cuda.current_stream())
    with t.cuda.stream(s):
        assert host.call(h, rr, n, dst.data_ptr(), cap, scr.data_ptr(), ss, res, stream=s) == 0
    t.cuda.current_stream().wait_stream(s)
    t.cuda.synchronize()
    g = t.cuda.CUDAGraph()
    with t.cuda.graph(g):
        assert host.call(h, rr, n, dst.data_ptr(), cap, scr.data_ptr(), ss, res,
                         stream=t.cuda.current_stream()) == 0
    for seed in (2, 3, 4):
        rs = draw(seed)
        if seed == 4:
            rs[5] = (data.size - 5, ln, 5 * ln)
        rr.copy_(host.ranges(rs))
        dst.zero_()
        res.zero_()
        g.replay()
        t.cuda.synchronize()
        got, out = res.tolist(), dst.cpu().numpy()
        fresh, fout = host.run(h, rs, cap)
        assert got == fresh
        for (o, k, dd), r in zip(rs, got):
            if r > 0:
                assert np.array_equal(out[dd:dd + k], data[o:o + k]) and np.array_equal(fout[dd:dd + k], out[dd:dd + k])
    host.L.zxc_b200_seekable_device_free(h)


@pytest.mark.gpu
def test_launch_count_and_scratch_query(host, prod):
    """9 launches for every range mix; a device handle's scratch query is the same with or without a host handle"""
    d, huf = next(iter(golden_dicts().values()))
    data = make_case("text", 300000)
    L = host.L
    for frame, dd in ((prod.compress(data, level=3, block_size=65536, checksum=1, seekable=1), None),
                      (prod.compress(data, level=6, block_size=4096, seekable=1, dict=d, dict_huf=huf), d)):
        hd, src = host.open(frame)
        queries = [(n, b) for n in (1, 7, 1000) for b in (0, 1, 65536, 10 << 20)]
        before = [L.zxc_b200_seekable_device_scratch_size(hd, n, b) for n, b in queries]
        h, buf = host.open_host(frame)
        assert [L.zxc_b200_seekable_device_scratch_size(hd, n, b) for n, b in queries] == before
        assert all(L.zxc_b200_seekable_device_scratch_size(h, n, b) > s for (n, b), s in zip(queries, before))
        if dd is not None:
            assert host.set_dict(h, d, huf) == 0
        for rs in ([(0, 0, 0)], [(5, 10, 0)], [(0, data.size, 0)], [(data.size, 5, 0)],
                   packed([(k * 999, 5000) for k in range(200)])[0]):
            cap = max(dd_ + n for _, n, dd_ in rs) + 1
            n0 = L.zxc_b200_launch_count()
            host.run(h, rs, cap)
            assert L.zxc_b200_launch_count() - n0 == LAUNCHES, len(rs)
        L.zxc_b200_seekable_device_free(h)
        L.zxc_b200_seekable_device_free(hd)


@pytest.mark.gpu
def test_python_seekable_frame_pinned(prod):
    import torch
    from zxc_b200 import device
    data = zc.silesia_shaped(3 << 20, seed=71)
    fr = torch.from_numpy(prod.compress(data, level=3, block_size=65536, checksum=1, seekable=1))
    pinned = fr.pin_memory()
    whole = torch.from_numpy(data).cuda()
    with device.SeekableFrame(pinned) as sf:
        assert sf.device == torch.device("cuda", torch.cuda.current_device())
        assert (sf.decompressed_size, sf.block_size, sf.n_blocks) == (data.size, 65536, 48)
        r = sf.read(12345, 200000)
        assert r.is_cuda and torch.equal(r, whole[12345:212345])
        offs = torch.tensor([0, 70000, 5, data.size - 9], dtype=torch.int64, device="cuda")
        lens = torch.tensor([100, 65536 * 2, 0, 9], dtype=torch.int64, device="cuda")
        out, res = sf.gather(offs, lens)
        torch.cuda.synchronize()
        assert res.tolist() == [100, 131072, 0, 9]
        assert torch.equal(out, torch.cat([whole[0:100], whole[70000:201072], whole[data.size - 9:]]))
        with pytest.raises(device.ZxcError) as e:
            sf.read(data.size - 5, 10)
        assert e.value.code == SRC_SMALL
    with device.SeekableFrame(pinned, device="cuda:0") as sf:
        assert sf.device == torch.device("cuda", 0)
    d, huf = next(iter(golden_dicts().values()))
    fd = torch.from_numpy(prod.compress(data[:100000], level=6, block_size=4096, seekable=1, dict=d,
                                        dict_huf=huf)).pin_memory()
    with device.SeekableFrame(fd, dict=d, dict_huf=huf) as sf:
        assert np.array_equal(sf.read(4000, 50000).cpu().numpy(), data[4000:54000])
    with pytest.raises(ValueError, match="pin_memory"):
        device.SeekableFrame(fr)
    plain = torch.from_numpy(prod.compress(data[:100000], level=3, block_size=4096)).pin_memory()
    with pytest.raises(ValueError):
        device.SeekableFrame(plain)
