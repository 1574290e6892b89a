"""zxc_b200_add_seek_table_device: a frame without a SEK table, in HBM, gets the table zxc_compress writes with
seekable = 1, found on the device by a parallel header search and proven against the sequential walk.

The oracle is built on the host from zxc_b200_plan_frame (the sequential walk) and zxc_write_seek_table, this
library's and the reference's where it is built."""
import ctypes as C
import os

import numpy as np
import pytest

import zxc_corpus as zc
import zxc_ctypes as z
from conftest import has_cuda
from test_oracle import G, INVALID, VALID, golden_dicts, make_case

NULL_INPUT, SRC_SMALL, DST_TOO_SMALL, MEMORY, NO_DEVICE = -12, -3, -2, -1, -100
BAD_HEADER, CORRUPT, BAD_BLOCK_TYPE, BAD_MAGIC = -6, -8, -13, -4
LAUNCHES = 43
PATH_SPEC, PATH_WALK = 1, 2
HDR, FTR = 16, 12


class Job(C.Structure):
    _fields_ = [("src_off", C.c_uint64), ("dst_off", C.c_uint64), ("src_len", C.c_uint32), ("dst_cap", C.c_uint32)]


def bind(L):
    L.zxc_b200_seek_table_device_bound.restype = C.c_uint64
    L.zxc_b200_seek_table_device_bound.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
    L.zxc_b200_seek_table_device_scratch_size.restype = C.c_size_t
    L.zxc_b200_seek_table_device_scratch_size.argtypes = [C.c_uint64, C.c_uint32]
    L.zxc_b200_add_seek_table_device.restype = C.c_int
    L.zxc_b200_add_seek_table_device.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_size_t,
                                                 C.c_void_p, C.c_void_p]
    L.zxc_b200_plan_frame.restype = C.c_int64
    L.zxc_b200_plan_frame.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    L.zxc_write_seek_table.restype = C.c_int64
    L.zxc_write_seek_table.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32]
    L.zxc_b200_launch_count.restype = C.c_uint64
    return L


def _ref():
    return z.ZxcLib(z.REF_SO) if z.have_ref() else None


def seek_table(L, sizes):
    """zxc_write_seek_table of library L for these entries"""
    s = np.zeros(max(len(sizes), 1), np.uint32)  # never NULL: zxc_write_seek_table rejects that even for 0 entries
    s[:len(sizes)] = sizes
    out = np.zeros(8 + 4 * len(sizes), np.uint8)
    L.zxc_write_seek_table.restype = C.c_int64
    L.zxc_write_seek_table.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32]
    assert L.zxc_write_seek_table(out.ctypes.data, out.size, s.ctypes.data, len(sizes)) == out.size
    return out


def oracle(L, frame, cap=None, max_blocks=None, table_lib=None):
    """-> (result, the buffer's first max(result, len) bytes afterwards), from the sequential walk of L"""
    f = np.asarray(frame, np.uint8)
    n = f.size
    cap = n if cap is None else cap
    if n < 36:
        return SRC_SMALL, f
    nb = L.zxc_b200_plan_frame(f.ctypes.data, n, None, 0, None)
    if nb < 0:
        return int(nb), f
    jobs = (Job * max(nb, 1))()
    assert L.zxc_b200_plan_frame(f.ctypes.data, n, jobs, nb, None) == nb
    sizes = [jobs[i].src_len for i in range(nb)]
    bs = 1 << int(f[5])
    footer = int(f[n - 12:n - 4].view(np.uint64)[0])
    need = -(-footer // bs)
    if max_blocks is not None and nb > max_blocks:
        return (CORRUPT if nb != need else MEMORY), f
    if any(f[jobs[i].src_off] > 2 for i in range(nb)):
        return BAD_BLOCK_TYPE, f
    eof = jobs[nb - 1].src_off + jobs[nb - 1].src_len if nb else HDR
    tail = f[eof + 8:]
    table = seek_table(table_lib or L, sizes)
    if tail.size == table.size + FTR and np.array_equal(tail[:table.size], table):
        return n, f
    if tail.size != FTR or nb != need:
        return CORRUPT, f
    if nb == 0:
        return n, f
    if cap < n + table.size:
        return DST_TOO_SMALL, f
    return n + table.size, np.concatenate([f[:n - FTR], table, f[n - FTR:]])


# ---------------------------------------------------------------------------------------------------------------
# no device
# ---------------------------------------------------------------------------------------------------------------
def test_host_verdicts_without_a_device(prod):
    """Without a device: the bound and the scratch size are 0, and the host's codes come in their order."""
    if has_cuda():
        pytest.skip("only meaningful without a GPU")
    L = bind(prod.lib)
    frame = np.fromfile(os.path.join(G, "valid", "text_1k.zxc"), np.uint8)
    fake = 1 << 40  # never dereferenced
    assert L.zxc_b200_seek_table_device_bound(frame.ctypes.data, frame.size, None) == 0
    assert L.zxc_b200_seek_table_device_bound(None, 100, None) == 0
    assert L.zxc_b200_seek_table_device_scratch_size(1 << 20, 16) == 0
    assert L.zxc_b200_seek_table_device_scratch_size(0, 0) == 0
    add = L.zxc_b200_add_seek_table_device
    assert add(None, 100, 200, fake, 1 << 20, fake, None) == NULL_INPUT
    assert add(fake, 100, 200, None, 1 << 20, fake, None) == NULL_INPUT
    assert add(fake, 100, 200, fake, 1 << 20, None, None) == NULL_INPUT
    assert add(fake, 201, 200, fake, 1 << 20, fake, None) == NULL_INPUT
    assert add(fake, 35, 200, fake, 1 << 20, fake, None) == SRC_SMALL
    assert add(fake, 0, 0, fake, 0, fake, None) == SRC_SMALL
    assert add(fake, 36, 36, fake, 0, fake, None) == NO_DEVICE
    assert add(fake, 100, 200, fake, 1 << 20, fake, None) == NO_DEVICE


def test_python_argument_checks():
    """add_seek_table rejects what it cannot seal before anything is enqueued (no device needed)"""
    import torch
    from zxc_b200 import device
    with pytest.raises(ValueError, match="CUDA"):
        device.add_seek_table(torch.zeros(64, dtype=torch.uint8))
    with pytest.raises(ValueError, match="CUDA"):
        device.add_seek_table(np.zeros(64, np.uint8))
    if not has_cuda():
        return
    with pytest.raises(ValueError, match="uint8"):
        device.add_seek_table(torch.zeros(64, dtype=torch.float32, device="cuda"))
    with pytest.raises(ValueError, match="contiguous"):
        device.add_seek_table(torch.zeros((8, 8), dtype=torch.uint8, device="cuda")[:, 0])
    with pytest.raises(ValueError, match="frame_size"):
        device.add_seek_table(torch.zeros(64, dtype=torch.uint8, device="cuda"), frame_size=65)
    with pytest.raises(ValueError, match="frame_size"):
        device.add_seek_table(torch.zeros(64, dtype=torch.uint8, device="cuda"), frame_size=-1)


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
class Dev:
    def __init__(self, prod):
        import torch
        self.t = torch
        self.L = bind(prod.lib)

    def scratch(self, frame_size, max_blocks, guard=0, fill=0):
        ss = int(self.L.zxc_b200_seek_table_device_scratch_size(frame_size, max_blocks))
        assert ss > 0
        return self.t.full((ss + 2 * guard,), fill, dtype=self.t.uint8, device="cuda"), ss

    def run(self, frame, cap=None, max_blocks=None, off=3, guard=64, stream=None):
        """-> (result, buffer bytes [0, max(result, len)), path); the frame at an odd offset with guard bytes around the
        buffer and the scratch, which must stay untouched"""
        t = self.t
        f = np.asarray(frame, np.uint8)
        n = f.size
        cap = n + 8 + 4 * (n // 8) if cap is None else cap
        if max_blocks is None:
            max_blocks = max((n - 36) // 8, 0) if n < (1 << 22) else (n // 1024)
        buf = t.full((off + cap + guard,), 0xA5, dtype=t.uint8, device="cuda")
        buf[off:off + n].copy_(t.from_numpy(f.copy()))
        scr, ss = self.scratch(n, max_blocks, guard=guard, fill=0x5A)
        res = t.full((1,), 12345, dtype=t.int64, device="cuda")
        rc = self.L.zxc_b200_add_seek_table_device(buf.data_ptr() + off, n, cap, scr.data_ptr() + guard, ss,
                                                   res.data_ptr(), stream.cuda_stream if stream else None)
        if rc != 0:  # the host's verdict: nothing was enqueued
            t.cuda.synchronize()
            assert (buf.cpu().numpy()[off:off + n] == f).all()
            return rc, f, 0
        t.cuda.synchronize()
        r = int(res.item())
        b = buf.cpu().numpy()
        assert (b[:off] == 0xA5).all() and (b[off + cap:] == 0xA5).all(), "buffer guard"
        s = scr.cpu().numpy()
        assert (s[:guard] == 0x5A).all() and (s[guard + ss:] == 0x5A).all(), "scratch guard"
        path = int(s[guard + (-(scr.data_ptr() + guard) % 256):][:4].view(np.uint32)[0])
        return r, b[off:off + max(r, n)], path


@pytest.fixture(scope="module")
def dev(prod):
    return Dev(prod)


def check(dev, prod, frame, what, cap=None, max_blocks=None, path=None, ref=None):
    """the device's result and bytes equal the oracle's (and, for a new table, the reference's table)"""
    f = np.asarray(frame, np.uint8)
    r, b, p = dev.run(f, cap=cap, max_blocks=max_blocks)
    want, wb = oracle(dev.L, f, cap=cap if cap is not None else f.size + 8 + 4 * (f.size // 8),
                      max_blocks=max_blocks, table_lib=None)
    assert r == want, (what, z.ERR.get(r, r), z.ERR.get(want, want))
    if r < 0 or r == f.size:
        assert np.array_equal(b[:f.size], f), (what, "buffer changed")
    else:
        assert np.array_equal(b[:r], wb[:r]), (what, "bytes")
        if ref is not None:
            rr, rb = oracle(dev.L, f, cap=f.size + 8 + 4 * (f.size // 8), table_lib=ref.lib)
            assert rr == r and np.array_equal(rb[:r], b[:r]), (what, "reference table")
    if path is not None:
        assert p == path, (what, "path", p)
    return r, b[:max(r, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, 2, 3, 4, 5, 6, 7])
def test_identity_with_the_seekable_encoder(dev, prod, level):
    """add_seek_table(compress(x, seekable=0)) == compress(x, seekable=1): host, device and reference encoders"""
    import torch
    from zxc_b200 import device
    ref = _ref()
    for bs in (4096, 65536, 2 << 20):
        data = make_case("silesia", 3 * bs + 12345)
        for cks in (0, 1):
            plain = prod.compress(data, level=level, block_size=bs, checksum=cks, seekable=0)
            want = prod.compress(data, level=level, block_size=bs, checksum=cks, seekable=1)
            r, b = check(dev, prod, plain, (level, bs, cks), path=PATH_SPEC, ref=ref)
            assert r == want.size and np.array_equal(b, want), (level, bs, cks)
            dplain = device.compress(torch.from_numpy(data).cuda(), level=level, block_size=bs, checksum=cks)
            assert np.array_equal(dplain.frame.cpu().numpy(), plain)
            sealed = device.add_seek_table(dplain.frame.clone())
            assert np.array_equal(sealed.cpu().numpy(), want), ("device encoder", level, bs, cks)
            if ref is not None:
                rp = ref.compress(data, level=level, block_size=bs, checksum=cks, seekable=0)
                rs = ref.compress(data, level=level, block_size=bs, checksum=cks, seekable=1)
                r, b = check(dev, prod, rp, ("ref", level, bs, cks))
                assert np.array_equal(b, rs), ("reference encoder", level, bs, cks)


@pytest.mark.gpu
def test_small_inputs_and_dictionaries(dev, prod):
    """an empty input (no table), one block, one byte, and dictionary frames"""
    for data in (np.zeros(0, np.uint8), np.frombuffer(b"x", np.uint8), make_case("silesia", 4000),
                 make_case("silesia", 65536)):
        for bs in (4096, 65536):
            plain = prod.compress(data, level=3, block_size=bs, checksum=1, seekable=0)
            want = prod.compress(data, level=3, block_size=bs, checksum=1, seekable=1)
            r, b = check(dev, prod, plain, (data.size, bs))
            assert r == want.size and np.array_equal(b, want), (data.size, bs)
    for name, (d, huf) in sorted(golden_dicts().items()):
        data = make_case("silesia", 50000)
        for level in (1, 5):
            plain = prod.compress(data, level=level, block_size=4096, dict=d, dict_huf=huf)
            want = prod.compress(data, level=level, block_size=4096, seekable=1, dict=d, dict_huf=huf)
            r, b = check(dev, prod, plain, (name, level), path=PATH_SPEC)
            assert np.array_equal(b, want), (name, level)


@pytest.mark.gpu
def test_stream_encoders(dev, prod):
    """frames written by the host and device push streams seal like those of zxc_compress"""
    import torch
    from zxc_b200 import device, stream
    data = make_case("silesia", 300000)
    for bs, cks in ((4096, 0), (65536, 1)):
        want = prod.compress(data, level=3, block_size=bs, checksum=cks, seekable=1)
        c = stream.compressobj(level=3, block_size=bs, checksum=cks)
        host = np.frombuffer(b"".join([c.compress(data[:100000].tobytes()), c.compress(data[100000:].tobytes()),
                                       c.flush()]), np.uint8)
        r, b = check(dev, prod, host, ("cstream", bs, cks))
        assert np.array_equal(b, want), ("cstream", bs)
        dc = device.compressobj(level=3, block_size=bs, checksum=cks)
        g = torch.from_numpy(data).cuda()
        parts = [dc.compress(g[:123457]), dc.compress(g[123457:]), dc.flush()]
        dframe = torch.cat([p.reshape(-1) for p in parts])
        assert np.array_equal(device.add_seek_table(dframe).cpu().numpy(), want), ("device cstream", bs)


@pytest.mark.gpu
@pytest.mark.parametrize("name", VALID)
def test_golden_frames(dev, prod, name):
    """every golden frame gets the oracle's result; a new table opens in the product and the reference"""
    frame = np.fromfile(os.path.join(G, "valid", name + ".zxc"), np.uint8)
    r, b = check(dev, prod, frame, name)
    if r > frame.size:
        for lib in [prod] + ([_ref()] if z.have_ref() else []):
            fb = b.tobytes()
            h = lib.lib.zxc_seekable_open(fb, len(fb))
            assert h, (name, lib.path)
            lib.lib.zxc_seekable_free(h)


@pytest.mark.gpu
def test_use_after_sealing(dev, prod):
    """a sealed frame serves ranges on the device handle and decodes as before"""
    import torch
    from zxc_b200 import device
    from test_seekable_device import Dev as SDev, same, standard_ranges
    sd = SDev(prod)
    for level, bs, cks in ((1, 4096, 0), (3, 65536, 1), (6, 2 << 20, 1)):
        data = make_case("silesia", 3 * bs + 777)
        plain = prod.compress(data, level=level, block_size=bs, checksum=cks)
        g = torch.from_numpy(plain).cuda()
        with pytest.raises(ValueError):
            device.SeekableFrame(g)
        sealed = device.add_seek_table(g)
        rs, cap = standard_ranges(data.size, bs, level)
        res = same(sd, prod, sealed.cpu().numpy(), rs, cap, what=(level, bs))
        assert res == [n for _, n, _ in rs]
        a = device.decompress_frame(torch.from_numpy(plain).cuda(), checksum=True).cpu().numpy()
        b = device.decompress_frame(sealed, checksum=True).cpu().numpy()
        assert np.array_equal(a, data) and np.array_equal(b, data)
        with device.SeekableFrame(sealed) as s:
            assert s.n_blocks == -(-data.size // bs)


@pytest.mark.gpu
def test_many_blocks(dev, prod):
    """2^18 + 5 blocks of 4 KiB: the doubling runs 19 rounds over many tiles"""
    nb = (1 << 18) + 5
    data = np.zeros(nb * 4096 - 100, np.uint8)  # blocks of a few bytes on disk: a 1 GiB input, a small frame
    data[::4096] = np.random.default_rng(5).integers(0, 256, -(-data.size // 4096), dtype=np.uint8)
    data[::997] = 7
    plain = prod.compress(data, level=1, block_size=4096, checksum=1)
    want = prod.compress(data, level=1, block_size=4096, checksum=1, seekable=1)
    r, b, p = dev.run(plain, cap=want.size, max_blocks=nb, guard=0)
    assert r == want.size and p == PATH_SPEC
    assert np.array_equal(b, want)


# ---- hand-stitched frames ----------------------------------------------------------------------------------------
def _h8(v):
    h = (v ^ 0x9E3779B97F4A7C15) & (2 ** 64 - 1)
    h ^= (h << 13) & (2 ** 64 - 1)
    h ^= h >> 7
    h ^= (h << 17) & (2 ** 64 - 1)
    return ((h >> 32) ^ h) & 0xFF


def bhdr(typ, comp):
    v = typ | (comp << 24)
    return (v | (_h8(v) << 56)).to_bytes(8, "little")


def raw_frame(prod, payloads, bs=4096, cks=0):
    """a valid frame of RAW blocks with these payloads (each at most bs bytes, all but the last exactly bs)"""
    hdr = prod.compress(np.zeros(0, np.uint8), level=1, block_size=bs, checksum=cks)[:HDR].tobytes()
    body = b""
    for p in payloads:
        body += bhdr(0, len(p)) + p + (b"\0\0\0\0" if cks else b"")
    total = sum(len(p) for p in payloads)
    return np.frombuffer(hdr + body + bhdr(255, 0) + total.to_bytes(8, "little") + b"\0" * 4, np.uint8)


def fakes(n, comp=16):
    """n back-to-back valid-looking RAW headers of `comp`-byte blocks"""
    return (bhdr(0, comp) * n)


@pytest.mark.gpu
def test_hostile_speculation(dev, prod):
    """valid frames whose payloads hold valid-looking headers: speculation or the walk, the exact result either way"""
    bs = 4096
    # one block's worth of fake headers: resolved by speculation
    one = raw_frame(prod, [fakes(bs // 8, comp=8)[:bs], b"tail" * 10])
    check(dev, prod, one, "one block of fakes", path=PATH_SPEC)
    # enough fakes to overflow the list of a scratch sized for the real blocks: the walk decides
    many = raw_frame(prod, [fakes(bs // 8)[:bs]] * 8 + [b"end"])
    check(dev, prod, many, "overflow", max_blocks=9, path=PATH_WALK)
    # false chains merging into the true one: fakes that step onto the next real header
    rng = np.random.default_rng(3)
    p = bytearray(rng.integers(0, 256, bs, dtype=np.uint8).tobytes())
    for k in range(0, 64, 8):  # payload offset k steps to k + 8 + (bs - k - 8) = bs: the next real header
        p[k:k + 8] = bhdr(k % 3, bs - k - 8)
    merge = raw_frame(prod, [bytes(p), bytes(p), b"x" * 100])
    check(dev, prod, merge, "merging chains", path=PATH_SPEC)
    # a false EOF candidate inside a payload, and a fake GHI header that steps onto it
    q = bytearray(rng.integers(0, 256, bs, dtype=np.uint8).tobytes())
    q[100:108] = bhdr(255, 0)
    q[0:8] = bhdr(2, 92)
    check(dev, prod, raw_frame(prod, [bytes(q), b"y" * 10]), "false EOF", path=PATH_SPEC)


# ---- damage ----------------------------------------------------------------------------------------------------
def _frame(prod, n=5, bs=4096, cks=1, level=3):
    return prod.compress(make_case("silesia", n * bs - 99), level=level, block_size=bs, checksum=cks)


def _offsets(L, f):
    nb = L.zxc_b200_plan_frame(f.ctypes.data, f.size, None, 0, None)
    jobs = (Job * nb)()
    L.zxc_b200_plan_frame(f.ctypes.data, f.size, jobs, nb, None)
    return [jobs[i].src_off for i in range(nb)], jobs[nb - 1].src_off + jobs[nb - 1].src_len


@pytest.mark.gpu
def test_damage(dev, prod):
    """exact verdicts on mutated headers, EOF block and footer, truncations and garbage tails; the buffer unchanged"""
    rng = np.random.default_rng(7)
    f = _frame(prod)
    offs, eof = _offsets(dev.L, f)
    for at in (offs[0], offs[len(offs) // 2], offs[-1], eof, f.size - 12, 0):
        for _ in range(12):
            g = f.copy()
            pos = at + int(rng.integers(0, 8))
            g[pos] ^= np.uint8(1 << int(rng.integers(0, 8)))
            check(dev, prod, g, ("flip", at, pos))
    for cut in (36, 40, offs[1], offs[1] + 5, eof, eof + 8, f.size - 1):
        check(dev, prod, f[:cut], ("truncated", cut))
    tail = f[eof + 8:]
    for junk in (1, 4, 8, 13):
        check(dev, prod, np.concatenate([f[:eof + 8], rng.integers(0, 256, junk).astype(np.uint8), tail]),
              ("garbage", junk))
    # a SEK-type block in the chain (with its checksum trailer)
    g = np.concatenate([f[:eof], np.frombuffer(bhdr(254, 0) + b"\0" * 4, np.uint8), f[eof:]])
    check(dev, prod, g, "SEK block in the chain")
    # N != ceil(footer / block_size)
    for d in (-4096, 4096):
        g = f.copy()
        g[-12:-4] = np.frombuffer((int(f[-12:-4].view(np.uint64)[0]) + d).to_bytes(8, "little"), np.uint8)
        check(dev, prod, g, ("footer", d))
    for name, code in sorted(INVALID.items()):
        g = np.fromfile(os.path.join(G, "invalid", name + ".zxc"), np.uint8)
        check(dev, prod, g, name)


@pytest.mark.gpu
def test_existing_tables(dev, prod):
    """a valid table is a no-op (twice equals once); a forged one is CORRUPT_DATA"""
    f = _frame(prod)
    sealed = prod.compress(make_case("silesia", 5 * 4096 - 99), level=3, block_size=4096, checksum=1, seekable=1)
    r, b = check(dev, prod, sealed, "sealed")
    assert r == sealed.size
    r2, b2 = check(dev, prod, sealed, "again")
    assert r2 == r and np.array_equal(b2, b)
    forged = sealed.copy()
    forged[-16] ^= 1  # the last entry
    assert check(dev, prod, forged, "forged entry")[0] == CORRUPT
    assert check(dev, prod, f, "plain")[0] == sealed.size


@pytest.mark.gpu
def test_limits(dev, prod):
    """DST_TOO_SMALL one byte short, MEMORY one block short; the buffer unchanged"""
    f = _frame(prod, n=7)
    nb = 7
    need = f.size + 8 + 4 * nb
    assert check(dev, prod, f, "exact", cap=need, max_blocks=nb)[0] == need
    assert check(dev, prod, f, "one byte short", cap=need - 1, max_blocks=nb)[0] == DST_TOO_SMALL
    assert check(dev, prod, f, "one block short", max_blocks=nb - 1)[0] == MEMORY
    g = dev.t.from_numpy(f).cuda()
    assert int(dev.L.zxc_b200_seek_table_device_bound(g.data_ptr(), f.size, None)) == need
    sealed = prod.compress(make_case("silesia", 7 * 4096 - 99), level=3, block_size=4096, checksum=1, seekable=1)
    h = dev.t.from_numpy(sealed).cuda()
    assert int(dev.L.zxc_b200_seek_table_device_bound(h.data_ptr(), sealed.size, None)) == sealed.size
    e = dev.t.from_numpy(prod.compress(np.zeros(0, np.uint8))).cuda()
    assert int(dev.L.zxc_b200_seek_table_device_bound(e.data_ptr(), e.numel(), None)) == e.numel()
    assert int(dev.L.zxc_b200_seek_table_device_bound(g.data_ptr(), 35, None)) == 0


@pytest.mark.gpu
def test_streams_graphs_and_launches(dev, prod):
    """the launch count; graph capture replayed on another frame of the same sizes; two calls on two streams"""
    t = dev.t
    L = dev.L
    rng = np.random.default_rng(11)
    frames = [raw_frame(prod, [rng.integers(0, 256, 4096, dtype=np.uint8).tobytes()] * 6 + [b"z" * 77])
              for _ in range(2)]
    size = frames[0].size
    buf = t.zeros(size + 100, dtype=t.uint8, device="cuda")
    scr, ss = dev.scratch(size, 7)
    res = t.zeros(1, dtype=t.int64, device="cuda")
    s = t.cuda.Stream()
    buf[:size].copy_(t.from_numpy(frames[0]))
    t.cuda.synchronize()
    before = L.zxc_b200_launch_count()
    assert L.zxc_b200_add_seek_table_device(buf.data_ptr(), size, buf.numel(), scr.data_ptr(), ss, res.data_ptr(),
                                            s.cuda_stream) == 0
    assert L.zxc_b200_launch_count() - before == LAUNCHES
    s.synchronize()
    want = oracle(L, frames[0], cap=buf.numel())
    assert int(res.item()) == want[0] > size
    assert np.array_equal(buf.cpu().numpy()[:want[0]], want[1])
    g = t.cuda.CUDAGraph()
    with t.cuda.graph(g, stream=s):
        assert L.zxc_b200_add_seek_table_device(buf.data_ptr(), size, buf.numel(), scr.data_ptr(), ss,
                                                res.data_ptr(), s.cuda_stream) == 0
    for fr in frames[::-1]:
        want = oracle(L, fr, cap=buf.numel())
        buf.zero_()
        buf[:size].copy_(t.from_numpy(fr))
        res.fill_(12345)
        t.cuda.synchronize()
        g.replay()
        t.cuda.synchronize()
        assert int(res.item()) == want[0]
        assert np.array_equal(buf.cpu().numpy()[:want[0]], want[1])
    # two calls on two streams, each with its own scratch
    work = []
    for fr in (_frame(prod, n=9, level=1), _frame(prod, n=3, bs=65536, level=5)):
        bb = t.zeros(fr.size + 64, dtype=t.uint8, device="cuda")
        bb[:fr.size].copy_(t.from_numpy(fr))
        sc, sz = dev.scratch(fr.size, 16)
        rr = t.zeros(1, dtype=t.int64, device="cuda")
        work.append((fr, bb, sc, sz, rr, t.cuda.Stream()))
    t.cuda.synchronize()
    for fr, bb, sc, sz, rr, st in work:
        assert L.zxc_b200_add_seek_table_device(bb.data_ptr(), fr.size, bb.numel(), sc.data_ptr(), sz, rr.data_ptr(),
                                                st.cuda_stream) == 0
    t.cuda.synchronize()
    for fr, bb, sc, sz, rr, st in work:
        want = oracle(L, fr, cap=bb.numel())
        assert int(rr.item()) == want[0] > fr.size
        assert np.array_equal(bb.cpu().numpy()[:want[0]], want[1])
