"""zxc_b200_compress_blocks_device / zxc_b200_decompress_blocks_device: the block API in HBM, many frameless blocks
per call.

Every item's result and bytes must equal this library's zxc_compress_block (on a fresh context) or
zxc_decompress_block / zxc_decompress_block_safe for that item alone, and the reference's where it is built."""
import ctypes as C

import numpy as np
import pytest

import zxc_corpus as zc
import zxc_ctypes as z
from conftest import has_cuda
from test_compress_device import opts
from test_oracle import make_case

NULL_INPUT, DST_TOO_SMALL, BAD_BS, DICT_BIG, MEMORY, NO_DEVICE = -12, -2, -14, -17, -1, -100
GUARD = 64
MIB2 = 1 << 21
TAIL_PAD = 2112


def bind(L):
    L.zxc_b200_compress_blocks_device_scratch_size.restype = C.c_size_t
    L.zxc_b200_compress_blocks_device_scratch_size.argtypes = [C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p]
    L.zxc_b200_compress_blocks_device.restype = C.c_int
    L.zxc_b200_compress_blocks_device.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t,
                                                  C.c_void_p, C.c_void_p]
    L.zxc_b200_decompress_blocks_device_scratch_size.restype = C.c_size_t
    L.zxc_b200_decompress_blocks_device_scratch_size.argtypes = [C.c_uint32, C.c_uint64]
    L.zxc_b200_decompress_blocks_device.restype = C.c_int
    L.zxc_b200_decompress_blocks_device.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_void_p,
                                                    C.c_size_t, C.c_void_p, C.c_void_p]
    L.zxc_b200_launch_count.restype = C.c_uint64
    return L


def dopts(cks=0, d=None):
    o = z.DecompressOpts(checksum_enabled=cks)
    o._keep = None
    if d is not None:
        o._keep = bytes(d)
        o.dict, o.dict_size = C.cast(C.c_char_p(o._keep), C.c_void_p), len(o._keep)
    return o


def test_host_verdicts_without_a_device(prod):
    """The whole-call verdicts come in order without a device; the size queries are 0."""
    if has_cuda():
        pytest.skip("only meaningful without a GPU")
    L = bind(prod.lib)
    fake = 1 << 40  # never dereferenced
    cb, db = L.zxc_b200_compress_blocks_device, L.zxc_b200_decompress_blocks_device
    for f in (lambda *a: cb(*a), lambda it, n, o, s, ss, r, st: db(it, n, o, 0, s, ss, r, st)):
        assert f(None, 1, None, fake, 1 << 20, fake, None) == NULL_INPUT
        assert f(fake, 1, None, None, 1 << 20, fake, None) == NULL_INPUT
        assert f(fake, 1, None, fake, 1 << 20, None, None) == NULL_INPUT
        assert f(fake, 1, None, fake, 0, fake, None) == NO_DEVICE
        assert f(None, 0, None, None, 0, None, None) == NO_DEVICE
    big = b"x" * 70000
    assert cb(fake, 1, C.byref(opts(3, d=big)), fake, 1 << 20, fake, None) == DICT_BIG
    assert cb(None, 0, C.byref(opts(3, d=big)), None, 0, None, None) == DICT_BIG
    assert db(fake, 1, C.byref(dopts(d=big)), 1, fake, 1 << 20, fake, None) == DICT_BIG
    assert cb(fake, 1, C.byref(opts(3, 5000, h=bytes(128), d=b"abcdefgh")), fake, 0, fake, None) == NO_DEVICE
    assert L.zxc_b200_compress_blocks_device_scratch_size(10, 1 << 20, 4096, None) == 0
    assert L.zxc_b200_decompress_blocks_device_scratch_size(10, 4096) == 0


def test_block_bytes_ignore_block_size(ref):
    """The fact the batched encode rests on: the reference's zxc_compress_block gives the same bytes whatever
    opts->block_size says, and on a context reused across calls with the same level and dictionary (the reference
    keeps dictionary state in a context, so a context reused across levels is not a fresh one)."""
    text = zc.silesia_shaped(MIB2 + 4096, seed=21)
    d = bytes(zc.silesia_shaped(16384, seed=22))
    keep = C.create_string_buffer(d)
    shared = {}
    try:
        for n in (1, 4095, 4096, 4097, 65536, MIB2):
            src = np.ascontiguousarray(text[:n])
            cap = int(ref.lib.zxc_compress_block_bound(n))
            for level in range(1, 8):
                if n == MIB2 and level >= 6:
                    src_l = np.ascontiguousarray(text[:n // 4])  # the optimal parser on the CPU: keep the run short
                else:
                    src_l = src
                for with_dict in (False, True):
                    want = None
                    if (level, with_dict) not in shared:
                        shared[level, with_dict] = ref.lib.zxc_create_cctx(None)
                    for bs, ctx in ((0, None), (4096, None), (65536, None), (MIB2, None), (0, shared[level, with_dict])):
                        o = z.CompressOpts(level=level, block_size=bs, checksum_enabled=1)
                        if with_dict:
                            o.dict, o.dict_size = C.cast(keep, C.c_void_p), len(d)
                        c = ctx or ref.lib.zxc_create_cctx(None)
                        out = np.zeros(cap, np.uint8)
                        r = ref.lib.zxc_compress_block(c, src_l.ctypes.data, src_l.size, out.ctypes.data, cap,
                                                       C.byref(o))
                        if ctx is None:
                            ref.lib.zxc_free_cctx(c)
                        assert r > 0, (n, level, bs, r)
                        got = out[:r].tobytes()
                        want = want or got
                        assert got == want, (n, level, with_dict, bs, ctx is not None)
    finally:
        for c in shared.values():
            ref.lib.zxc_free_cctx(c)


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
class Host:
    """this library's host block calls, one item at a time"""

    def __init__(self, lib):
        self.L = lib

    def compress(self, data, cap, o):
        c = self.L.zxc_create_cctx(None)
        try:
            data = np.ascontiguousarray(data, np.uint8)
            out = np.zeros(max(cap, 1), np.uint8)
            r = self.L.zxc_compress_block(c, data.ctypes.data if data.size else None, data.size, out.ctypes.data,
                                          cap, C.byref(o) if o is not None else None)
            return r, (out[:r].tobytes() if r > 0 else None)
        finally:
            self.L.zxc_free_cctx(c)

    def decompress(self, block, cap, o, safe):
        c = self.L.zxc_create_dctx()
        try:
            block = np.frombuffer(bytes(block), np.uint8) if len(block) else np.zeros(1, np.uint8)[:0]
            buf = np.zeros(max(block.size, 1), np.uint8)
            buf[:block.size] = block
            out = np.zeros(max(cap, 1), np.uint8)
            f = self.L.zxc_decompress_block_safe if safe else self.L.zxc_decompress_block
            r = f(c, buf.ctypes.data, block.size, out.ctypes.data, cap, C.byref(o) if o is not None else None)
            return r, (out[:r].tobytes() if r > 0 else None)
        finally:
            self.L.zxc_free_dctx(c)


class Dev:
    """the two batch calls through the C ABI with torch buffers: every dst has GUARD bytes of 0xA5 on either side,
    every src GUARD readable bytes behind it, and the scratch GUARD bytes of 0x5A behind it"""

    def __init__(self, prod):
        import torch
        self.t = torch
        self.L = bind(prod.lib)

    def upload(self, srcs, caps, src_off=0, dst_off=0):
        """srcs: bytes-like (None: a NULL src of 0 bytes; ("null", n): a NULL src of n bytes); caps: capacities
        (("null", c): a NULL dst of capacity c)"""
        t = self.t
        keep, dsts, desc = [], [], []
        for s, c in zip(srcs, caps):
            if s is None or isinstance(s, tuple):
                sp, n = 0, (s[1] if s else 0)
            else:
                a = np.frombuffer(bytes(s), np.uint8)
                buf = t.zeros(src_off + a.size + GUARD, dtype=t.uint8, device="cuda")
                if a.size:
                    buf[src_off:src_off + a.size].copy_(t.from_numpy(a.copy()))
                keep.append(buf)
                sp, n = buf.data_ptr() + src_off, a.size
            null_dst = isinstance(c, tuple)
            cap = c[1] if null_dst else c
            dd = t.full((dst_off + cap + 2 * GUARD,), 0xA5, dtype=t.uint8, device="cuda")
            dsts.append((dd, cap))
            desc.append([sp, n, 0 if null_dst else dd.data_ptr() + GUARD + dst_off, cap])
        return keep, dsts, t.tensor(desc, dtype=t.int64).reshape(-1, 4).cuda()

    def enqueue(self, kind, desc, n, o, scratch, results, size, safe=0, stream=None):
        st = stream.cuda_stream if stream is not None else None
        ob = C.byref(o) if o is not None else None
        if kind == "c":
            return self.L.zxc_b200_compress_blocks_device(desc.data_ptr(), n, ob, scratch.data_ptr(), size,
                                                          results.data_ptr(), st)
        return self.L.zxc_b200_decompress_blocks_device(desc.data_ptr(), n, ob, safe, scratch.data_ptr(), size,
                                                        results.data_ptr(), st)

    def csize(self, srcs, o):
        sizes = [len(s) if s is not None and not isinstance(s, tuple) else 0 for s in srcs]
        return int(self.L.zxc_b200_compress_blocks_device_scratch_size(len(srcs), sum(sizes),
                                                                       min(max(sizes + [1]), MIB2),
                                                                       C.byref(o) if o is not None else None))

    def dsize(self, caps):
        return int(self.L.zxc_b200_decompress_blocks_device_scratch_size(
            len(caps), max(c[1] if isinstance(c, tuple) else c for c in caps)))

    def run(self, kind, srcs, caps, o, safe=0, src_off=0, dst_off=0, scratch_size=None):
        """-> list of (result, bytes); checks the guards around every dst and behind the scratch"""
        t = self.t
        keep, dsts, desc = self.upload(srcs, caps, src_off, dst_off)
        if scratch_size is None:
            scratch_size = self.csize(srcs, o) if kind == "c" else self.dsize(caps)
        assert scratch_size > 0
        scratch = t.full((scratch_size + GUARD,), 0x5A, dtype=t.uint8, device="cuda")
        results = t.full((len(srcs),), 12345, dtype=t.int64, device="cuda")
        rc = self.enqueue(kind, desc, len(srcs), o, scratch, results, scratch_size, safe)
        assert rc == 0, rc
        t.cuda.synchronize()
        assert bool((scratch[scratch_size:] == 0x5A).all()), "scratch guard"
        out = []
        for i, (dd, cap) in enumerate(dsts):
            a = dd.cpu().numpy()
            lo, hi = GUARD + dst_off, GUARD + dst_off + cap
            assert (a[:lo] == 0xA5).all() and (a[hi:] == 0xA5).all(), ("dst guard", i)
            r = int(results[i].item())
            if kind == "c" and r <= 0:
                assert (a == 0xA5).all(), ("a failing item wrote its dst", i, r)
            out.append((r, a[lo:lo + r].tobytes() if r > 0 else None))
        return out


@pytest.fixture(scope="module")
def dev(prod):
    if not has_cuda():
        pytest.skip("needs a CUDA device")
    return Dev(prod)


@pytest.fixture(scope="module")
def host(prod):
    return Host(prod.lib)


def mixed_inputs(seed=0):
    rng = np.random.default_rng(seed)
    text = zc.silesia_shaped(MIB2 + 8192, seed=31 + seed)
    out = []
    for i, n in enumerate((1, 5, 31, 4095, 4096, 4097, 65536, 100000, MIB2)):
        kind = ("text", "random", "runs")[i % 3]
        if kind == "text":
            out.append(text[i:i + n].tobytes())
        elif kind == "random":
            out.append(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
        else:
            out.append(make_case("runs", n).tobytes() if n > 64 else bytes([7]) * n)
    return out


def bound(n):
    return n + 8 + 68 + 4


def check_compress(dev, host, srcs, caps, o, ref=None, **kw):
    got = dev.run("c", srcs, caps, o, **kw)
    for i, (s, c) in enumerate(zip(srcs, caps)):
        want = host.compress(np.frombuffer(s, np.uint8), c, o)
        assert got[i] == want, (i, len(s), got[i][0], want[0])
        if ref is not None and want[0] > 0:
            assert Host(ref.lib).compress(np.frombuffer(s, np.uint8), c, o) == want, ("reference", i)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("level", range(1, 8))
def test_mixed_batch_per_level(dev, host, libs, level):
    ref = libs[2]
    srcs = mixed_inputs(level)
    caps = [bound(len(s)) for s in srcs]
    for cks in (0, 1):
        o = opts(level, cks=cks)
        got = check_compress(dev, host, srcs, caps, o, ref)
        # and back through the batched decode, plain and safe
        blocks = [b for _, b in got]
        for safe in (0, 1):
            back = dev.run("d", blocks, [len(s) for s in srcs], dopts(cks), safe=safe)
            assert [r for r, _ in back] == [len(s) for s in srcs]
            assert [b for _, b in back] == srcs


@pytest.mark.gpu
def test_default_options_and_dictionary(dev, host, ref):
    data = zc.records(512, 4096, seed=5)
    d = zc.train_dict_ref(ref, data, n_samples=256)
    srcs = [data[i * 4096:(i + 1) * 4096].tobytes() for i in range(512)]
    caps = [bound(4096)] * 512
    check_compress(dev, host, srcs[:8], caps[:8], None)  # opts NULL: level 3, no checksum
    for level in (3, 5, 6):
        for cks in (0, 1):
            o = opts(level, cks=cks, d=d)
            got = check_compress(dev, host, srcs[:64], caps[:64], o, ref)
            blocks = [b for _, b in got]
            back = dev.run("d", blocks, [4096] * 64, dopts(cks, d))
            assert [b for _, b in back] == srcs[:64]
            for i in (0, 17, 63):
                assert host.decompress(blocks[i], 4096, dopts(cks, d), 0) == back[i]


@pytest.mark.gpu
def test_compress_verdicts_among_neighbours(dev, host):
    text = zc.silesia_shaped(1 << 20, seed=8)
    a = text[:50000].tobytes()
    size = host.compress(np.frombuffer(a, np.uint8), bound(len(a)), opts(3, cks=1))[0]
    srcs = [a, ("null", 100), a, b"", bytes(MIB2 + 1), a, a, a, a]
    caps = [bound(len(a)), 200, ("null", 100), 100, bound(MIB2), size, size - 1, 8, bound(len(a))]
    o = opts(3, cks=1)
    got = dev.run("c", srcs, caps, o)
    want = [size, NULL_INPUT, NULL_INPUT, NULL_INPUT, BAD_BS, size, DST_TOO_SMALL, DST_TOO_SMALL, size]
    assert [r for r, _ in got] == want
    assert got[0][1] == got[5][1] == got[8][1]


@pytest.mark.gpu
def test_decompress_verdicts_among_neighbours(dev, host):
    text = zc.silesia_shaped(1 << 20, seed=9)
    a = text[:60000].tobytes()
    o = opts(4, cks=1)
    blk = host.compress(np.frombuffer(a, np.uint8), bound(len(a)), o)[1]
    bad = bytearray(blk)
    bad[-1] ^= 0x55  # its checksum
    d = bytes(text[200000:216384])
    dblk = host.compress(np.frombuffer(a, np.uint8), bound(len(a)), opts(4, d=d))[1]
    n = len(a)
    for safe in (0, 1):
        lim = MIB2 if safe else MIB2 + TAIL_PAD
        srcs = [blk, ("null", len(blk)), blk, blk[:7], blk, blk, blk, blk, bytes(bad), dblk, blk]
        caps = [n, n, ("null", n), n, lim, lim + 1, n, n - 1, n, n, 0]
        for cks in (0, 1):
            got = dev.run("d", srcs, caps, dopts(cks), safe=safe)
            for i, (s, c) in enumerate(zip(srcs, caps)):
                if isinstance(s, tuple) or isinstance(c, tuple):
                    assert got[i][0] == NULL_INPUT
                    continue
                want = host.decompress(s, c, dopts(cks), safe)
                assert got[i] == want, (safe, cks, i, got[i][0], want[0])
            assert got[0] == (n, a)
            assert got[5][0] == BAD_BS and got[4][0] == n
            assert got[8][0] == (n if not cks else host.decompress(bytes(bad), n, dopts(1), safe)[0])
            assert got[9][0] < 0  # its dictionary is missing


@pytest.mark.gpu
def test_damaged_blocks_match_the_host_call(dev, host):
    rng = np.random.default_rng(3)
    text = zc.silesia_shaped(1 << 20, seed=10)
    blocks, caps = [], []
    for level in (1, 2, 3, 5, 6, 7):
        for n in (300, 4096, 20000):
            src = text[level * 1000:level * 1000 + n]
            b = bytearray(host.compress(src, bound(n), opts(level))[1])
            for k in range(6):
                m = bytearray(b)
                if k == 0:
                    m = m[:len(m) - 1 - int(rng.integers(0, 16))]  # truncated
                else:
                    for _ in range(k):
                        m[int(rng.integers(0, len(m)))] ^= int(rng.integers(1, 256))
                blocks.append(bytes(m))
                caps.append(n if k % 2 else n + int(rng.integers(0, 5000)))
    for safe in (0, 1):
        got = dev.run("d", blocks, caps, dopts(0), safe=safe)
        for i, (b, c) in enumerate(zip(blocks, caps)):
            assert got[i] == host.decompress(b, c, dopts(0), safe), (safe, i)


@pytest.mark.gpu
def test_unaligned_items(dev, host):
    srcs = mixed_inputs(11)[:8]
    o = opts(5, cks=1)
    for off in (1, 3, 15):
        got = check_compress(dev, host, srcs, [bound(len(s)) for s in srcs], o, src_off=off, dst_off=off)
        back = dev.run("d", [b for _, b in got], [len(s) for s in srcs], dopts(1), src_off=off, dst_off=off)
        assert [b for _, b in back] == srcs


@pytest.mark.gpu
def test_scratch_rules(dev, host):
    L = dev.L
    text = zc.silesia_shaped(1 << 20, seed=12)
    srcs = [text[i * 5000:i * 5000 + 3000 + 27 * i].tobytes() for i in range(40)]
    caps = [bound(len(s)) for s in srcs]
    o = opts(3)
    full = dev.csize(srcs, o)
    want = check_compress(dev, host, srcs, caps, o)
    # below the full size: the same bytes from fewer warps, down to the minimum
    minimum = int(L.zxc_b200_compress_blocks_device_scratch_size(40, 0, 0, C.byref(o)))
    pool = sum(((n + 64 + 255) // 256 + (n + 12 + 255) // 256) * 256 for n in map(len, srcs))
    for size in (full - 1000000, minimum + pool + 600000):
        assert dev.run("c", srcs, caps, o, scratch_size=size) == want
    # the pool running out: MEMORY from the first item that no longer fits, in index order
    got = dev.run("c", srcs, caps, o, scratch_size=minimum + pool // 2)
    rs = [r for r, _ in got]
    k = rs.index(MEMORY)
    assert 0 < k < 40 and all(r == MEMORY for r in rs[k:]) and got[:k] == want[:k]
    # a large item that no longer fits with its encode slot: it and every later one get MEMORY
    big = text[:MIB2].tobytes()
    got = dev.run("c", srcs[:3] + [big] + srcs[3:6], caps[:3] + [bound(MIB2)] + caps[3:6], o,
                  scratch_size=dev.csize(srcs[:6], o) + MIB2)
    assert [r for r, _ in got] == [w for w, _ in want[:3]] + [MEMORY] * 4
    # below the minimum
    keep, dsts, desc = dev.upload(srcs, caps)
    t = dev.t
    scr = t.empty(minimum, dtype=t.uint8, device="cuda")
    res = t.zeros(40, dtype=t.int64, device="cuda")
    assert dev.enqueue("c", desc, 40, o, scr, res, minimum - 1) == MEMORY
    assert dev.enqueue("c", desc, 40, o, scr, res, minimum) == 0
    t.cuda.synchronize()
    # decompress: items above the scratch's block size get MEMORY; below the minimum the call does
    blocks = [b for _, b in want]
    dcaps = [len(s) for s in srcs]
    dcaps[5] = 8192
    small = int(L.zxc_b200_decompress_blocks_device_scratch_size(40, 4096))
    got = dev.run("d", blocks, dcaps, dopts(0), scratch_size=small)
    assert [r for r, _ in got] == [len(s) if i != 5 else MEMORY for i, s in enumerate(srcs)]
    keep, dsts, desc = dev.upload(blocks, dcaps)
    scr = t.empty(small, dtype=t.uint8, device="cuda")
    assert dev.enqueue("d", desc, 40, dopts(0), scr, res, small - 1) == MEMORY


@pytest.mark.gpu
def test_many_records_with_a_dictionary(dev, host, ref):
    n = 65536
    data = zc.records(n, 4096, seed=13)
    d = zc.train_dict_ref(ref, data)
    srcs = [data[i * 4096:(i + 1) * 4096].tobytes() for i in range(n)]
    o = opts(5, d=d)
    got = dev.run("c", srcs, [bound(4096)] * n, o)
    for i in range(0, n, 4099):
        assert got[i] == host.compress(np.frombuffer(srcs[i], np.uint8), bound(4096), o), i
    blocks = [b for _, b in got]
    back = dev.run("d", blocks, [4096] * n, dopts(0, d))
    assert all(r == 4096 for r, _ in back)
    assert b"".join(b for _, b in back) == data.tobytes()


@pytest.mark.gpu
def test_two_streams_graph_and_launches(dev, host):
    t, L = dev.t, dev.L
    text = zc.silesia_shaped(1 << 20, seed=14)
    srcs = [text[i * 7000:i * 7000 + 6000 + i].tobytes() for i in range(6)]
    other = [s[::-1] for s in srcs]
    caps = [bound(len(s)) for s in srcs]
    o = opts(3, cks=1)
    want = [host.compress(np.frombuffer(s, np.uint8), c, o) for s, c in zip(srcs, caps)]
    want2 = [host.compress(np.frombuffer(s, np.uint8), c, o) for s, c in zip(other, caps)]
    s1, s2 = t.cuda.Stream(), t.cuda.Stream()
    runs = []
    for x in (srcs, other):
        keep, dsts, desc = dev.upload(x, caps)
        scr = t.empty(dev.csize(x, o), dtype=t.uint8, device="cuda")
        runs.append((keep, dsts, desc, scr, t.zeros(6, dtype=t.int64, device="cuda")))
    t.cuda.synchronize()
    for (keep, dsts, desc, scr, res), s in zip(runs, (s1, s2)):
        assert dev.enqueue("c", desc, 6, o, scr, res, scr.numel(), stream=s) == 0
    t.cuda.synchronize()
    for (keep, dsts, desc, scr, res), w in zip(runs, (want, want2)):
        assert res.tolist() == [r for r, _ in w]
        for (dd, cap), (r, b) in zip(dsts, w):
            assert dd[GUARD:GUARD + r].cpu().numpy().tobytes() == b
    # launches: 5 per compress call, 4 + k (2 + c) per decompress call, whatever the batch
    keep, dsts, desc, scr, res = runs[0]
    c0 = L.zxc_b200_launch_count()
    assert dev.enqueue("c", desc, 6, o, scr, res, scr.numel()) == 0
    assert dev.enqueue("c", desc, 2, o, scr, res, scr.numel()) == 0
    assert L.zxc_b200_launch_count() - c0 == 10
    blocks = [b for _, b in want]
    bk, bd, bdesc = dev.upload(blocks, [len(s) for s in srcs])
    for cks, cap_max, k in ((0, 4096, 1), (1, 8192, 2), (0, 65536, 5)):
        dsz = int(L.zxc_b200_decompress_blocks_device_scratch_size(6, cap_max))
        dscr = t.empty(dsz, dtype=t.uint8, device="cuda")
        c0 = L.zxc_b200_launch_count()
        assert dev.enqueue("d", bdesc, 6, dopts(cks), dscr, res, dsz) == 0
        assert L.zxc_b200_launch_count() - c0 == 4 + k * (2 + cks)
    t.cuda.synchronize()
    # graph capture, then replay with rewritten descriptors and inputs
    s = t.cuda.Stream()
    g = t.cuda.CUDAGraph()
    t.cuda.synchronize()
    with t.cuda.graph(g, stream=s):
        assert dev.enqueue("c", desc, 6, o, scr, res, scr.numel(), stream=s) == 0
    for dd, cap in dsts:
        dd[GUARD:GUARD + cap].fill_(0)
    g.replay()
    t.cuda.synchronize()
    assert res.tolist() == [r for r, _ in want]
    keep[0].copy_(t.from_numpy(np.frombuffer(other[0] + bytes(GUARD), np.uint8).copy()))
    desc[1, 1] = 100  # a shorter input
    desc[2, 3] = 10  # a capacity the block does not fit
    res.fill_(0)
    g.replay()
    t.cuda.synchronize()
    w100 = host.compress(np.frombuffer(srcs[1][:100], np.uint8), caps[1], o)
    assert res.tolist() == [want2[0][0], w100[0], DST_TOO_SMALL] + [r for r, _ in want[3:]]
    assert dsts[1][0][GUARD:GUARD + w100[0]].cpu().numpy().tobytes() == w100[1]


@pytest.mark.gpu
def test_python_helpers(prod):
    if not has_cuda():
        pytest.skip("needs a CUDA device")
    import torch
    from zxc_b200 import device as D
    text = zc.silesia_shaped(1 << 20, seed=15)
    srcs = [torch.from_numpy(text[i * 9000:i * 9000 + 1000 + 313 * i].copy()).cuda() for i in range(10)]
    outs, res = D.compress_blocks(srcs, level=5, checksum=True)
    torch.cuda.synchronize()
    rs = res.tolist()
    assert all(r > 0 for r in rs)
    assert [o.numel() for o in outs] == [int(prod.lib.zxc_compress_block_bound(s.numel())) for s in srcs]
    blocks = [o[:r] for o, r in zip(outs, rs)]
    back, res2 = D.decompress_blocks(blocks, [s.numel() for s in srcs], checksum=True, safe=True,
                                     stream=torch.cuda.Stream())
    torch.cuda.synchronize()
    assert res2.tolist() == [s.numel() for s in srcs]
    assert all(torch.equal(a, b) for a, b in zip(back, srcs))
    with pytest.raises(ValueError):
        D.compress_blocks([])
    with pytest.raises(ValueError):
        D.compress_blocks([srcs[0], srcs[1].cpu()])
    with pytest.raises(ValueError):
        D.decompress_blocks(blocks, [1])
    with pytest.raises(ValueError):
        D.decompress_blocks(blocks[:1], [5], out=[torch.empty(4, dtype=torch.uint8, device="cuda")])
    with pytest.raises(D.ZxcError) as e:
        D.compress_blocks(srcs[:1], dict=bytes(70000))
    assert e.value.code == DICT_BIG
