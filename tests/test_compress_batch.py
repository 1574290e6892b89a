"""zxc_b200_compress_device_batch: many buffers in HBM compressed into one frame each in one call.

Every frame's result and bytes must equal zxc_b200_compress_device's for that buffer alone with the same options and
capacity, zxc_compress's, and the reference's where it is built; every frame decodes back with zxc_decompress and
with zxc_b200_decompress_device_batch."""
import ctypes as C

import numpy as np
import pytest

import zxc_corpus as zc
import zxc_ctypes as z
from conftest import has_cuda
from test_compress_device import bind, opts
from test_oracle import golden_dicts, make_case

NULL_INPUT, DST_TOO_SMALL, CORRUPT, BAD_BS, DICT_BIG, MEMORY, NO_DEVICE = -12, -2, -8, -14, -17, -1, -100
GUARD = 64
HDR, EOF, FOOT, SEK_HDR = 16, 8, 12, 8


def bind_batch(L):
    bind(L)
    L.zxc_b200_compress_device_batch_scratch_size.restype = C.c_size_t
    L.zxc_b200_compress_device_batch_scratch_size.argtypes = [C.c_uint32, C.c_uint64, C.c_void_p]
    L.zxc_b200_compress_device_batch.restype = C.c_int
    L.zxc_b200_compress_device_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t,
                                                 C.c_void_p, C.c_void_p]
    L.zxc_compress_bound.restype = C.c_uint64
    L.zxc_compress_bound.argtypes = [C.c_size_t]
    return L


def test_host_verdicts_without_a_device(prod):
    """The whole-call verdicts come in order without a device; the size query is 0."""
    if has_cuda():
        pytest.skip("only meaningful without a GPU")
    L = bind_batch(prod.lib)
    fake = 1 << 40  # never dereferenced
    cb = L.zxc_b200_compress_device_batch
    assert cb(None, 1, None, fake, 1 << 20, fake, None) == NULL_INPUT
    assert cb(fake, 1, None, None, 1 << 20, fake, None) == NULL_INPUT
    assert cb(fake, 1, None, fake, 1 << 20, None, None) == NULL_INPUT
    big = opts(3, 3000, d=b"x" * 70000)  # dictionary first, then block size
    assert cb(fake, 1, C.byref(big), fake, 1 << 20, fake, None) == DICT_BIG
    assert cb(None, 0, C.byref(big), None, 0, None, None) == DICT_BIG
    assert cb(fake, 1, C.byref(opts(3, 3000)), fake, 1 << 20, fake, None) == BAD_BS
    assert cb(fake, 1, C.byref(opts(3, 1 << 22)), fake, 1 << 20, fake, None) == BAD_BS
    assert cb(fake, 1, C.byref(opts(3, 65536, h=bytes(128))), fake, 0, fake, None) == NO_DEVICE
    assert cb(None, 0, None, None, 0, None, None) == NO_DEVICE
    assert L.zxc_b200_compress_device_batch_scratch_size(10, 1 << 20, None) == 0
    assert L.zxc_b200_compress_device_batch_scratch_size(10, 1 << 20, C.byref(opts(3, 5000))) == 0


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
def _bound(L, n):
    return int(L.zxc_compress_bound(n))


def _fixed(n, bs, seek):
    nb = -(-n // bs)
    return HDR + EOF + (SEK_HDR + 4 * nb if seek and nb else 0) + FOOT


class Batch:
    """the batch call through the C ABI with torch buffers; every dst has GUARD bytes of 0xA5 on either side, the
    scratch GUARD bytes of 0x5A behind it"""

    def __init__(self, prod):
        import torch
        self.t = torch
        self.L = bind_batch(prod.lib)

    def scratch_size(self, n, total, o):
        return int(self.L.zxc_b200_compress_device_batch_scratch_size(n, total, C.byref(o)))

    def upload(self, datas, caps, src_off=0, dst_off=0):
        """datas: numpy inputs (("null", n): a NULL src of n bytes); caps: capacities (None: the bound; ("null", c):
        a NULL dst of capacity c)"""
        t = self.t
        srcs, dsts, desc = [], [], []
        for d, c in zip(datas, caps):
            if isinstance(d, tuple):
                s, sp, n = None, 0, d[1]
            else:
                d = np.asarray(d, np.uint8)
                s = t.empty(src_off + d.size, dtype=t.uint8, device="cuda")  # the input ends where its tensor ends
                if d.size:
                    s[src_off:].copy_(t.from_numpy(d.copy()))
                sp, n = (s.data_ptr() + src_off if d.size else 0), d.size
            null_dst = isinstance(c, tuple)
            cap = c[1] if null_dst else (_bound(self.L, n) if c is None else c)
            dd = t.full((dst_off + cap + 2 * GUARD,), 0xA5, dtype=t.uint8, device="cuda")
            srcs.append(s)
            dsts.append((dd, cap))
            desc.append([sp, n, 0 if null_dst else dd.data_ptr() + GUARD + dst_off, cap])
        return srcs, dsts, t.tensor(desc, dtype=t.int64).reshape(-1, 4).cuda()

    def enqueue(self, desc, n, o, scratch, results, scratch_size, stream=None):
        return self.L.zxc_b200_compress_device_batch(
            desc.data_ptr(), n, C.byref(o) if o is not None else None, scratch.data_ptr(), scratch_size,
            results.data_ptr(), stream.cuda_stream if stream is not None else None)

    def run(self, datas, caps, o, src_off=0, dst_off=0, scratch_size=None):
        """-> list of (result, frame bytes); checks the guards around every dst and behind the scratch"""
        t = self.t
        srcs, dsts, desc = self.upload(datas, caps, src_off, dst_off)
        total = sum(d[1] if isinstance(d, tuple) else np.asarray(d).size for d in datas)
        size = self.scratch_size(len(datas), total, o) if scratch_size is None else scratch_size
        assert size > 0
        scratch = t.full((size + GUARD,), 0x5A, dtype=t.uint8, device="cuda")
        results = t.full((len(datas),), 12345, dtype=t.int64, device="cuda")
        rc = self.enqueue(desc, len(datas), o, scratch, results, size)
        assert rc == 0, rc
        t.cuda.synchronize()
        assert bool((scratch[size:] == 0x5A).all()), "scratch guard"
        out = []
        for i, (dd, cap) in enumerate(dsts):
            a = dd.cpu().numpy()
            lo, hi = GUARD + dst_off, GUARD + dst_off + cap
            assert (a[:lo] == 0xA5).all() and (a[hi:] == 0xA5).all(), ("dst guard", i)
            r = int(results[i].item())
            if r <= 0:
                assert (a == 0xA5).all(), ("a failing frame wrote its dst", i, r)
            out.append((r, a[lo:lo + r] if r > 0 else None))
        return out

    def single(self, data, cap, o):
        """zxc_b200_compress_device alone: its return code, or its *d_result and frame"""
        t = self.t
        if isinstance(data, tuple):
            n, sp, keep = data[1], None, None
        else:
            n = data.size
            keep = t.from_numpy(np.asarray(data, np.uint8).copy()).cuda() if n else None
            sp = keep.data_ptr() if n else None
        null_dst = isinstance(cap, tuple)
        cap = cap[1] if null_dst else (_bound(self.L, n) if cap is None else cap)
        dst = t.zeros(max(cap, 1), dtype=t.uint8, device="cuda")
        size = int(self.L.zxc_b200_encode_scratch_size(n, C.byref(o)))
        scratch = t.empty(max(size, 1), dtype=t.uint8, device="cuda")
        res = t.zeros(1, dtype=t.int64, device="cuda")
        rc = self.L.zxc_b200_compress_device(sp, n, None if null_dst else dst.data_ptr(), cap, C.byref(o),
                                             scratch.data_ptr(), size, res.data_ptr(), None, None)
        if rc != 0:
            return rc, None
        t.cuda.synchronize()
        r = int(res.item())
        return r, (dst[:r].cpu().numpy() if r > 0 else None)

    def check(self, prod, datas, caps, level=3, bs=65536, cks=0, seek=0, d=None, h=None, ref=None, what=None, **kw):
        o = opts(level, bs, cks, seek, d, h)
        got = self.run(datas, caps, o, **kw)
        for i, ((r, fr), data, cap) in enumerate(zip(got, datas, caps)):
            r1, f1 = self.single(data, cap, o)
            assert r == r1, (what, i, z.ERR.get(r, r), z.ERR.get(r1, r1))
            if r <= 0:
                continue
            assert np.array_equal(fr, f1), (what, i)
            want = prod.compress(data, level=level, block_size=bs, checksum=cks, seekable=seek, dict=d, dict_huf=h)
            assert np.array_equal(fr, want), (what, i, "zxc_compress")
            if ref is not None:
                rf = ref.compress(data, level=level, block_size=bs, checksum=cks, seekable=seek, dict=d, dict_huf=h)
                assert np.array_equal(fr, rf), (what, i, "reference")
            r0, o0 = prod.decompress(fr, data.size, checksum=cks, dict=d, dict_huf=h)
            assert r0 == data.size and np.array_equal(o0, data), (what, i, "decodes")
        return got


@pytest.fixture(scope="module")
def batch(prod):
    return Batch(prod)


def _ref():
    return z.ZxcLib(z.REF_SO) if z.have_ref() else None


def _inputs(bs, seed, big=3):
    rng = np.random.default_rng(seed)
    out = []
    for kind in ("random", "text", "zero"):
        for n in (0, 1, 15, 16, bs - 1, bs, bs + 1, big * bs + 77):
            if kind == "random":
                out.append(rng.integers(0, 256, n, dtype=np.uint8))
            elif kind == "zero":
                out.append(np.zeros(n, np.uint8))
            else:
                out.append(make_case("text", n) if n else np.zeros(0, np.uint8))
    return out


def _decode_batch(frames, sizes, cks=False, d=None, h=None):
    import torch as t
    from zxc_b200 import device as zd
    outs, res = zd.decompress_frames([t.from_numpy(f.copy()).cuda() for f in frames], sizes, checksum=cks, dict=d,
                                     dict_huf=h)
    return res.tolist(), [o.cpu().numpy() for o in outs]


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, 2, 3, 4, 5, 6, 7])
def test_levels_in_one_mixed_batch(batch, prod, level):
    ref = _ref()
    for bs, cks, seek in ((65536, level % 2, (level // 2) % 2), (4096, 1 - level % 2, 1 - (level // 2) % 2)):
        datas = _inputs(bs, level, big=3 if bs == 65536 else 5)
        got = batch.check(prod, datas, [None] * len(datas), level, bs, cks, seek, ref=ref, what=(level, bs))
        rs, outs = _decode_batch([f for _, f in got], [x.size for x in datas], cks=bool(cks))
        assert rs == [x.size for x in datas]
        assert all(np.array_equal(o, x) for o, x in zip(outs, datas))


@pytest.mark.gpu
def test_block_sizes_checksums_seekable(batch, prod):
    ref = _ref()
    data = zc.silesia_shaped(8 << 20, seed=6)
    for bs in (4096, 65536, 2 << 20):
        sizes = (0, 1, bs - 1, bs, bs + 1, 2 * bs + 3) if bs < (2 << 20) else (0, 100, bs + 1)
        datas = [data[:n].copy() for n in sizes]
        for cks in (0, 1):
            for seek in (0, 1):
                batch.check(prod, datas, [None] * len(datas), 3 if bs > 65536 else 2 + cks + 2 * seek, bs, cks, seek,
                            ref=ref, what=(bs, cks, seek))


@pytest.mark.gpu
@pytest.mark.parametrize("level", [5, 6, 7])
def test_dictionaries(batch, prod, level):
    ref = _ref()
    (d, h) = list(golden_dicts().values())[0]
    datas = [make_case("text", n) for n in (100, 5000, 70000, 150000)] + [np.zeros(0, np.uint8)]
    for hh in (h, None):
        got = batch.check(prod, datas, [None] * len(datas), level, 65536, 1, level % 2, d, hh, ref=ref)
        rs, outs = _decode_batch([f for _, f in got], [x.size for x in datas], True, d, hh)
        assert rs == [x.size for x in datas] and all(np.array_equal(o, x) for o, x in zip(outs, datas))
    t = batch.t
    srcs, dsts, desc = batch.upload(datas, [None] * len(datas))
    o = opts(level, 65536, 1, 0, d, bytes([0x11]) * 128)  # a malformed table: the whole call
    scratch = t.empty(batch.scratch_size(len(datas), 10 ** 6, opts(level, 65536, 1, 0, d)), dtype=t.uint8,
                      device="cuda")
    res = t.full((len(datas),), 7, dtype=t.int64, device="cuda")
    assert batch.enqueue(desc, len(datas), o, scratch, res, scratch.numel()) == CORRUPT
    assert res.tolist() == [7] * len(datas)


@pytest.mark.gpu
def test_per_frame_verdicts_among_healthy_neighbours(batch, prod):
    """each verdict equals the single call's, and every neighbour keeps its frame"""
    data = make_case("text", 50000)
    bs = 4096
    fr = prod.compress(data, level=3, block_size=bs, checksum=1, seekable=1)
    fixed = _fixed(data.size, bs, 1)
    cases = [(("null", 100), None), (data, ("null", 1000)), (data, 0), (data, fixed - 1), (data, fr.size),
             (data, fr.size - 1), (data, fixed)]
    datas, caps = [], []
    for dd, cc in cases:
        datas += [data, dd]
        caps += [None, cc]
    datas.append(data)
    caps.append(None)
    got = batch.check(prod, datas, caps, 3, bs, 1, 1)
    rs = [r for r, _ in got]
    assert rs[1::2] == [NULL_INPUT, NULL_INPUT, NULL_INPUT, DST_TOO_SMALL, fr.size, DST_TOO_SMALL, DST_TOO_SMALL]
    assert rs[0::2] == [fr.size] * 8


@pytest.mark.gpu
@pytest.mark.parametrize("off", [1, 3, 15])
def test_unaligned_buffers(batch, prod, off):
    datas = [make_case("text", n) for n in (70000, 5, 4096 * 3)] + [zc.silesia_shaped(1 << 20, seed=1)[:200001]]
    batch.check(prod, datas, [None] * 4, 3, 4096, 1, 1, src_off=off, dst_off=(off * 7) % 16)
    batch.check(prod, datas, [None] * 4, 6, 65536, 0, 0, src_off=off, dst_off=off)


def _share(n, bs):
    return 0 if n == 0 else -(-(n + 64) // 256) * 256 + -(-n // bs) * ((bs + 80 + 255) // 256 * 256)


@pytest.mark.gpu
def test_scratch(batch, prod):
    """the size function's scratch, one that holds one warp, one byte below the minimum, and the pool overflow in
    index order (frames that fail their checks take no share)"""
    t = batch.t
    bs = 4096
    data = zc.silesia_shaped(1 << 20, seed=12)[:300000]
    datas = [data[:n].copy() for n in (300000, 70000, 0, 9000, 120000)]
    o = opts(3, bs, 1, 1)
    full = batch.run(datas, [None] * 5, o)
    assert all(r > 0 for r, _ in full)
    need = sum(_share(x.size, bs) for x in datas)
    lo = batch.scratch_size(5, 0, o)
    one = lo + need + need * 12 // (bs + 80 + 255 + 256) + 1024  # the pool for these shares, no second warp slot
    got = batch.run(datas, [None] * 5, o, scratch_size=one)
    assert [r for r, _ in got] == [r for r, _ in full]
    assert all(np.array_equal(a, b) for (_, a), (_, b) in zip(got, full))
    srcs, dsts, desc = batch.upload(datas, [None] * 5)
    scr = t.empty(lo, dtype=t.uint8, device="cuda")
    res = t.full((5,), 7, dtype=t.int64, device="cuda")
    assert batch.enqueue(desc, 5, o, scr, res, lo - 1) == MEMORY
    assert batch.enqueue(desc, 5, o, scr, res, lo) == 0
    t.cuda.synchronize()
    assert res.tolist() == [MEMORY] * 5  # the empty frame too: it comes after the first frame past the pool
    # a pool that holds the first two shares and the NULL frame's nothing, not the third
    datas2 = [datas[1], ("null", 500), datas[3], datas[0], datas[3], datas[2]]
    part = lo + (_share(70000, bs) + _share(9000, bs)) * 1.01 + 2048
    got = batch.run(datas2, [None] * 6, o, scratch_size=int(part))
    assert [r for r, _ in got] == [full[1][0], NULL_INPUT, full[3][0], MEMORY, MEMORY, MEMORY]
    assert np.array_equal(got[0][1], full[1][1]) and np.array_equal(got[2][1], full[3][1])


@pytest.mark.gpu
def test_many_small_frames(batch, prod):
    t = batch.t
    rng = np.random.default_rng(4)
    base = zc.silesia_shaped(1 << 20, seed=2)
    n = 100_000
    lens = rng.integers(100, 700, n)
    starts = rng.integers(0, base.size - 700, n)
    src = t.from_numpy(base).cuda()
    cap = 1024
    outs = t.full((n, cap), 0xA5, dtype=t.uint8, device="cuda")
    desc = t.stack([src.data_ptr() + t.from_numpy(starts).cuda(), t.from_numpy(lens).cuda(),
                    outs.data_ptr() + cap * t.arange(n, device="cuda"), t.full((n,), cap, device="cuda")], 1)
    o = opts(2, 4096, 1, 1)
    size = batch.scratch_size(n, int(lens.sum()), o)
    scratch = t.empty(size, dtype=t.uint8, device="cuda")
    res = t.zeros(n, dtype=t.int64, device="cuda")
    assert batch.enqueue(desc.contiguous(), n, o, scratch, res, size) == 0
    r = res.cpu().numpy()
    a = outs.cpu().numpy()
    for i in list(range(0, n, 997)) + [n - 1]:
        raw = base[starts[i]:starts[i] + lens[i]]
        want = prod.compress(raw, level=2, block_size=4096, checksum=1, seekable=1)
        assert r[i] == want.size and np.array_equal(a[i, :r[i]], want), i
    assert (r > 0).all()
    rs, back = _decode_batch([a[i, :r[i]] for i in range(0, n, 101)], [int(lens[i]) for i in range(0, n, 101)], True)
    assert rs == [int(lens[i]) for i in range(0, n, 101)]


@pytest.mark.gpu
def test_256_mib_frame_next_to_small_ones(batch, prod):
    t = batch.t
    from zxc_b200 import device as zd
    big = t.from_numpy(zc.silesia_shaped(64 << 20, seed=8)).cuda().repeat(4)
    small = t.from_numpy(make_case("text", 30000)).cuda()
    outs, res = zd.compress_frames([small, big, small], level=1, block_size=65536, checksum=True)
    fb = zd.compress(big, level=1, block_size=65536, checksum=True)
    fs = zd.compress(small, level=1, block_size=65536, checksum=True)
    r = res.tolist()
    assert r == [fs.frame.numel(), fb.frame.numel(), fs.frame.numel()]
    assert t.equal(outs[1][:r[1]], fb.frame) and t.equal(outs[0][:r[0]], fs.frame) and t.equal(outs[2][:r[2]], fs.frame)


@pytest.mark.gpu
def test_two_streams_graph_and_launches(batch, prod):
    t = batch.t
    data = make_case("text", 120000)
    other = data[::-1].copy()
    o = opts(3, 4096, 1, 1)
    want = prod.compress(data, level=3, block_size=4096, checksum=1, seekable=1)
    want2 = prod.compress(other, level=3, block_size=4096, checksum=1, seekable=1)
    s1, s2 = t.cuda.Stream(), t.cuda.Stream()
    runs = []
    for x in (data, other):
        srcs, dsts, desc = batch.upload([x] * 3, [None] * 3)
        scr = t.empty(batch.scratch_size(3, 3 * x.size, o), dtype=t.uint8, device="cuda")
        res = t.zeros(3, dtype=t.int64, device="cuda")
        runs.append((srcs, dsts, desc, scr, res))
    t.cuda.synchronize()
    for (srcs, dsts, desc, scr, res), s in zip(runs, (s1, s2)):
        assert batch.enqueue(desc, 3, o, scr, res, scr.numel(), stream=s) == 0
    t.cuda.synchronize()
    for (srcs, dsts, desc, scr, res), w in zip(runs, (want, want2)):
        assert res.tolist() == [w.size] * 3
        for dd, cap in dsts:
            assert np.array_equal(dd[GUARD:GUARD + w.size].cpu().numpy(), w)
    # graph capture, then replay with rewritten descriptors and inputs
    srcs, dsts, desc, scr, res = runs[0]
    s = t.cuda.Stream()
    g = t.cuda.CUDAGraph()
    t.cuda.synchronize()
    with t.cuda.graph(g, stream=s):
        assert batch.enqueue(desc, 3, o, scr, res, scr.numel(), stream=s) == 0
    for dd, cap in dsts:
        dd[GUARD:GUARD + cap].fill_(0)
    g.replay()
    t.cuda.synchronize()
    assert res.tolist() == [want.size] * 3
    assert np.array_equal(dsts[0][0][GUARD:GUARD + want.size].cpu().numpy(), want)
    srcs[0].copy_(t.from_numpy(other))  # rewritten input
    desc[1, 1] = 5000  # rewritten descriptor: a shorter input
    desc[2, 3] = 10  # and a capacity below header + trailer
    res.fill_(0)
    g.replay()
    t.cuda.synchronize()
    w5 = prod.compress(data[:5000], level=3, block_size=4096, checksum=1, seekable=1)
    assert res.tolist() == [want2.size, w5.size, DST_TOO_SMALL]
    assert np.array_equal(dsts[0][0][GUARD:GUARD + want2.size].cpu().numpy(), want2)
    assert np.array_equal(dsts[1][0][GUARD:GUARD + w5.size].cpu().numpy(), w5)
    # the fixed launch count: 12, plus the seeding kernel with a dictionary; nothing for n_frames == 0
    L = batch.L
    (d, h) = list(golden_dicts().values())[0]
    for n in (1, 7, 10_000):
        srcs, dsts, desc = batch.upload([data[:3000]], [None])
        desc = desc.repeat(n, 1)
        scr = t.empty(batch.scratch_size(n, 3000 * n, o), dtype=t.uint8, device="cuda")
        res = t.zeros(n, dtype=t.int64, device="cuda")
        before = L.zxc_b200_launch_count()
        assert batch.enqueue(desc, n, o, scr, res, scr.numel()) == 0
        assert L.zxc_b200_launch_count() - before == 12
        t.cuda.synchronize()
        assert (res[:1] > 0).all().item()
    od = opts(5, 4096, 1, 1, d, h)
    scr = t.empty(batch.scratch_size(1, 3000, od), dtype=t.uint8, device="cuda")
    before = L.zxc_b200_launch_count()
    assert batch.enqueue(desc[:1].contiguous(), 1, od, scr, res, scr.numel()) == 0
    assert L.zxc_b200_launch_count() - before == 13
    before = L.zxc_b200_launch_count()
    assert batch.enqueue(desc, 0, o, scr, res, 0) == 0
    assert L.zxc_b200_launch_count() == before
    t.cuda.synchronize()


@pytest.mark.gpu
def test_python_compress_frames(prod):
    import torch as t
    from zxc_b200 import device as zd
    data = [make_case("text", n) for n in (5000, 70000, 0, 200000)]
    srcs = [t.from_numpy(d).cuda() for d in data]
    outs, res = zd.compress_frames(srcs, level=4, block_size=4096, checksum=True, seekable=True)
    r = res.tolist()
    for o, d, k in zip(outs, data, r):
        want = prod.compress(d, level=4, block_size=4096, checksum=1, seekable=1)
        assert k == want.size and np.array_equal(o[:k].cpu().numpy(), want)
    back, rb = zd.decompress_frames([o[:k] for o, k in zip(outs, r)], checksum=True)
    assert rb.tolist() == [d.size for d in data]
    assert all(np.array_equal(b.cpu().numpy(), d) for b, d in zip(back, data))
    # a float tensor compresses its bytes; `out` on another stream
    f = t.arange(10000, dtype=t.float32, device="cuda")
    out = [t.empty(70000, dtype=t.uint8, device="cuda") for _ in range(2)]
    s = t.cuda.Stream()
    o2, r2 = zd.compress_frames([f, srcs[0]], level=1, out=out, stream=s)
    s.synchronize()
    assert all(a is b for a, b in zip(o2, out))
    want = prod.compress(f.cpu().numpy().view(np.uint8), level=1)
    assert r2[0].item() == want.size and np.array_equal(out[0][:want.size].cpu().numpy(), want)
    with pytest.raises(zd.ZxcError) as e:
        zd.compress_frames(srcs, dict=b"x" * 70000)
    assert e.value.code == DICT_BIG
    with pytest.raises(zd.ZxcError) as e:
        zd.compress_frames(srcs, block_size=5000)
    assert e.value.code == BAD_BS
    with pytest.raises(ValueError):
        zd.compress_frames([])
    with pytest.raises(ValueError):
        zd.compress_frames([srcs[0].cpu()])
    with pytest.raises(ValueError):
        zd.compress_frames([srcs[0][::2]])
    with pytest.raises(ValueError):
        zd.compress_frames(srcs, out=out)
    with pytest.raises(ValueError):
        zd.compress_frames(srcs[:2], out=[out[0], out[1].cpu()])
