"""zxc_b200_decompress_device_batch: many frames in HBM planned, decoded and checked in one call.

Every frame's result and bytes must equal zxc_b200_decompress_device's for that frame alone with a scratch sized for
(its capacity, the batch's block size), and zxc_decompress's (and the reference's, where built) apart from that call's
two ZXC_ERROR_MEMORY limits."""
import ctypes as C
import os

import numpy as np
import pytest

import zxc_corpus as zc
import zxc_ctypes as z
from conftest import has_cuda
from test_decompress_device import Dev, _mutants, _ref, _stitched, bind, dopts
from test_oracle import G, INVALID, VALID, golden_dicts, make_case

NULL_INPUT, SRC_SMALL, DICT_BIG, MEMORY, NO_DEVICE = -12, -3, -17, -1, -100
GUARD = 64


def bind_batch(L):
    bind(L)
    L.zxc_b200_decompress_device_batch_scratch_size.restype = C.c_size_t
    L.zxc_b200_decompress_device_batch_scratch_size.argtypes = [C.c_uint32, C.c_uint64, C.c_uint32]
    L.zxc_b200_decompress_device_batch.restype = C.c_int
    L.zxc_b200_decompress_device_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t,
                                                   C.c_void_p, C.c_void_p]
    return L


def test_host_verdicts_without_a_device(prod):
    """The whole-call verdicts come in order without a device; the size query is 0."""
    if has_cuda():
        pytest.skip("only meaningful without a GPU")
    L = bind_batch(prod.lib)
    fake = 1 << 40  # never dereferenced
    db = L.zxc_b200_decompress_device_batch
    assert db(None, 1, None, fake, 1 << 20, fake, None) == NULL_INPUT
    assert db(fake, 1, None, None, 1 << 20, fake, None) == NULL_INPUT
    assert db(fake, 1, None, fake, 1 << 20, None, None) == NULL_INPUT
    assert db(fake, 1, C.byref(dopts(d=b"x" * 70000)), fake, 1 << 20, fake, None) == DICT_BIG
    assert db(None, 0, C.byref(dopts(d=b"x" * 70000)), None, 0, None, None) == DICT_BIG
    assert db(fake, 1, C.byref(dopts(1)), fake, 0, fake, None) == NO_DEVICE
    assert db(None, 0, None, None, 0, None, None) == NO_DEVICE
    assert L.zxc_b200_decompress_device_batch_scratch_size(10, 1 << 20, 65536) == 0
    assert L.zxc_b200_decompress_device_batch_scratch_size(10, 1 << 20, 5000) == 0


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
class Batch:
    """the batch call through the C ABI with torch buffers; every dst has GUARD bytes of 0xA5 on either side"""

    def __init__(self, prod):
        import torch
        self.t = torch
        self.L = bind_batch(prod.lib)
        self.dev = Dev(prod)

    def scratch_size(self, n, total, bs):
        return int(self.L.zxc_b200_decompress_device_batch_scratch_size(n, total, bs))

    def upload(self, frames, caps, src_off=0):
        """frames: numpy frames (None: NULL src); caps: capacities (None: NULL dst with that capacity's entry)"""
        t = self.t
        srcs, dsts, desc = [], [], []
        for f, c in zip(frames, caps):
            if f is None:
                s, sp, n = None, 0, 0
            else:
                f = np.asarray(f, np.uint8)
                s = t.empty(src_off + max(f.size, 1), dtype=t.uint8, device="cuda")
                if f.size:
                    s[src_off:src_off + f.size].copy_(t.from_numpy(f.copy()))
                sp, n = s.data_ptr() + src_off, f.size
            cap, null_dst = (c[0], True) if isinstance(c, tuple) else (c, False)
            d = t.full((cap + 2 * GUARD,), 0xA5, dtype=t.uint8, device="cuda")
            srcs.append(s)
            dsts.append(d)
            desc.append([sp, n, 0 if null_dst else d.data_ptr() + GUARD, cap])
        return srcs, dsts, t.tensor(desc, dtype=t.int64).reshape(-1, 4).cuda()

    def enqueue(self, desc, n, o, scratch, results, stream=None, scratch_size=None):
        return self.L.zxc_b200_decompress_device_batch(
            desc.data_ptr(), n, C.byref(o) if o is not None else None, scratch.data_ptr(),
            scratch.numel() - GUARD if scratch_size is None else scratch_size, results.data_ptr(),
            stream.cuda_stream if stream is not None else None)

    def run(self, frames, caps, cks=0, d=None, h=None, bs=65536, src_off=0, total=None):
        """-> list of (result, output bytes); checks the guards around every dst and behind the scratch"""
        t = self.t
        srcs, dsts, desc = self.upload(frames, caps, src_off)
        plain = [c[0] if isinstance(c, tuple) else c for c in caps]
        size = self.scratch_size(len(frames), sum(plain) if total is None else total, bs)
        assert size > 0
        scratch = t.full((size + GUARD,), 0x5A, dtype=t.uint8, device="cuda")
        results = t.full((len(frames),), 12345, dtype=t.int64, device="cuda")
        rc = self.enqueue(desc, len(frames), dopts(cks, d, h), scratch, results)
        assert rc == 0, rc
        t.cuda.synchronize()
        assert bool((scratch[size:] == 0x5A).all()), "scratch guard"
        out = []
        for i, (dd, c) in enumerate(zip(dsts, plain)):
            a = dd.cpu().numpy()
            assert (a[:GUARD] == 0xA5).all() and (a[GUARD + c:] == 0xA5).all(), ("dst guard", i)
            r = int(results[i].item())
            out.append((r, a[GUARD:GUARD + r] if r > 0 else np.zeros(0, np.uint8)))
        return out

    def check(self, prod, frames, caps, cks=0, d=None, h=None, bs=65536, ref=None, what=None, **kw):
        """every frame's result and bytes against the single call (same opts, scratch for (cap, bs)) and
        zxc_decompress"""
        got = self.run(frames, caps, cks, d, h, bs, **kw)
        for i, (f, c) in enumerate(zip(frames, caps)):
            r, o = got[i]
            if f is None or isinstance(c, tuple):
                assert r == NULL_INPUT, (what, i, r)
                continue
            f = np.asarray(f, np.uint8)
            if f.size < 28:
                assert r == SRC_SMALL, (what, i, r)
                continue
            r1, o1 = self.dev.run(f, c, cks, d, h, bs=bs)
            assert r == r1, (what, i, z.ERR.get(r, r), z.ERR.get(r1, r1))
            if r > 0:
                assert np.array_equal(o, o1), (what, i)
            if r1 != MEMORY:
                r0, o0 = prod.decompress(f, c, checksum=cks, dict=d, dict_huf=h)
                assert r == r0, (what, i, r, r0)
                if r0 > 0:
                    assert np.array_equal(o, o0), (what, i)
                if ref is not None and r0 >= 0:
                    rr, orr = ref.decompress(f, c, checksum=cks, dict=d, dict_huf=h)
                    assert rr == r0 and (rr <= 0 or np.array_equal(orr, o0)), (what, i, "reference")
        return [r for r, _ in got]


@pytest.fixture(scope="module")
def batch(prod):
    return Batch(prod)


def _golden(dir_):
    for name in sorted(VALID if dir_ == "valid" else INVALID):
        f = np.fromfile(os.path.join(G, dir_, name + ".zxc"), np.uint8)
        exp = os.path.join(G, dir_, name + ".expected")
        yield name, f, (os.path.getsize(exp) if os.path.exists(exp) else 1 << 20)


@pytest.mark.gpu
def test_mixed_batch(batch, prod):
    """levels 1-7, 4 KiB / 64 KiB / 2 MiB blocks with a scratch for 64 KiB, checksums, seekable frames, empty frames,
    capacity 0 and one byte short, the golden vectors, and per-frame argument verdicts, in one batch"""
    ref = _ref()
    data = zc.silesia_shaped(1 << 20, seed=31)[:300000]
    frames, caps = [], []
    for level in range(1, 8):
        for bs in (4096, 65536, 2 << 20):
            for cks, seek in ((0, 0), (1, 1), (1, 0), (0, 1)):
                n = data.size if level < 6 else 100000
                f = prod.compress(data[:n], level=level, block_size=bs, checksum=cks, seekable=seek)
                frames.append(f)
                caps.append(n if (level + cks) % 3 else n - 1)
    e = prod.compress(np.zeros(0, np.uint8), level=3, checksum=1)
    frames += [e, e, frames[0], frames[1]]
    caps += [0, 100, 0, 1]
    for name, f, cap in _golden("valid"):
        if f[6] & 0x40:
            continue  # dictionary frames: test_dictionaries
        frames.append(f)
        caps.append(cap)
    for name, f, cap in _golden("invalid"):
        frames.append(f)
        caps.append(cap)
    frames += [None, frames[0], frames[0][:27], frames[0][:0]]
    caps += [1000, (1000,), 1000, 1000]
    for cks in (0, 1):
        rs = batch.check(prod, frames, caps, cks, ref=ref, what=("mixed", cks))
        assert MEMORY in rs  # the 2 MiB frames, as the single call with a scratch for 64 KiB


@pytest.mark.gpu
def test_dictionaries(batch, prod):
    ref = _ref()
    data = make_case("text", 150000)
    (d, h), (d2, h2) = list(golden_dicts().values())[:2]
    frames = []
    for dd, hh in ((d, h), (d, None), (d2, h2)):
        for bs, cks, seek in ((4096, 1, 1), (65536, 0, 0)):
            frames.append(prod.compress(data, level=5, block_size=bs, checksum=cks, seekable=seek, dict=dd,
                                        dict_huf=hh))
    frames.append(prod.compress(data, level=3, block_size=65536))  # no dictionary
    caps = [data.size] * len(frames)
    batch.check(prod, frames, caps, 1, d, h, ref=ref)  # own id decodes, the other gives DICT_MISMATCH
    batch.check(prod, frames, caps, 1)  # DICT_REQUIRED
    batch.check(prod, frames, caps, 0, d, None)
    batch.check(prod, frames, caps, 1, d, bytes([0x11]) * 128)  # malformed table


@pytest.mark.gpu
def test_damage_stays_in_its_frame(batch, prod):
    """payload mutations and forged SEK tables among healthy frames: every neighbour keeps its result and bytes"""
    data = zc.silesia_shaped(1 << 20, seed=5)[:90000]
    healthy = prod.compress(data, level=3, block_size=4096, checksum=1, seekable=1)
    frames, caps = [], []
    for k, m in _mutants(healthy, 60, seed=3):
        frames += [healthy, m]
        caps += [data.size, data.size]
    nb = (data.size + 4095) // 4096
    ent = healthy.size - 12 - 4 * nb
    sizes = np.frombuffer(healthy[ent:ent + 4 * nb].tobytes(), "<u4").copy()
    for forge in ((3, 4), (0, 1), (-1, None)):
        s = sizes.copy()
        if forge[1] is None:
            s[-1] += 4
        else:
            s[forge[0]] += 1
            s[forge[1]] -= 1
        f = healthy.copy()
        f[ent:ent + 4 * nb] = np.frombuffer(s.astype("<u4").tobytes(), np.uint8)
        frames += [f, healthy]
        caps += [data.size, data.size]
    rs = batch.check(prod, frames, caps, 1)
    assert all(r == data.size for i, r in enumerate(rs) if frames[i] is healthy)


@pytest.mark.gpu
def test_general_split(batch, prod):
    """stitched frames with short non-final blocks among regular ones; one with more blocks than its table share
    (MEMORY, as the single call gives)"""
    data = zc.silesia_shaped(1 << 20, seed=21)[:400000]
    frames, caps = [], []
    for seed in range(4):
        st, _ = _stitched(prod, data, 65536, 1 + seed, seed)
        frames += [st, prod.compress(data, level=2, block_size=4096)]
        caps += [data.size, data.size]
    st, _ = _stitched(prod, data, 65536, 3, 9)
    many, nb = _stitched(prod, data, 4096, 3, 9)
    assert nb > -(-data.size // 4096) + 2
    frames += [st, st, many]
    caps += [data.size - 1, data.size + 70000, data.size]
    rs = batch.check(prod, frames, caps, 0)
    assert rs[:8] == [data.size] * 8 and rs[9] == data.size and rs[10] == MEMORY, rs


@pytest.mark.gpu
@pytest.mark.parametrize("src_off", [1, 3, 7])
def test_unaligned_sources(batch, prod, src_off):
    data = make_case("text", 70000)
    frames = [prod.compress(data, level=lv, block_size=4096, checksum=1, seekable=lv % 2) for lv in (1, 3, 6)]
    batch.check(prod, frames, [data.size] * 3, 1, bs=4096, src_off=src_off)


@pytest.mark.gpu
def test_table_overflow_in_index_order(batch, prod):
    """a scratch sized for less than the capacities: MEMORY from the first frame that no longer fits, in index order;
    frames that fail the argument checks take no entries"""
    data = make_case("text", 40000)
    f = prod.compress(data, level=3, block_size=4096)
    frames = [f, None, f, f, f, f]
    caps = [data.size, 10 ** 9, data.size, data.size, data.size, data.size]
    J = -(-data.size // 4096) + 2
    total = 2 * data.size + 5 * 4096
    got = batch.run(frames, caps, bs=4096, total=total)  # a table of at least ceil(total / 4096) + 18 entries
    rs = [r for r, _ in got]
    assert rs[1] == NULL_INPUT
    ok = [r for i, r in enumerate(rs) if i != 1]
    fit = ok.index(MEMORY)
    assert (-(-total // 4096) + 18) // J <= fit < 5, rs
    assert ok[:fit] == [data.size] * fit and all(r == MEMORY for r in ok[fit:]), rs


@pytest.mark.gpu
def test_many_small_frames(batch, prod):
    t = batch.t
    rng = np.random.default_rng(4)
    base = zc.silesia_shaped(1 << 20, seed=2)
    protos = []
    for k in range(16):
        n = int(rng.integers(100, 700))
        a = int(rng.integers(0, base.size - n))
        protos.append((base[a:a + n].copy(), prod.compress(base[a:a + n], level=1 + k % 5, block_size=4096,
                                                            checksum=k % 2, seekable=k % 3 == 0)))
    n = 100_000
    pick = rng.integers(0, len(protos), n)
    srcs = [t.from_numpy(p[1]).cuda() for p in protos]
    outs = t.zeros((n, 1024), dtype=t.uint8, device="cuda")
    desc = t.tensor([[srcs[j].data_ptr(), srcs[j].numel(), outs.data_ptr() + 1024 * i, protos[j][0].size]
                     for i, j in enumerate(pick)], dtype=t.int64).cuda()
    size = batch.scratch_size(n, int(sum(protos[j][0].size for j in pick)), 4096)
    scratch = t.empty(size, dtype=t.uint8, device="cuda")
    res = t.zeros(n, dtype=t.int64, device="cuda")
    assert batch.enqueue(desc, n, dopts(1), scratch, res, scratch_size=size) == 0
    r = res.cpu().numpy()
    o = outs.cpu().numpy()
    for j, (raw, _) in enumerate(protos):
        sel = np.nonzero(pick == j)[0]
        assert (r[sel] == raw.size).all(), j
        assert (o[sel, :raw.size] == raw).all(), j


@pytest.mark.gpu
def test_one_gib_frame_next_to_small_ones(batch, prod):
    t = batch.t
    from zxc_b200 import device as zd
    big = t.from_numpy(zc.silesia_shaped(64 << 20, seed=8)).cuda().repeat(16)
    fb = zd.compress(big, level=1, block_size=65536)
    small = t.from_numpy(make_case("text", 30000)).cuda()
    fs = zd.compress(small, level=3, block_size=4096, checksum=True)
    outs, res = zd.decompress_frames([fs.frame, fb.frame, fs.frame], checksum=True)
    assert res.tolist() == [small.numel(), big.numel(), small.numel()]
    assert t.equal(outs[1], big) and t.equal(outs[0], small) and t.equal(outs[2], small)


@pytest.mark.gpu
def test_two_streams_graph_and_launches(batch, prod):
    t = batch.t
    data = make_case("text", 120000)
    f1 = prod.compress(data, level=3, block_size=4096, checksum=1)
    f2 = prod.compress(data[::-1].copy(), level=5, block_size=65536, seekable=1)
    # two batches on two streams with separate scratch
    s1, s2 = t.cuda.Stream(), t.cuda.Stream()
    runs = []
    for f, s in ((f1, s1), (f2, s2)):
        srcs, dsts, desc = batch.upload([f] * 3, [data.size] * 3)
        scr = t.empty(batch.scratch_size(3, 3 * data.size, 65536), dtype=t.uint8, device="cuda")
        res = t.zeros(3, dtype=t.int64, device="cuda")
        runs.append((srcs, dsts, desc, scr, res))
    t.cuda.synchronize()
    for (srcs, dsts, desc, scr, res), s in zip(runs, (s1, s2)):
        assert batch.enqueue(desc, 3, dopts(1), scr, res, stream=s, scratch_size=scr.numel()) == 0
    t.cuda.synchronize()
    for (srcs, dsts, desc, scr, res), want in zip(runs, (data, data[::-1])):
        assert res.tolist() == [data.size] * 3
        for d in dsts:
            assert np.array_equal(d[GUARD:GUARD + data.size].cpu().numpy(), want)
    # graph capture, then replay with rewritten descriptors and frames
    srcs, dsts, desc, scr, res = runs[0]
    s = t.cuda.Stream()
    g = t.cuda.CUDAGraph()
    t.cuda.synchronize()
    with t.cuda.graph(g, stream=s):
        assert batch.enqueue(desc, 3, dopts(0), scr, res, stream=s, scratch_size=scr.numel()) == 0
    for d in dsts:
        d.fill_(0)
    g.replay()
    t.cuda.synchronize()
    assert res.tolist() == [data.size] * 3
    other = batch.upload([f2], [data.size])
    desc[1, 0] = other[0][0].data_ptr()
    desc[1, 1] = f2.size
    desc[2, 1] = 27
    res.fill_(0)
    g.replay()
    t.cuda.synchronize()
    assert res.tolist() == [data.size, data.size, SRC_SMALL]
    assert np.array_equal(dsts[1][GUARD:GUARD + data.size].cpu().numpy(), data[::-1])
    # the fixed launch count: 14 + k * (2 + c), k = 5 block sizes up to 64 KiB
    L = batch.L
    for n in (1, 7, 10_000):
        srcs, dsts, desc = batch.upload([f1], [data.size])
        desc = desc.repeat(n, 1)
        desc[:, 2] = 0
        desc[:, 3] = 0
        scr = t.empty(batch.scratch_size(n, 0, 65536), dtype=t.uint8, device="cuda")
        res = t.zeros(n, dtype=t.int64, device="cuda")
        for cks in (0, 1):
            before = L.zxc_b200_launch_count()
            assert batch.enqueue(desc, n, dopts(cks), scr, res, scratch_size=scr.numel()) == 0
            assert L.zxc_b200_launch_count() - before == 14 + 5 * (2 + cks)
        t.cuda.synchronize()
        assert (res == -2).all().item()  # DST_TOO_SMALL: capacity 0 with a non-empty footer


@pytest.mark.gpu
def test_python_decompress_frames(prod):
    import torch as t
    from zxc_b200 import device as zd
    data = [make_case("text", n) for n in (5000, 70000, 0, 200000)]
    frames = [t.from_numpy(prod.compress(d, level=3, block_size=65536 if i % 2 else 4096, checksum=1)).cuda()
              for i, d in enumerate(data)]
    outs, res = zd.decompress_frames(frames, checksum=True)
    assert res.tolist() == [d.size for d in data]
    for o, d, f in zip(outs, data, frames):
        assert np.array_equal(o.cpu().numpy(), d)
        assert t.equal(zd.decompress_frame(f, checksum=True), o)
    caps = [d.size + 10 for d in data]
    outs, res = zd.decompress_frames(frames, caps)
    assert res.tolist() == [d.size for d in data] and [o.numel() for o in outs] == caps
    out = [t.empty(c, dtype=t.uint8, device="cuda") for c in caps]
    s = t.cuda.Stream()
    outs, res = zd.decompress_frames(frames, out=out, stream=s)
    s.synchronize()
    assert all(a is b for a, b in zip(outs, out)) and res.tolist() == [d.size for d in data]
    with pytest.raises(ValueError):
        zd.decompress_frames([])
    with pytest.raises(ValueError):
        zd.decompress_frames([frames[0].cpu()])
    with pytest.raises(ValueError):
        zd.decompress_frames(frames, caps[:-1])
    with pytest.raises(ValueError):
        zd.decompress_frames(frames, out=out[:-1])
    with pytest.raises(ValueError):
        zd.decompress_frames(frames, block_size=5000)
    with pytest.raises(ValueError):
        zd.decompress_frames([frames[0][:20]])
