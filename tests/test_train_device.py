"""Dictionary trainers on samples in HBM (zxc_b200_train_dict_device, zxc_b200_train_dict_huf_device,
zxc_b200_dict_train_device and the Python helpers of zxc_b200.device): the same return values and bytes as this
library's host trainers on host copies of the samples, and as the reference (oracle/_ref/libzxc_ref.so) where it is
built.  Also: samples in separate allocations at every misalignment, repeated and NULL samples, stream order, launch
counts, two threads, a corpus over 4 GiB, and the Python forms."""
import ctypes as C
import hashlib
import os
import threading

import numpy as np
import pytest

import test_train_gpu as T
import zxc_corpus as zc
from test_oracle import GC_DICT, G
from test_train_device_host import Twins

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def H(prod):
    return T.bind(prod)


@pytest.fixture(scope="module")
def D(prod):
    return Twins(prod)


@pytest.fixture(scope="module")
def Ropt(libs):
    return T.bind(libs[2]) if libs[2] is not None else None


class DevSamples:
    """the samples of T.Samples(data, sizes) copied into one CUDA tensor, with the same layout; ptrs holds device
    addresses (None: a NULL sample of size 0)"""

    def __init__(self, data, sizes):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        self.t = torch.from_numpy(data).cuda() if data.size else torch.zeros(1, dtype=torch.uint8, device="cuda")
        host = T.Samples(data, sizes)
        self.n = host.n
        self.ptrs = (C.c_void_p * max(self.n, 1))()
        self.sizes = host.sizes
        hb, db = data.ctypes.data, self.t.data_ptr()
        for i in range(self.n):
            self.ptrs[i] = None if host.ptrs[i] is None else db + (host.ptrs[i] - hb)
        self.host = host


def outputs(L, S, cap, table=True, zxd=False):
    r, d = T.train_content(L, S, cap)
    out = [(r, d)]
    if table and r > 0:
        out.append(T.train_table(L, S, d))
    if zxd:
        out.append(T.train_zxd(L, S))
    return out


def check(H, D, Ropt, data, sizes, cap, table=True, zxd=False):
    """the twins on device copies against the host trainers (and the reference) on the host samples"""
    DS = DevSamples(data, sizes)
    want = outputs(H, DS.host, cap, table, zxd)
    assert outputs(D, DS, cap, table, zxd) == want
    if Ropt is not None:
        assert outputs(Ropt, DS.host, cap, table, zxd) == want
    return want


@pytest.mark.parametrize("kind", T.KINDS)
@pytest.mark.parametrize("shp", ["one", "gaps", "tiny"])
def test_twins_match_host_trainers(H, D, Ropt, kind, shp):
    n = 60000 if shp == "tiny" else 300000
    check(H, D, Ropt, T.corpus(kind, n), T.shape(shp, n), 16384, zxd=shp == "gaps")


@pytest.mark.parametrize("kind", ["records", "text", "random"])
def test_many_small_samples(H, D, Ropt, kind):
    sizes = T.shape("small", 10_800_000, seed=4)[:100_000]
    check(H, D, Ropt, T.corpus(kind, sum(sizes)), sizes, 4096)


@pytest.mark.parametrize("n", [(1 << 19) + 3, (1 << 19) + 4, (1 << 19) + 5, (1 << 20) + 3, (1 << 20) + 4, (1 << 20) + 5,
                               327675, 327679, 327680, 327685, 327690])
def test_sampling_boundaries(H, D, Ropt, n):
    check(H, D, Ropt, T.corpus("silesia", n), [n], 16384, table=False)


@pytest.mark.parametrize("total", [(8 << 20) - 1, 8 << 20, (8 << 20) + 1, 16 << 20, (16 << 20) + 1])
def test_slice_stride_boundaries(H, D, Ropt, total):
    data = T.corpus("records", total)
    sizes = [4096] * (total // 4096) + ([total % 4096] if total % 4096 else [])
    DS = DevSamples(data, sizes)
    d = T.train_content(H, T.Samples.one(data[:200000]), 2048)[1]
    want = T.train_table(H, DS.host, d)
    assert T.train_table(D, DS, d) == want
    if Ropt is not None:
        assert T.train_table(Ropt, DS.host, d) == want


@pytest.mark.parametrize("cap", [1, 5, 100, 4096, 16384, 65535])
@pytest.mark.parametrize("kind", ["records", "zeros", "text"])
def test_capacities(H, D, Ropt, cap, kind):
    check(H, D, Ropt, T.corpus(kind, 400000), [400000], cap, table=cap >= 100)


def test_ties(H, D, Ropt):
    data = T.tie_corpus()
    for cap in (256, 1024, 4096):
        check(H, D, Ropt, data, [data.size], cap)


def test_golden_12_table_from_device_samples(D, prod):
    """golden case 12's table, trained on the case's payload in HBM, reproduces the archive"""
    sha = {l.split()[1]: l.split()[0] for l in open(os.path.join(G, "format", "golden.sha256"))}
    s, buf = 0x5EEDCAFE, b""

    def nxt():
        nonlocal s
        s = (s * 1103515245 + 12345) & 0xFFFFFFFF
        return s

    while len(buf) + 160 < 4096:
        uid, sess, page = nxt() % 100000, nxt(), nxt() % 64
        buf += (b"GET /api/v1/users/%d/profile?session=%08x&page=%d HTTP/1.1\r\nHost: api.example.com\r\n"
                b"Accept: application/json\r\nUser-Agent: zxc-client\r\n\r\n" % (uid, sess, page))
    payload = np.frombuffer(buf, np.uint8).copy()
    rc, huf = T.train_table(D, DevSamples(payload, [payload.size]), GC_DICT)
    assert rc == 0
    fr = prod.compress(payload, level=6, dict=GC_DICT, dict_huf=huf)
    assert hashlib.sha256(fr.tobytes()).hexdigest() == sha["12_glo_huffman_dict.zxc"]


def _separate(data, sizes, offsets):
    """every sample in its own allocation, at its offset: (tensors kept alive, device pointers)"""
    keep, ptrs, o = [], [], 0
    for s, off in zip(sizes, offsets):
        t = torch.empty(off + s, dtype=torch.uint8, device="cuda")
        t[off:] = torch.from_numpy(data[o:o + s]).cuda()
        keep.append(t)
        ptrs.append(t.data_ptr() + off)
        o += s
    return keep, ptrs


def _arrays(ptrs, sizes):
    P = (C.c_void_p * len(ptrs))(*ptrs)
    S = (C.c_size_t * len(sizes))(*sizes)
    return P, S


class _Raw:
    def __init__(self, ptrs, sizes, host=None):
        self.ptrs, self.sizes = _arrays(ptrs, sizes)
        self.n = len(ptrs)
        self.host = host


def test_separate_allocations_every_misalignment(H, D):
    """offsets 1-15 and 0 in separate allocations, in address order, in reverse address order"""
    rng = np.random.default_rng(5)
    sizes = [int(x) for x in rng.integers(1, 9000, 600)]
    data = T.corpus("records", sum(sizes))
    want = outputs(H, T.Samples(data, sizes), 8192, zxd=True)
    offs = [i % 16 for i in range(len(sizes))]
    keep, ptrs = _separate(data, sizes, offs)
    assert outputs(D, _Raw(ptrs, sizes), 8192, zxd=True) == want
    # reverse address order: the last sample allocated first
    rev_s, rev_o = sizes[::-1], [1 + i % 15 for i in range(len(sizes))]
    starts = np.concatenate(([0], np.cumsum(sizes)))
    rdata = np.concatenate([data[starts[i]:starts[i + 1]] for i in range(len(sizes) - 1, -1, -1)])
    keep2, rptrs = _separate(rdata, rev_s, rev_o)
    assert outputs(D, _Raw(rptrs[::-1], rev_s[::-1]), 8192, zxd=True) == want
    del keep, keep2


def test_repeated_and_overlapping_samples(H, D):
    data = T.corpus("text", 200000)
    t = torch.from_numpy(data).cuda()
    base, hb = t.data_ptr(), data.ctypes.data
    spans = [(0, 50000), (0, 50000), (17, 40000), (3, 100001), (17, 40000), (150000, 50000), (149999, 3)]
    want = outputs(H, _Raw([hb + o for o, _ in spans], [n for _, n in spans]), 4096, zxd=True)
    assert outputs(D, _Raw([base + o for o, _ in spans], [n for _, n in spans]), 4096, zxd=True) == want


@pytest.mark.parametrize("nullsize", [0, 1, 4096, 70000])
def test_null_samples(H, D, nullsize):
    """NULL samples read as zeros in the content trainer and are skipped by the table trainer, as on the host"""
    data = T.corpus("records", 120000)
    t = torch.from_numpy(data).cuda()
    sizes = [30000, nullsize, 30000, nullsize, 60000]
    hp, dp, o = [], [], 0
    for i, s in enumerate(sizes):
        if i in (1, 3):
            hp.append(None)
            dp.append(None)
        else:
            hp.append(data.ctypes.data + o)
            dp.append(t.data_ptr() + o)
            o += s
    want = outputs(H, _Raw(hp, sizes), 4096, zxd=True)
    assert outputs(D, _Raw(dp, sizes), 4096, zxd=True) == want
    only = outputs(H, _Raw([None], [max(nullsize, 5)]), 64, zxd=True)
    assert outputs(D, _Raw([None], [max(nullsize, 5)]), 64, zxd=True) == only


def test_stream_order(prod, H):
    """samples written behind a long kernel on a side stream are trained on that stream"""
    data = T.corpus("silesia", 400000)
    want = outputs(H, T.Samples.one(data), 16384, zxd=True)
    src = torch.from_numpy(data).cuda()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    got = []
    for k in range(3):
        with torch.cuda.stream(side):
            t = torch.zeros_like(src)
            torch.cuda._sleep(50_000_000)
            t.copy_(src)
        tw = Twins(prod, stream=side.cuda_stream)
        S = _Raw([t.data_ptr()], [t.numel()])
        fn = [lambda: T.train_content(tw, S, 16384), lambda: T.train_table(tw, S, want[0][1]), lambda: T.train_zxd(tw, S)][k]
        got.append(fn())
    assert got == want


@pytest.mark.parametrize("n", [1000, 100_000])
def test_launch_counts(prod, H, D, n):
    """one more launch than the host trainer per trainer that gathers (the gather), whatever the number of samples"""
    prod.lib.zxc_b200_launch_count.restype = C.c_uint64
    lc = prod.lib.zxc_b200_launch_count
    data = T.corpus("records", 100 * 100_000)
    DS = DevSamples(data[: 100 * n], [100] * n)
    for fn, extra in ((lambda L, S: T.train_content(L, S, 16384), 1),
                      (lambda L, S: T.train_table(L, S, bytes(data[:4096])), 1),
                      (lambda L, S: T.train_zxd(L, S), 2)):
        a = lc()
        h = fn(H, DS.host)
        b = lc()
        d = fn(D, DS)
        c = lc()
        assert d == h
        assert c - b == (b - a) + extra, (b - a, c - b)


def test_two_threads(prod, H):
    jobs = [(T.corpus(k, 300000), s, c) for k, s, c in (("records", "gaps", 16384), ("text", "tiny", 4096),
                                                         ("silesia", "one", 65535), ("numeric", "gaps", 100))]
    dev = [DevSamples(d, T.shape(s, d.size)) for d, s, _ in jobs]
    want = [outputs(H, DS.host, c, zxd=True) for DS, (_, _, c) in zip(dev, jobs)]
    streams = [torch.cuda.Stream() for _ in range(2)]
    got = [None] * 8

    def run(k):
        tw = Twins(prod, stream=streams[k].cuda_stream)
        for i in range(k, 8, 2):
            got[i] = outputs(tw, dev[i % 4], jobs[i % 4][2], zxd=True)

    th = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert got == want + want


def test_corpus_over_4_gib(H, D, Ropt):
    """32-bit segment offsets wrap past 4 GiB on the device path exactly as on the host path"""
    n = (4 << 30) + (3 << 20)
    avail = 0
    for line in open("/proc/meminfo"):
        if line.startswith("MemAvailable:"):
            avail = int(line.split()[1]) << 10
    free, _ = torch.cuda.mem_get_info()
    if avail < 2 * n or free < 3 * n:
        pytest.skip("needs about 9 GiB of free host memory and 13 GiB of free device memory")
    data = np.empty(n, np.uint8)
    data[: 1 << 30] = zc.gen_random(1 << 30, seed=9)
    for k in range(1, 4):
        data[k << 30:(k + 1) << 30] = data[: 1 << 30]
    data[4 << 30:] = T.corpus("records", n - (4 << 30))
    sizes = [1 << 30] * 4 + [n - (4 << 30)]
    S = T.Samples(data, sizes)
    want = T.train_content(H, S, 16384)
    assert want[0] > 0
    t = torch.from_numpy(data).cuda()
    base = t.data_ptr()
    DS = _Raw([base + (p - data.ctypes.data) for p in S.ptrs], sizes)
    assert T.train_content(D, DS, 16384) == want
    del t


def test_python_forms(H, prod):
    import zxc_b200.device as zd
    rng = np.random.default_rng(8)
    sizes = [int(x) for x in rng.integers(50, 6000, 500)]
    data = T.corpus("records", sum(sizes))
    HS = T.Samples(data, sizes)
    want_d = T.train_content(H, HS, 65535)[1]
    want_h = T.train_table(H, HS, want_d)[1]
    want_z = T.train_zxd(H, HS)[1]
    buf = torch.from_numpy(data).cuda()
    ends = np.cumsum(sizes)
    views = [buf[e - s:e] for s, e in zip(sizes, ends)]
    for form in ((buf, sizes), (buf, torch.tensor(sizes)), (buf, np.array(sizes)), (views, None)):
        assert zd.train_dict(form[0], form[1]) == want_d
        assert zd.train_dict_huf(form[0], want_d, form[1]) == want_h
        assert zd.dict_train(form[0], form[1]) == want_z
    assert zd.train_dict(views, capacity=1000) == T.train_content(H, HS, 1000)[1]
    # one tensor without sizes is one sample
    assert zd.train_dict(buf) == T.train_content(H, T.Samples.one(data), 65535)[1]
    with pytest.raises(zd.ZxcError) as e:
        zd.train_dict(buf, [2, 2])
    assert e.value.code == T.train_content(H, T.Samples(data, [2, 2]), 65535)[0]
    with pytest.raises(zd.ZxcError):
        zd.train_dict(views, capacity=65536)
    with pytest.raises(ValueError):
        zd.train_dict(buf, [data.size + 1])
    # DeviceDict.train, then the block API: the bytes of the host-trained dictionary
    dd = zd.DeviceDict.train(views)
    host_dd = zd.DeviceDict(want_d, want_h)
    assert (dd.id, dd.dict, dd.dict_huf) == (host_dd.id, want_d, want_h)
    plain = zd.DeviceDict.train(buf, sizes, table=False, capacity=4096)
    assert plain.dict == T.train_content(H, HS, 4096)[1] and plain.dict_huf is None
    recs = [torch.from_numpy(zc.records(64, 4096, seed=21)[i * 4096:(i + 1) * 4096].copy()).cuda() for i in range(64)]
    outs, res = zd.compress_blocks(recs, level=5, dict=dd)
    outs_h, res_h = zd.compress_blocks(recs, level=5, dict=want_d)
    assert torch.equal(res, res_h) and bool((res > 0).all())
    for o, oh, r in zip(outs, outs_h, res.cpu().tolist()):
        assert torch.equal(o[:r], oh[:r])
