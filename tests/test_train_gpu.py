"""Dictionary trainers (zxc_train_dict, zxc_train_dict_huf, zxc_dict_train): the same bytes and the same return codes
as the unmodified reference (oracle/_ref/libzxc_ref.so) for every input.

CPU tests check the argument verdicts, which need no device.  GPU tests compare the product's output with the
reference's over corpus kinds, sample shapes and the sampling boundaries of both trainers, and check golden case 12
without the reference."""
import ctypes as C
import hashlib
import os
import threading

import numpy as np
import pytest

import zxc_corpus as zc
import zxc_ctypes as z
from conftest import has_cuda
from test_oracle import GC_DICT, G

DICT_MAX = 65535
KGRAM = 5


def bind(lib):
    L = lib.lib
    L.zxc_train_dict.restype = C.c_int64
    L.zxc_train_dict.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    L.zxc_train_dict_huf.restype = C.c_int
    L.zxc_train_dict_huf.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    L.zxc_dict_train.restype = C.c_int64
    L.zxc_dict_train.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    return L


class Samples:
    """n sample pointers and sizes over one contiguous buffer; a size of None makes a NULL sample of size 0"""

    def __init__(self, data, sizes):
        self.data = np.ascontiguousarray(data, dtype=np.uint8)
        n = len(sizes)
        self.ptrs = (C.c_void_p * max(n, 1))()
        self.sizes = (C.c_size_t * max(n, 1))()
        base, off = self.data.ctypes.data, 0
        for i, s in enumerate(sizes):
            if s is None:
                self.ptrs[i], self.sizes[i] = None, 0
            else:
                self.ptrs[i], self.sizes[i] = base + off, s
                off += s
        assert off <= self.data.size
        self.n = n

    @classmethod
    def one(cls, data):
        return cls(data, [data.size])


def train_content(L, S, cap):
    out = np.zeros(max(cap, 1), np.uint8)
    r = L.zxc_train_dict(S.ptrs, S.sizes, S.n, out.ctypes.data, cap)
    return r, (out[:r].tobytes() if r > 0 else b"")


def train_table(L, S, d):
    huf = np.zeros(128, np.uint8)
    db = np.frombuffer(d, np.uint8).copy() if d else np.zeros(1, np.uint8)
    r = L.zxc_train_dict_huf(S.ptrs, S.sizes, S.n, db.ctypes.data if d else None, len(d), huf.ctypes.data)
    return r, huf.tobytes()


def train_zxd(L, S, cap=DICT_MAX + 16 + 128):
    out = np.zeros(cap, np.uint8)
    r = L.zxc_dict_train(S.ptrs, S.sizes, S.n, out.ctypes.data, cap)
    return r, (out[:r].tobytes() if r > 0 else b"")


@pytest.fixture(scope="module")
def P(prod):
    return bind(prod)


@pytest.fixture(scope="module")
def R(ref):
    return bind(ref)


# ---- argument verdicts (no device) ----------------------------------------------------------------------------
def _verdict_cases():
    d5 = np.arange(64, dtype=np.uint8)
    yield "null arrays", lambda L: L.zxc_train_dict(None, None, 1, d5.ctypes.data, 16)
    s = Samples.one(np.arange(100, dtype=np.uint8))
    yield "null sizes", lambda L: L.zxc_train_dict(s.ptrs, None, 1, d5.ctypes.data, 16)
    yield "n_samples 0", lambda L: L.zxc_train_dict(s.ptrs, s.sizes, 0, d5.ctypes.data, 16)
    yield "null output", lambda L: L.zxc_train_dict(s.ptrs, s.sizes, 1, None, 16)
    yield "capacity 0", lambda L: L.zxc_train_dict(s.ptrs, s.sizes, 1, d5.ctypes.data, 0)
    yield "capacity 65536", lambda L: L.zxc_train_dict(s.ptrs, s.sizes, 1, d5.ctypes.data, 65536)
    for total, parts in ((0, [0]), (0, [0, 0, 0]), (1, [1]), (3, [1, 0, 2]), (4, [1, 1, 1, 1]), (4, [2, None, 2])):
        t = Samples(np.arange(8, dtype=np.uint8), parts)
        yield f"corpus {total} bytes in {parts}", (lambda t: lambda L: L.zxc_train_dict(t.ptrs, t.sizes, t.n, d5.ctypes.data, 64))(t)
    huf = np.zeros(128, np.uint8)
    big = np.zeros(65536, np.uint8)
    yield "table: dict_size 0", lambda L: L.zxc_train_dict_huf(s.ptrs, s.sizes, 1, d5.ctypes.data, 0, huf.ctypes.data)
    yield "table: NULL dict", lambda L: L.zxc_train_dict_huf(s.ptrs, s.sizes, 1, None, 10, huf.ctypes.data)
    yield "table: NULL output", lambda L: L.zxc_train_dict_huf(s.ptrs, s.sizes, 1, d5.ctypes.data, 10, None)
    yield "table: n_samples 0", lambda L: L.zxc_train_dict_huf(s.ptrs, s.sizes, 0, d5.ctypes.data, 10, huf.ctypes.data)
    yield "table: dict_size 65536", lambda L: L.zxc_train_dict_huf(s.ptrs, s.sizes, 1, big.ctypes.data, 65536, huf.ctypes.data)
    zxd = np.zeros(70000, np.uint8)
    yield "zxd: NULL arrays", lambda L: L.zxc_dict_train(None, None, 1, zxd.ctypes.data, zxd.size)
    yield "zxd: capacity 0", lambda L: L.zxc_dict_train(s.ptrs, s.sizes, 1, zxd.ctypes.data, 0)
    t4 = Samples(np.arange(8, dtype=np.uint8), [2, 2])
    yield "zxd: 4-byte corpus", lambda L: L.zxc_dict_train(t4.ptrs, t4.sizes, 2, zxd.ctypes.data, zxd.size)


VERDICTS = list(_verdict_cases())


@pytest.mark.parametrize("name", [n for n, _ in VERDICTS])
def test_argument_verdicts_match_reference(P, R, name):
    call = dict(VERDICTS)[name]
    want = call(R)
    assert want < 0, (name, want)
    assert call(P) == want, (name, z.ERR.get(want))


def test_valid_call_without_device_reports_no_device(P):
    if has_cuda():
        pytest.skip("a CUDA device is present")
    s = Samples.one(zc.gen_text(20000))
    assert train_content(P, s, 4096)[0] == -100
    assert train_table(P, s, b"some dictionary bytes")[0] == -100
    assert train_zxd(P, s)[0] == -100


# ---- a Python model of the content trainer, for the tie order --------------------------------------------------
def _hashes(a):
    a = a.astype(np.uint32)
    v = a[:-4] | (a[1:-3] << 8) | (a[2:-2] << 16) | (a[3:-1] << 24)
    return (((v ^ a[4:]).astype(np.uint64) * 0x2D35182D) & 0xFFFFFFFF) >> 16


def _heap_desc(segs):
    a = list(segs)

    def sift(root, n):
        while True:
            c = 2 * root + 1
            if c >= n:
                return
            if c + 1 < n and a[c + 1][2] < a[c][2]:
                c += 1
            if a[root][2] <= a[c][2]:
                return
            a[root], a[c] = a[c], a[root]
            root = c

    n = len(a)
    for i in range(n // 2 - 1, -1, -1):
        sift(i, n)
    for end in range(n - 1, 0, -1):
        a[0], a[end] = a[end], a[0]
        sift(0, end)
    return a


def model_train(data, cap, order):
    """zxc_train_dict restated in Python (small corpora), with the segment order given by `order`"""
    C_ = data.size
    H = _hashes(data).astype(np.int64)
    freq = np.zeros(65536, np.int64)
    fs = max(1, (C_ - 4) // (1 << 19))
    np.add.at(freq, H[0:C_ - 4:fs], 1)
    freq = np.minimum(freq, 65535)
    seg_alloc = min(C_ // 5, 65536)
    stride = max(5, C_ // seg_alloc)
    segs, i = [], 0
    while i + 5 <= C_ and len(segs) < seg_alloc:
        f = int(freq[H[i]])
        if f >= 2:
            cov, end = f, i + 5
            while end + 5 <= C_ and end - i < 4096:
                nf = int(freq[H[end]])
                if nf < 2:
                    break
                cov += nf
                end += 5
            segs.append((i, end - i, cov))
        i += stride
    picks, total = [], 0
    for off, ln, sc in order(segs):
        if total >= cap:
            break
        ks = H[off:off + ln - 4:5]
        if int(freq[ks].sum()) * 2 < sc:
            continue
        cp = min(ln, cap - total)
        freq[ks] = 0
        picks.append((off, cp))
        total += cp
    out = b"".join(data[o:o + c].tobytes() for o, c in reversed(picks))
    return out or data[C_ - min(C_, cap):].tobytes()


def tie_corpus():
    """many identical records with a few varying bytes: many segments share one score"""
    rng = np.random.default_rng(11)
    recs = []
    for k in range(400):
        recs.append(b'{"id":%05d,"kind":"event","state":"ok","tag":"%s"}\n' % (k, bytes(rng.choice(list(b"abcd"), 3))))
    return np.frombuffer(b"".join(recs), np.uint8).copy()


def test_tie_order_is_the_heap_order(R):
    """the reference's dictionary is the heap order's; a stable sort of the same segments gives another one"""
    data = tie_corpus()
    want = train_content(R, Samples.one(data), 1024)[1]
    assert model_train(data, 1024, _heap_desc) == want
    stable = model_train(data, 1024, lambda s: sorted(s, key=lambda t: -t[2]))
    assert stable != want


# ---- GPU: byte-for-byte against the reference ------------------------------------------------------------------
def _records(n, size=512, seed=7):
    return zc.records(n, size, seed)


def corpus(kind, n):
    if kind == "records":
        return _records((n + 511) // 512)[:n]
    if kind == "text":
        return zc.gen_text(n)
    if kind == "numeric":
        return zc.gen_numeric(n)
    if kind == "silesia":
        return zc.silesia_shaped(n, seed=5)
    if kind == "random":
        return zc.gen_random(n)
    if kind == "zeros":
        return np.zeros(n, np.uint8)
    if kind == "alphabet2":
        return np.random.default_rng(3).choice(np.array([97, 98], np.uint8), n)
    if kind == "ties":
        t = tie_corpus()
        return np.tile(t, n // t.size + 1)[:n].copy()
    raise KeyError(kind)


def shape(kind, n, seed=1):
    """sample sizes summing to n"""
    rng = np.random.default_rng(seed)
    if kind == "one":
        return [n]
    if kind == "small":  # 16-200 byte samples
        out, left = [], n
        while left > 0:
            s = min(left, int(rng.integers(16, 201)))
            out.append(s)
            left -= s
        return out
    if kind == "gaps":  # empty and NULL samples in between
        out, left = [], n
        while left > 0:
            s = min(left, int(rng.integers(1, 3000)))
            out += [s, 0, None] if rng.integers(0, 2) else [s]
            left -= s
        return out
    if kind == "tiny":  # 1-4 bytes: k-grams span sample boundaries
        out, left = [], n
        while left > 0:
            s = min(left, int(rng.integers(1, 5)))
            out.append(s)
            left -= s
        return out
    raise KeyError(kind)


def check_all(P, R, data, sizes, cap, table=True):
    S = Samples(data, sizes)
    rp, dp = train_content(P, S, cap)
    rr, dr = train_content(R, S, cap)
    assert (rp, dp) == (rr, dr), (rp, rr, len(dp), len(dr))
    if table and rr > 0:
        hp, hr = train_table(P, S, dr), train_table(R, S, dr)
        assert hp == hr, (hp[0], hr[0], hp[1].hex(), hr[1].hex())
    return dr


KINDS = ["records", "text", "numeric", "silesia", "random", "zeros", "alphabet2", "ties"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shp", ["one", "gaps", "tiny"])
def test_trainers_match_reference(P, R, kind, shp):
    n = 60000 if shp == "tiny" else 300000
    data = corpus(kind, n)
    check_all(P, R, data, shape(shp, n), 16384)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["records", "text", "random"])
def test_many_small_samples(P, R, kind):
    """100 k samples of 16-200 bytes (over 8 MiB: the table trainer keeps every second slice)"""
    sizes = shape("small", 10_800_000, seed=4)[:100_000]
    data = corpus(kind, sum(sizes))
    check_all(P, R, data, sizes, 4096)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [(1 << 19) + 3, (1 << 19) + 4, (1 << 19) + 5, (1 << 20) + 3, (1 << 20) + 4, (1 << 20) + 5,
                               327675, 327679, 327680, 327685, 327690])
def test_sampling_boundaries(P, R, n):
    """freq_stride 1 -> 2 (kgram_limit 2^20) and the seg_alloc cap (corpus_size / 5 = 65 536)"""
    check_all(P, R, corpus("silesia", n), [n], 16384, table=False)


@pytest.mark.gpu
@pytest.mark.parametrize("total", [(8 << 20) - 1, 8 << 20, (8 << 20) + 1, 16 << 20, (16 << 20) + 1])
def test_slice_stride_boundaries(P, R, total):
    """the table trainer's slice stride 1 -> 2 -> 3 around 8 MiB and 16 MiB of samples"""
    data = corpus("records", total)
    sizes = [4096] * (total // 4096) + ([total % 4096] if total % 4096 else [])
    S = Samples(data, sizes)
    d = train_content(R, Samples.one(data[:200000]), 2048)[1]
    assert train_table(P, S, d) == train_table(R, S, d)


@pytest.mark.gpu
@pytest.mark.parametrize("cap", [1, 5, 100, 4096, 16384, 65535])
@pytest.mark.parametrize("kind", ["records", "zeros", "text"])
def test_capacities(P, R, cap, kind):
    """capacities from 1 byte to the maximum, a final pick truncated by the capacity, 4 096-byte segments (zeros)"""
    check_all(P, R, corpus(kind, 400000), [400000], cap, table=cap >= 100)


@pytest.mark.gpu
def test_ties_on_the_gpu(P, R):
    data = tie_corpus()
    for cap in (256, 1024, 4096):
        check_all(P, R, data, [data.size], cap)


@pytest.mark.gpu
def test_corpus_over_4_gib(P, R):
    """offsets are 32-bit in the reference: picks past 4 GiB read the corpus at the wrapped offset"""
    n = (4 << 30) + (3 << 20)
    avail = 0
    for line in open("/proc/meminfo"):
        if line.startswith("MemAvailable:"):
            avail = int(line.split()[1]) << 10
    if avail < 3 * n:
        pytest.skip("needs about 13 GiB of free host memory")
    data = np.empty(n, np.uint8)
    data[: 1 << 30] = zc.gen_random(1 << 30, seed=9)
    for k in range(1, 4):
        data[k << 30:(k + 1) << 30] = data[: 1 << 30]
    data[4 << 30:] = corpus("records", n - (4 << 30))  # the only frequent k-grams lie past 4 GiB
    sizes = [1 << 30] * 4 + [n - (4 << 30)]
    S = Samples(data, sizes)
    rp, dp = train_content(P, S, 16384)
    rr, dr = train_content(R, S, 16384)
    assert rr > 0 and (rp, dp) == (rr, dr)


@pytest.mark.gpu
def test_golden_12_table_without_reference(P, prod):
    """golden case 12: the product trains the table on the case's payload and GC_DICT, and reproduces the archive"""
    sha = {l.split()[1]: l.split()[0] for l in open(os.path.join(G, "format", "golden.sha256"))}

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
    rc, huf = train_table(P, Samples.one(payload), GC_DICT)
    assert rc == 0
    fr = prod.compress(payload, level=6, dict=GC_DICT, dict_huf=huf)
    assert hashlib.sha256(fr.tobytes()).hexdigest() == sha["12_glo_huffman_dict.zxc"]
    golden = np.fromfile(os.path.join(G, "format", "12_glo_huffman_dict.zxc"), np.uint8)
    r, out = prod.decompress(golden, payload.size, dict=GC_DICT, dict_huf=huf)
    assert r == payload.size and np.array_equal(out, payload)


@pytest.mark.gpu
def test_zxd_round_trip(P, R, prod, ref):
    """the product's .zxd equals the reference's; frames made with each are identical at levels 5 and 6"""
    data = _records(2048)
    sizes = [512] * 2048
    S = Samples(data, sizes)
    rp, zp = train_zxd(P, S)
    rr, zr = train_zxd(R, S)
    assert rr > 0 and (rp, zp) == (rr, zr)
    rc, content, huf, _ = prod.dict_load(zp)
    assert rc == 0
    body = _records(256, seed=21)
    for level in (5, 6):
        a = prod.compress(body, level=level, block_size=4096, dict=content, dict_huf=huf)
        b = ref.compress(body, level=level, block_size=4096, dict=content, dict_huf=huf)
        assert not isinstance(a, int) and a.size == b.size and np.array_equal(a, b), level
        r, out = prod.decompress(a, body.size, dict=content, dict_huf=huf)
        assert r == body.size and np.array_equal(out, body)


@pytest.mark.gpu
def test_concurrent_training(P, R):
    """eight threads train at once on four corpora: .zxd images on four, content alone on the other four"""
    jobs = [(corpus(k, 250000), c) for k, c in (("records", 16384), ("text", 4096), ("silesia", 65535), ("numeric", 100))]
    want = [train_zxd(R, Samples.one(d)) for d, _ in jobs] + [train_content(R, Samples.one(d), c) for d, c in jobs]
    got = [None] * len(want)

    def run(i):
        d, c = jobs[i % 4]
        got[i] = train_zxd(P, Samples.one(d)) if i < 4 else train_content(P, Samples.one(d), c)

    th = [threading.Thread(target=run, args=(i,)) for i in range(len(want))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert got == want


@pytest.mark.gpu
def test_phase_times_reported(P):
    P.zxc_b200_train_phase_times.restype = C.c_int
    P.zxc_b200_train_phase_times.argtypes = [C.c_void_p, C.c_int]
    assert train_zxd(P, Samples.one(corpus("records", 200000)))[0] > 0
    ms = np.zeros(8)
    assert P.zxc_b200_train_phase_times(ms.ctypes.data, 8) == 8
    assert ms[1] > 0 and ms[6] > 0
