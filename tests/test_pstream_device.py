"""Push streaming in HBM: every call of zxc_b200_cstream_device_* / zxc_b200_dstream_device_* against the reference's
zxc_cstream_* / zxc_dstream_* on the same schedule.  The device driver below is tests/zxc_pstream_driver.py's loop with
each chunk in its own device allocation (at an odd offset, ending at the allocation's end) and each out buffer between
guard bytes; after every call the guards and the chunk are checked unchanged."""
import ctypes as C
import random
import threading

import numpy as np
import pytest

import zxc_ctypes as z
import zxc_pstream_driver as pd
import test_pstream_gpu as tg

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu
KB = 1024
_CUDART = []


def cudart():
    """the CUDA runtime torch loaded, for chunks in cudaMalloc allocations of their exact size"""
    if not _CUDART:
        L = C.CDLL("libcudart.so.12")
        L.cudaMalloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t]
        L.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
        L.cudaFree.argtypes = [C.c_void_p]
        _CUDART.append(L)
    return _CUDART[0]
GUARD = 64
vp = C.c_void_p


def bind_device(P):
    """Sets the device-stream prototypes on the product's CDLL; returns it."""
    P.zxc_b200_launch_count.restype = C.c_uint64
    for k in ("c", "d"):
        getattr(P, f"zxc_b200_{k}stream_device_create").restype = vp
        getattr(P, f"zxc_b200_{k}stream_device_create").argtypes = [vp]
        getattr(P, f"zxc_b200_{k}stream_device_free").argtypes = [vp]
        for h in ("in_size", "out_size"):
            getattr(P, f"zxc_b200_{k}stream_device_{h}").restype = C.c_size_t
            getattr(P, f"zxc_b200_{k}stream_device_{h}").argtypes = [vp]
    P.zxc_b200_cstream_device_compress.restype = C.c_int64
    P.zxc_b200_cstream_device_compress.argtypes = [vp, C.POINTER(pd.OutBuf), C.POINTER(pd.InBuf), vp]
    P.zxc_b200_cstream_device_end.restype = C.c_int64
    P.zxc_b200_cstream_device_end.argtypes = [vp, C.POINTER(pd.OutBuf), vp]
    P.zxc_b200_dstream_device_decompress.restype = C.c_int64
    P.zxc_b200_dstream_device_decompress.argtypes = [vp, C.POINTER(pd.OutBuf), C.POINTER(pd.InBuf), vp]
    P.zxc_b200_dstream_device_finished.restype = C.c_int
    P.zxc_b200_dstream_device_finished.argtypes = [vp]
    return P


@pytest.fixture(scope="module")
def libs2(prod, ref):
    P = pd.bind(prod.lib)
    if P.zxc_b200_device_count() <= 0 or not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return bind_device(P), pd.bind(ref.lib)


class DevStream:
    """One device stream with the interface of zxc_pstream_driver.Stream."""

    def __init__(self, P, kind, opts, stream=None, offset=1):
        self.P, self.kind, self.offset = P, kind, offset
        self.h = getattr(P, f"zxc_b200_{kind}stream_device_create")(C.byref(opts) if opts is not None else None)
        self.stream = stream or torch.cuda.current_stream()
        self.chunk = None

    def close(self):
        self.free_chunk()
        if self.h:
            getattr(self.P, f"zxc_b200_{self.kind}stream_device_free")(self.h)
            self.h = None

    def hints(self):
        return (getattr(self.P, f"zxc_b200_{self.kind}stream_device_in_size")(self.h),
                getattr(self.P, f"zxc_b200_{self.kind}stream_device_out_size")(self.h))

    def finished(self):
        return self.P.zxc_b200_dstream_device_finished(self.h) if self.kind == "d" else 0

    def put(self, chunk):
        """the chunk in its own cudaMalloc allocation of exactly offset + len bytes, `offset` bytes in, so that it ends
        at the allocation's end (memcheck flags any read past it); an InBuf on it"""
        self.free_chunk()
        n = len(chunk)
        p = C.c_void_p()
        assert cudart().cudaMalloc(C.byref(p), n + self.offset) == 0
        host = b"\x5a" * self.offset + bytes(chunk)
        assert cudart().cudaMemcpy(p, host, n + self.offset, 1) == 0  # cudaMemcpyHostToDevice
        self.chunk = (p, bytes(chunk))
        return pd.InBuf(p.value + self.offset if n else None, n, 0)

    def free_chunk(self):
        if self.chunk is not None:
            assert cudart().cudaFree(self.chunk[0]) == 0
            self.chunk = None

    def chunk_bytes(self):
        p, want = self.chunk
        h = C.create_string_buffer(len(want) + self.offset)
        assert cudart().cudaMemcpy(h, p, len(want) + self.offset, 2) == 0  # cudaMemcpyDeviceToHost
        return h.raw[self.offset:], want

    def call(self, inbuf, cap, fin=False):
        out = torch.full((cap + 2 * GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
        ob = pd.OutBuf(out.data_ptr() + GUARD, cap, 0)
        st = self.stream.cuda_stream
        if self.kind == "c":
            r = self.P.zxc_b200_cstream_device_end(self.h, C.byref(ob), st) if fin else \
                self.P.zxc_b200_cstream_device_compress(self.h, C.byref(ob), C.byref(inbuf), st)
        else:
            r = self.P.zxc_b200_dstream_device_decompress(self.h, C.byref(ob), C.byref(inbuf), st)
        host = out.cpu().numpy()  # no synchronisation needed: the call has completed its work
        assert (host[:GUARD] == 0xA5).all() and (host[GUARD + cap:] == 0xA5).all(), "write outside out"
        if self.chunk is not None and not fin:
            got, want = self.chunk_bytes()
            assert got == want, "in was written"
        return r, ob.pos, host[GUARD:GUARD + ob.pos].tobytes()


def drive_dev(P, make, schedule, end_cap=None, offset=1, stream=None, max_calls=1 << 20):
    """zxc_pstream_driver.drive for the device streams"""
    kind, opts = make
    s = DevStream(P, kind, opts, stream, offset)
    if not s.h:
        return None
    t = []
    big = sum(len(c) for c, _ in schedule) * 8 + (1 << 20)
    cap_of = lambda cap: s.hints()[1] if cap == "out_size" else (big if cap == pd.UNLIMITED else cap)  # noqa: E731
    try:
        def record(r, inb, pos, data):
            t.append((r, inb.pos if inb is not None else None, pos, data, s.finished()) + tuple(s.hints()))

        for chunk, cap in schedule:
            inb = s.put(chunk)
            while len(t) < max_calls:
                before = inb.pos
                r, pos, data = s.call(inb, cap_of(cap))
                record(r, inb, pos, data)
                if r < 0:
                    return t
                if kind == "c":
                    if r == 0 and inb.pos == inb.size:
                        break
                else:
                    if s.finished() or (inb.pos == before and pos == 0):
                        break
                    if inb.pos == inb.size and pos < cap_of(cap):
                        break
        ec = end_cap if end_cap is not None else (schedule[-1][1] if schedule else pd.UNLIMITED)
        s.free_chunk()
        empty = pd.InBuf(None, 0, 0)
        while len(t) < max_calls:
            r, pos, data = s.call(empty, cap_of(ec), fin=(kind == "c"))
            record(r, empty if kind == "d" else None, pos, data)
            if r <= 0:
                break
        return t
    finally:
        s.close()


def same(libs2, make, sched, end_cap=None, offset=1):
    P, R = libs2
    tp = drive_dev(P, make, sched, end_cap=end_cap, offset=offset)
    tr = pd.drive(R, make, sched, end_cap=end_cap)
    assert tp is not None and tr is not None
    if tp != tr:
        for i, (a, b) in enumerate(zip(tp, tr)):
            if a != b:
                pytest.fail(f"call {i}: device {a[:3] + a[4:]} len {len(a[3])}, reference {b[:3] + b[4:]} len {len(b[3])}; "
                            f"bytes equal: {a[3] == b[3]}")
        pytest.fail(f"transcript lengths {len(tp)} vs {len(tr)}")
    return tp


data, copts, dopts, rnd_chunks = tg.data, tg.copts, tg.dopts, tg.rnd_chunks


# ---------------------------------------------------------------------------------------------------------------------
# cstream
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("checksum", [0, 1])
@pytest.mark.parametrize("bs", [4 * KB, 64 * KB, 512 * KB, tg.BS_MAX])
@pytest.mark.parametrize("level", range(1, 8))
def test_cstream_levels(libs2, ref, level, bs, checksum):
    for n in tg._sizes(bs):
        src = data(n)
        t = same(libs2, copts(level, bs, checksum), [(src, pd.UNLIMITED)])
        want = ref.compress(np.frombuffer(src, np.uint8), level=level, block_size=bs, checksum=checksum)
        assert pd.joined(t) == want.tobytes(), n


@pytest.mark.parametrize("sched", ["random", "cap1", "cap13", "out_size", "unlimited_random", "resume"])
@pytest.mark.parametrize("level,bs,checksum", [(3, 4 * KB, 1), (1, 64 * KB, 0), (6, 4 * KB, 0), (5, 64 * KB, 1)])
def test_cstream_schedules(libs2, ref, sched, level, bs, checksum):
    src = data(5 * bs + 17 if sched != "cap1" or bs == 4 * KB else bs + 17, seed=2)  # cap1: one call per byte out
    s, end_cap = tg._csched(src, sched, bs)
    t = same(libs2, copts(level, bs, checksum), s, end_cap, offset=15)
    want = ref.compress(np.frombuffer(src, np.uint8), level=level, block_size=bs, checksum=checksum)
    assert pd.joined(t) == want.tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# dstream
# ---------------------------------------------------------------------------------------------------------------------
D_SCHED = ["one", "random", "cap1", "cap13", "capbelow", "capat", "capabove", "out_size"]


@pytest.mark.parametrize("verify", [0, 1])
@pytest.mark.parametrize("seekable", [0, 1])
@pytest.mark.parametrize("checksum", [0, 1])
@pytest.mark.parametrize("level", [1, 3, 6])
def test_dstream_reference_frames(libs2, ref, level, checksum, seekable, verify):
    bs = 16 * KB
    src = data(7 * bs + 333, seed=level)
    frame = ref.compress(np.frombuffer(src, np.uint8), level=level, block_size=bs, checksum=checksum,
                         seekable=seekable).tobytes()
    for kind in D_SCHED:
        s, end_cap = tg._dsched(frame, kind, bs)
        t = same(libs2, dopts(verify), s, end_cap, offset=1 + 14 * verify)
        assert pd.joined(t) == src and t[-1][4] == 1, kind


@pytest.mark.parametrize("name", tg._golden_valid())
def test_dstream_golden_valid(libs2, name):
    frame = tg._read("valid", name + ".zxc")
    for verify in (0, 1):
        for kind in ("one", "random", "cap13", "capat", "out_size"):
            s, end_cap = tg._dsched(frame, kind, 4 * KB)
            same(libs2, dopts(verify), s, end_cap)


@pytest.mark.parametrize("name", ["bad_block_checksum", "bad_block_type", "bad_enc_lit", "bad_eof_compsize",
                                  "corrupt_payload", "dict_required", "ghi_forged_offset", "glo_forged_enc_off",
                                  "glo_insufficient_slack", "truncated_mid_block", "bad_block_size_field"])
def test_dstream_golden_invalid(libs2, name):
    frame = tg._read("invalid", name + ".zxc")
    for verify in (0, 1):
        for kind in ("one", "random", "cap1", "capat"):
            s, end_cap = tg._dsched(frame, kind, 4 * KB)
            same(libs2, dopts(verify), s, end_cap)


def test_dstream_every_truncation(libs2, ref):
    src, frame = tg._three_block_frame(ref)
    for cut in range(len(frame)):
        t = same(libs2, dopts(cut & 1), [(frame[:cut], pd.UNLIMITED)])
        assert not any(x[4] for x in t), cut


def test_dstream_byte_flips(libs2, ref):
    src, frame = tg._three_block_frame(ref, seekable=1)
    blocks = tg._block_offsets(frame, True)
    p1, _, c1 = blocks[1]
    eof = blocks[-1][0]
    for pos in (blocks[0][0] + 4, p1 + 8 + c1 // 2, p1 + 8 + c1 + 3, eof + 3, len(frame) - 12, len(frame) - 1):
        bad = bytearray(frame)
        bad[pos] ^= 0x80
        for verify in (0, 1):
            for kind in ("one", "random", "cap13"):
                s, end_cap = tg._dsched(bytes(bad), kind, 4 * KB)
                same(libs2, dopts(verify), s, end_cap)


def test_dstream_raw_block_at_chunk_end(libs2, ref):
    """incompressible data gives RAW blocks; every chunk ends right after a block, so the batch's last RAW block ends
    at in->size -- and at its allocation's end -- and is decoded from the staged copy.  A read past in->size does not
    change the result, so it is memcheck over this test (and tests/sanitize_pstream_device.py) that pins the bound."""
    bs = 4 * KB
    rng = np.random.default_rng(5)
    src = rng.integers(0, 256, 6 * bs + 100, dtype=np.uint8).tobytes()
    for cs in (0, 1):
        frame = ref.compress(np.frombuffer(src, np.uint8), level=1, block_size=bs, checksum=cs).tobytes()
        blocks = tg._block_offsets(frame, bool(cs))
        cuts = [0] + [b[0] for b in blocks] + [len(frame)]
        sched = [(frame[a:b], pd.UNLIMITED) for a, b in zip(cuts, cuts[1:]) if b > a]
        t = same(libs2, dopts(cs), sched)
        assert pd.joined(t) == src
        t = same(libs2, dopts(cs), [(frame[:cuts[4]], pd.UNLIMITED), (frame[cuts[4]:], pd.UNLIMITED)], offset=15)
        assert pd.joined(t) == src


def test_dstream_stitched_blocks(libs2, ref):
    bs = 64 * KB
    R = ref.lib
    o = z.CompressOpts(level=3, block_size=bs)
    cctx = R.zxc_create_cctx(C.byref(o))
    parts, total = [], 0
    for i, n in enumerate([1000, bs, 3000, 20000, bs, 1]):
        src = data(n, seed=20 + i)
        dst = (C.c_uint8 * (n + 4096))()
        r = R.zxc_compress_block(cctx, C.cast(C.c_char_p(src), C.c_void_p), n, dst, len(dst), C.byref(o))
        assert r > 0
        parts.append(bytes(dst[:r]))
        total += n
    R.zxc_free_cctx(cctx)
    good = ref.compress(np.frombuffer(b"x", np.uint8), level=3, block_size=bs).tobytes()
    stream = good[:16] + b"".join(parts) + good[-20:-12] + total.to_bytes(8, "little") + b"\0" * 4
    for verify in (0, 1):
        for kind in ("one", "random", "cap1", "cap13", "capbelow", "capat", "out_size"):
            s, end_cap = tg._dsched(stream, kind, bs)
            assert same(libs2, dopts(verify), s, end_cap)[-1][4] == 1


# ---------------------------------------------------------------------------------------------------------------------
# argument verdicts, launches, stream order, threads
# ---------------------------------------------------------------------------------------------------------------------
def test_arguments(libs2):
    P, R = libs2
    st = torch.cuda.current_stream().cuda_stream
    assert not P.zxc_b200_cstream_device_create(C.byref(z.CompressOpts(block_size=1000)))
    d = (C.c_uint8 * 16)()
    assert not P.zxc_b200_cstream_device_create(C.byref(z.CompressOpts(dict=C.cast(d, vp), dict_size=16)))
    assert not P.zxc_b200_dstream_device_create(C.byref(z.DecompressOpts(dict=C.cast(d, vp), dict_size=16)))
    ob, ib = pd.OutBuf(None, 0, 0), pd.InBuf(None, 0, 0)
    assert P.zxc_b200_cstream_device_compress(None, C.byref(ob), C.byref(ib), st) == \
        R.zxc_cstream_compress(None, C.byref(ob), C.byref(ib)) < 0
    for kind in ("c", "d"):
        h = getattr(P, f"zxc_b200_{kind}stream_device_create")(None)
        hr = getattr(R, f"zxc_{kind}stream_create")(None)
        try:
            call = P.zxc_b200_cstream_device_compress if kind == "c" else P.zxc_b200_dstream_device_decompress
            rcall = R.zxc_cstream_compress if kind == "c" else R.zxc_dstream_decompress
            for o, i in ((pd.OutBuf(None, 0, 0), pd.InBuf(None, 5, 0)), (pd.OutBuf(None, 0, 1), pd.InBuf(None, 0, 0)),
                         (pd.OutBuf(None, 0, 0), pd.InBuf(None, 3, 4)), (pd.OutBuf(None, 10, 0), pd.InBuf(None, 0, 0))):
                assert call(h, C.byref(o), C.byref(i), st) == rcall(hr, C.byref(o), C.byref(i))
            assert call(h, None, C.byref(pd.InBuf(None, 0, 0)), st) == rcall(hr, None, C.byref(pd.InBuf(None, 0, 0)))
            assert call(h, C.byref(pd.OutBuf(None, 0, 0)), None, st) == rcall(hr, C.byref(pd.OutBuf(None, 0, 0)), None)
        finally:
            getattr(P, f"zxc_b200_{kind}stream_device_free")(h)
            getattr(R, f"zxc_{kind}stream_free")(hr)
    assert P.zxc_b200_dstream_device_decompress(None, C.byref(ob), C.byref(ib), st) == \
        R.zxc_dstream_decompress(None, C.byref(ob), C.byref(ib)) < 0
    assert P.zxc_b200_dstream_device_finished(None) == 0 and P.zxc_b200_dstream_device_in_size(None) == 0


def _launches(P, make, chunk, cap):
    s = DevStream(P, *make)
    try:
        ib = s.put(chunk)
        before = P.zxc_b200_launch_count()
        r, pos, _ = s.call(ib, cap)
        return P.zxc_b200_launch_count() - before, r, ib.pos, pos
    finally:
        s.close()


def test_launches(libs2, ref):
    """a call that takes one block launches as many kernels as one that takes 1 000"""
    P, _ = libs2
    bs = 4 * KB
    src = data(1000 * bs, seed=31)
    frame = ref.compress(np.frombuffer(src, np.uint8), level=3, block_size=bs).tobytes()
    ends = [b[0] for b in tg._block_offsets(frame, False)]
    l1 = _launches(P, dopts(), frame[:ends[1]], bs)
    l1000 = _launches(P, dopts(), frame[:ends[1000]], 1000 * bs)
    assert l1000[2] == ends[1000] and l1000[3] == 1000 * bs and l1[3] == bs
    assert l1[0] == l1000[0] == 4  # walk, lean and general decode, gather
    # verified checksums: the verifying instance alone decodes
    cframe = ref.compress(np.frombuffer(src, np.uint8), level=3, block_size=bs, checksum=1).tobytes()
    cends = [b[0] for b in tg._block_offsets(cframe, True)]
    v1 = _launches(P, dopts(1), cframe[:cends[1]], bs)
    v1000 = _launches(P, dopts(1), cframe[:cends[1000]], 1000 * bs)
    assert v1000[2] == cends[1000] and v1000[3] == 1000 * bs
    assert v1[0] == v1000[0] == 3  # walk, verifying decode, gather
    c1 = _launches(P, copts(3, bs), src[:bs], 16 + bs + 80)
    c1000 = _launches(P, copts(3, bs), src, 16 + 1000 * (bs + 80))
    assert c1000[1] == 0 and c1000[2] == 1000 * bs
    # the file header's gather (run before the batch reuses the staging slots), encode, trailers, the blocks' gather
    assert c1[0] == c1000[0] == 4


def test_stream_order(libs2, ref):
    """the chunk is written by an async copy on a side stream right before the call that reads it, on that stream"""
    P, _ = libs2
    src = data(3 << 20, seed=41)
    frame = ref.compress(np.frombuffer(src, np.uint8), level=3, block_size=64 * KB, checksum=1).tobytes()
    side = torch.cuda.Stream()
    host = torch.frombuffer(bytearray(frame), dtype=torch.uint8).pin_memory()
    dev = torch.empty(len(frame), dtype=torch.uint8, device="cuda")
    out = torch.empty(len(src) + 4096, dtype=torch.uint8, device="cuda")
    h = P.zxc_b200_dstream_device_create(C.byref(z.DecompressOpts(checksum_enabled=1)))
    try:
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)  # keeps the copy behind a long kernel
            dev.copy_(host, non_blocking=True)
        ib, ob = pd.InBuf(dev.data_ptr(), len(frame), 0), pd.OutBuf(out.data_ptr(), out.numel(), 0)
        r = P.zxc_b200_dstream_device_decompress(h, C.byref(ob), C.byref(ib), side.cuda_stream)
        assert r == len(src) and ob.pos == len(src) and P.zxc_b200_dstream_device_finished(h)
        assert out[:len(src)].cpu().numpy().tobytes() == src
    finally:
        P.zxc_b200_dstream_device_free(h)


def test_two_threads(libs2, ref):
    P, _ = libs2
    srcs = [data(2 << 20, seed=51), data(2 << 20, seed=52)]
    frames = [ref.compress(np.frombuffer(s, np.uint8), level=3, block_size=64 * KB, checksum=1).tobytes() for s in srcs]
    res = [None] * 4

    def work(i):
        st = torch.cuda.Stream()
        if i < 2:
            res[i] = pd.joined(drive_dev(P, dopts(1), [(c, 50000) for c in rnd_chunks(frames[i], i, 200000)], stream=st))
        else:
            res[i] = pd.joined(drive_dev(P, copts(3, 64 * KB, 1), [(c, 50000) for c in rnd_chunks(srcs[i - 2], i, 200000)],
                                         stream=st))

    th = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert res[0] == srcs[0] and res[1] == srcs[1]
    assert res[2] == frames[0] and res[3] == frames[1]


# ---------------------------------------------------------------------------------------------------------------------
# Python
# ---------------------------------------------------------------------------------------------------------------------
def test_python_wrapper(libs2, ref):
    import zxc_b200.device as dv
    import zxc_b200.stream as hs
    src = data(1 << 20, seed=61)
    pieces = rnd_chunks(src, 1, 200000)
    c = dv.compressobj(level=3, block_size=64 * KB, checksum=True)
    dev_frame = torch.cat([c.compress(torch.frombuffer(bytearray(p), dtype=torch.uint8).cuda()) for p in pieces]
                          + [c.flush()]).cpu().numpy().tobytes()
    # the file header, then calls that only fill the accumulator: results of their own size, not 64 MiB views
    c2 = dv.compressobj(level=3, block_size=64 * KB)
    parts = [c2.compress(torch.zeros(100, dtype=torch.uint8, device="cuda")) for _ in range(3)]
    assert [p.numel() for p in parts] == [16, 0, 0] and all(p.untyped_storage().nbytes() <= 16 for p in parts)
    hc = hs.compressobj(level=3, block_size=64 * KB, checksum=True)
    assert dev_frame == b"".join(hc.compress(p) for p in pieces) + hc.flush()
    assert dev_frame == ref.compress(np.frombuffer(src, np.uint8), level=3, block_size=64 * KB, checksum=1).tobytes()
    d = dv.decompressobj(checksum=True)
    g = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()  # noqa: E731
    outs = [d.decompress(g(p)) for p in rnd_chunks(dev_frame + b"tail", 2, 100000)]
    # every piece owns storage of its own size, not the call's whole out buffer
    assert all(o.untyped_storage().nbytes() <= max(o.numel(), 1) for o in outs)
    out = torch.cat(outs)
    assert out.cpu().numpy().tobytes() == src and d.eof and d.unused_data.cpu().numpy().tobytes() == b"tail"
    assert d.decompress(g(b"more")).numel() == 0 and d.unused_data.cpu().numpy().tobytes() == b"tailmore"
    bad = bytearray(dev_frame)
    bad[40] ^= 0x10
    with pytest.raises(dv.ZxcError) as e:
        dv.decompressobj(checksum=True).decompress(g(bytes(bad)))
    tr = pd.drive(pd.bind(ref.lib), dopts(1), [(bytes(bad), pd.UNLIMITED)])
    assert e.value.code == tr[-1][0] < 0
    with pytest.raises(ValueError):
        dv.compressobj(block_size=1000)
    with pytest.raises(ValueError):
        dv.compressobj().compress(torch.zeros(10, dtype=torch.uint8))
    with pytest.raises(ValueError):
        dv.decompressobj().decompress(torch.zeros(10, 2, dtype=torch.uint8, device="cuda").t())
