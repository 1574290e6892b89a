"""Push streaming on the GPU: every call of the product's zxc_cstream_* / zxc_dstream_* against the reference's on
the same schedule (tests/zxc_pstream_driver.py), damaged streams, the batching (one launch for many blocks), two
streams on two threads, and the zxc_b200.stream wrapper."""
import ctypes as C
import os
import random
import threading

import numpy as np
import pytest

import zxc_corpus as zc
import zxc_ctypes as z
import zxc_pstream_driver as pd

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KB = 1024
BS_MAX = 1 << 21


def _read(*p):
    with open(os.path.join(GOLD, *p), "rb") as f:
        return f.read()


@pytest.fixture(scope="module")
def libs2(prod, ref):
    P = pd.bind(prod.lib)
    if P.zxc_b200_device_count() <= 0:
        pytest.skip("no CUDA device")
    P.zxc_b200_launch_count.restype = C.c_uint64
    return P, pd.bind(ref.lib)


_DATA = {}


def data(n, seed=1):
    key = (n, seed)
    if key not in _DATA:
        _DATA[key] = zc.silesia_shaped(max(n, 1), seed=seed)[:n].tobytes()
    return _DATA[key]


def same(libs2, make, sched, end_cap=None):
    P, R = libs2
    tp = pd.drive(P, make, sched, end_cap=end_cap)
    tr = pd.drive(R, make, sched, end_cap=end_cap)
    assert tp is not None and tr is not None
    if tp != tr:  # the first call that differs, without megabytes of payload in the message
        for i, (a, b) in enumerate(zip(tp, tr)):
            if a != b:
                pytest.fail(f"call {i}: product {a[:3] + a[4:]} len {len(a[3])}, reference {b[:3] + b[4:]} len {len(b[3])}; "
                            f"bytes equal: {a[3] == b[3]}")
        pytest.fail(f"transcript lengths {len(tp)} vs {len(tr)}")
    return tp


def copts(level=3, bs=65536, checksum=0):
    return ("c", z.CompressOpts(level=level, block_size=bs, checksum_enabled=checksum))


def dopts(checksum=0):
    return ("d", z.DecompressOpts(checksum_enabled=checksum))


def rnd_chunks(buf, seed, hi):
    r = random.Random(seed)
    out, i = [], 0
    while i < len(buf):
        n = r.randint(1, hi)
        out.append(buf[i:i + n])
        i += n
    return out


# ---------------------------------------------------------------------------------------------------------------------
# cstream
# ---------------------------------------------------------------------------------------------------------------------
def _sizes(bs):
    s = [1, bs - 1, bs, bs + 1]
    if bs <= 512 * KB:
        s.append(5 * bs + 17)
    return s


@pytest.mark.parametrize("checksum", [0, 1])
@pytest.mark.parametrize("bs", [4 * KB, 64 * KB, 512 * KB, BS_MAX])
@pytest.mark.parametrize("level", range(1, 8))
def test_cstream_levels(libs2, ref, level, bs, checksum):
    """every level, block size and checksum flag, the whole input in one call: transcript, and the stream equals the
    reference's non-seekable zxc_compress frame"""
    for n in _sizes(bs):
        src = data(n)
        t = same(libs2, copts(level, bs, checksum), [(src, pd.UNLIMITED)])
        want = ref.compress(np.frombuffer(src, np.uint8), level=level, block_size=bs, checksum=checksum)
        assert pd.joined(t) == want.tobytes(), n


SCHEDULES = ["one", "bytes", "random", "cap1", "cap13", "out_size", "unlimited_random", "resume"]


def _csched(src, kind, bs, seed=5):
    if kind == "one":
        return [(src, pd.UNLIMITED)], None
    if kind == "bytes":
        return [(src[i:i + 1], pd.UNLIMITED) for i in range(len(src))], None
    if kind == "random":
        r = random.Random(seed)
        return [(c, r.choice([1, 13, 100, 4096, bs, 3 * bs, pd.UNLIMITED])) for c in rnd_chunks(src, seed, 3 * bs)], 7
    if kind == "cap1":
        return [(src, 1)], 1
    if kind == "cap13":
        return [(c, 13) for c in rnd_chunks(src, seed, 2 * bs)], 13
    if kind == "out_size":
        return [(c, "out_size") for c in pd.chunks(src, [bs])], "out_size"
    if kind == "unlimited_random":
        return [(c, pd.UNLIMITED) for c in rnd_chunks(src, seed, 4 * bs)], None
    if kind == "resume":  # out fills in the middle of the second block, then drains
        return [(src, 16 + bs // 3), (b"", 5), (b"", 1000), (b"", pd.UNLIMITED)], 50
    raise ValueError(kind)


@pytest.mark.parametrize("sched", SCHEDULES)
@pytest.mark.parametrize("level,bs,checksum", [(3, 4 * KB, 1), (1, 64 * KB, 0), (6, 4 * KB, 0), (5, 64 * KB, 1)])
def test_cstream_schedules(libs2, ref, sched, level, bs, checksum):
    n = 5 * bs + 17
    if sched == "bytes" and bs > 4 * KB:
        n = bs + 17
    src = data(n, seed=2)
    s, end_cap = _csched(src, sched, bs)
    t = same(libs2, copts(level, bs, checksum), s, end_cap)
    want = ref.compress(np.frombuffer(src, np.uint8), level=level, block_size=bs, checksum=checksum)
    assert pd.joined(t) == want.tobytes()


@pytest.mark.parametrize("bs", [64 * KB, 512 * KB])
def test_cstream_corpus(libs2, bs):
    src = data(6 << 20, seed=11)
    for seed in (1, 2):
        same(libs2, copts(3, bs, 1), [(c, pd.UNLIMITED) for c in rnd_chunks(src, seed, 3 << 20)])
    same(libs2, copts(1, bs, 0), [(c, "out_size") for c in pd.chunks(src, [bs])], "out_size")


# ---------------------------------------------------------------------------------------------------------------------
# dstream
# ---------------------------------------------------------------------------------------------------------------------
def _dsched(frame, kind, bs, seed=3):
    if kind == "one":
        return [(frame, pd.UNLIMITED)], None
    if kind == "bytes":
        return [(frame[i:i + 1], pd.UNLIMITED) for i in range(len(frame))], None
    if kind == "random":
        r = random.Random(seed)
        return [(c, r.choice([1, 13, 777, bs, bs + 2111, bs + 2112, bs + 2113, 3 * bs, pd.UNLIMITED]))
                for c in rnd_chunks(frame, seed, 2 * bs)], pd.UNLIMITED
    if kind.startswith("cap"):
        cap = {"cap1": 1, "cap13": 13, "capbs": bs, "capbelow": bs + 2111, "capat": bs + 2112, "capabove": bs + 2113,
               "cap3bs": 3 * bs + 5}[kind]
        return [(c, cap) for c in rnd_chunks(frame, seed, 3 * bs)], cap
    if kind == "out_size":
        return [(c, "out_size") for c in pd.chunks(frame, [bs])], "out_size"
    raise ValueError(kind)


D_SCHED = ["one", "random", "cap1", "cap13", "capbs", "capbelow", "capat", "capabove", "cap3bs", "out_size"]


@pytest.mark.parametrize("verify", [0, 1])
@pytest.mark.parametrize("seekable", [0, 1])
@pytest.mark.parametrize("checksum", [0, 1])
@pytest.mark.parametrize("level", range(1, 8))
def test_dstream_reference_frames(libs2, ref, level, checksum, seekable, verify):
    bs = 16 * KB
    src = data(7 * bs + 333, seed=level)
    frame = ref.compress(np.frombuffer(src, np.uint8), level=level, block_size=bs, checksum=checksum,
                         seekable=seekable).tobytes()
    for kind in D_SCHED:
        s, end_cap = _dsched(frame, kind, bs)
        t = same(libs2, dopts(verify), s, end_cap)
        assert pd.joined(t) == src and t[-1][4] == 1, kind


def test_dstream_one_byte(libs2, ref):
    bs = 4 * KB
    src = data(3 * bs + 100, seed=4)
    frame = ref.compress(np.frombuffer(src, np.uint8), level=3, block_size=bs, checksum=1, seekable=1).tobytes()
    for cap in (pd.UNLIMITED, 1):
        t = same(libs2, dopts(1), [(frame[i:i + 1], cap) for i in range(len(frame))], cap)
        assert pd.joined(t) == src


def _golden_valid():
    d = os.path.join(GOLD, "valid")
    return sorted(f[:-4] for f in os.listdir(d) if f.endswith(".zxc"))


@pytest.mark.parametrize("name", _golden_valid())
def test_dstream_golden_valid(libs2, name):
    """every valid vector; the dictionary frames are decoded without their dictionary (the reference's verdict)"""
    frame = _read("valid", name + ".zxc")
    for verify in (0, 1):
        for kind in ("one", "random", "cap13", "capat", "out_size"):
            s, end_cap = _dsched(frame, kind, 4 * KB)
            same(libs2, dopts(verify), s, end_cap)


@pytest.mark.parametrize("name", ["bad_block_checksum", "bad_block_type", "bad_enc_lit", "bad_eof_compsize",
                                  "corrupt_payload", "dict_required", "ghi_forged_offset", "glo_forged_enc_off",
                                  "glo_insufficient_slack", "truncated_mid_block", "bad_block_size_field"])
def test_dstream_golden_invalid(libs2, name):
    frame = _read("invalid", name + ".zxc")
    for verify in (0, 1):
        for kind in ("one", "random", "cap1", "capat"):
            s, end_cap = _dsched(frame, kind, 4 * KB)
            same(libs2, dopts(verify), s, end_cap)


def _three_block_frame(ref, seekable=0):
    bs = 4 * KB
    src = data(2 * bs + 1500, seed=9)
    return src, ref.compress(np.frombuffer(src, np.uint8), level=3, block_size=bs, checksum=1,
                             seekable=seekable).tobytes()


def test_dstream_every_truncation(libs2, ref):
    src, frame = _three_block_frame(ref)
    for cut in range(len(frame)):
        for verify in (0, 1):
            t = same(libs2, dopts(verify), [(frame[:cut], pd.UNLIMITED)])
            assert not any(x[4] for x in t), cut


def _block_offsets(frame, has_cs):
    """(offset, comp_size) of every block header from the first data block to the EOF block"""
    p, out = 16, []
    while p + 8 <= len(frame):
        comp = int.from_bytes(frame[p + 3:p + 7], "little")
        out.append((p, frame[p], comp))
        if frame[p] == 255:
            break
        p += 8 + comp + (4 if has_cs else 0)
    return out


def test_dstream_byte_flips(libs2, ref):
    """single-byte flips in a block header, a payload, a checksum trailer, the EOF block, the SEK block and the footer"""
    src, frame = _three_block_frame(ref, seekable=1)
    blocks = _block_offsets(frame, True)
    p1, _, c1 = blocks[1]
    eof = blocks[-1][0]
    spots = [blocks[0][0] + 0, blocks[0][0] + 4, blocks[0][0] + 7, p1 + 8 + 3, p1 + 8 + c1 // 2, p1 + 8 + c1,
             p1 + 8 + c1 + 3, eof, eof + 3, eof + 7, eof + 8, eof + 8 + 3, eof + 8 + 8 + 2, len(frame) - 12,
             len(frame) - 5, len(frame) - 1]
    for pos in spots:
        for x in (0x01, 0x80):
            bad = bytearray(frame)
            bad[pos] ^= x
            for verify in (0, 1):
                for kind in ("one", "random", "cap13"):
                    s, end_cap = _dsched(bytes(bad), kind, 4 * KB)
                    same(libs2, dopts(verify), s, end_cap)


def test_dstream_stitched_blocks(libs2, ref):
    """blocks of different decoded sizes, from the reference's block API, stitched into one stream"""
    bs = 64 * KB
    R = ref.lib
    o = z.CompressOpts(level=3, block_size=bs)
    cctx = R.zxc_create_cctx(C.byref(o))
    parts = []
    total = 0
    for i, n in enumerate([1000, bs, 3000, 20000, bs, 1]):
        src = data(n, seed=20 + i)
        dst = (C.c_uint8 * (n + 4096))()
        r = R.zxc_compress_block(cctx, C.cast(C.c_char_p(src), C.c_void_p), n, dst, len(dst), C.byref(o))
        assert r > 0
        parts.append(bytes(dst[:r]))
        total += n
    R.zxc_free_cctx(cctx)
    good = ref.compress(np.frombuffer(b"x", np.uint8), level=3, block_size=bs).tobytes()
    header = good[:16]
    eof = good[-20:-12]
    stream = header + b"".join(parts) + eof + total.to_bytes(8, "little") + b"\0" * 4
    for verify in (0, 1):
        for kind in ("one", "random", "cap1", "cap13", "capbelow", "capat", "out_size"):
            s, end_cap = _dsched(stream, kind, bs)
            t = same(libs2, dopts(verify), s, end_cap)
            assert t[-1][4] == 1


# ---------------------------------------------------------------------------------------------------------------------
# batching
# ---------------------------------------------------------------------------------------------------------------------
def _launches_for(P, make, chunk, cap):
    s = pd.Stream(P, *make)
    try:
        buf = C.create_string_buffer(chunk, len(chunk))
        ib = pd.InBuf(C.cast(buf, C.c_void_p), len(chunk), 0)
        before = P.zxc_b200_launch_count()
        r, pos, _ = s.call(ib, cap)
        return P.zxc_b200_launch_count() - before, r, ib.pos, pos
    finally:
        s.close()


def test_batching_dstream(libs2, ref):
    P, _ = libs2
    bs = 64 * KB
    src = data(64 * bs, seed=31)
    frame = ref.compress(np.frombuffer(src, np.uint8), level=3, block_size=bs).tobytes()
    blocks = _block_offsets(frame, False)
    ends = [b[0] for b in blocks]  # block k ends where block k + 1 starts
    l1 = _launches_for(P, dopts(), frame[:ends[1]], bs)
    l8 = _launches_for(P, dopts(), frame[:ends[8]], 8 * bs)
    l64 = _launches_for(P, dopts(), frame[:ends[64]], 64 * bs)
    assert l8[2] == ends[8] and l8[3] == 8 * bs
    assert l64[2] == ends[64] and l64[3] == 64 * bs
    assert l1[0] == l8[0] == l64[0] > 0
    tiny = _launches_for(P, dopts(), frame, 1)  # one byte of room: a one-block batch
    assert tiny[0] <= l1[0] and tiny[3] == 1


def test_batching_cstream(libs2):
    P, _ = libs2
    bs = 64 * KB
    src = data(64 * bs, seed=32)
    bound = bs + 80
    l1 = _launches_for(P, copts(3, bs), src[:bs], 16 + bound)
    l8 = _launches_for(P, copts(3, bs), src[:8 * bs], 16 + 8 * bound)
    l64 = _launches_for(P, copts(3, bs), src, 16 + 64 * bound)
    assert l8[1] == 0 and l8[2] == 8 * bs and l64[1] == 0 and l64[2] == 64 * bs
    assert l1[0] == l8[0] == l64[0] > 0
    tiny = _launches_for(P, copts(3, bs), src, 1)
    assert tiny[0] <= l1[0]


# ---------------------------------------------------------------------------------------------------------------------
# round trips, threads, Python wrapper
# ---------------------------------------------------------------------------------------------------------------------
def test_round_trip(libs2, ref):
    P, _ = libs2
    src = data(3 << 20, seed=41)
    for level, bs, cs in ((1, 64 * KB, 1), (3, 512 * KB, 0), (7, 64 * KB, 1)):
        t = pd.drive(P, copts(level, bs, cs), [(c, 100000) for c in rnd_chunks(src, level, 1 << 20)])
        frame = pd.joined(t)
        r, out = ref.decompress(frame, len(src), checksum=1)
        assert r == len(src) and out.tobytes() == src
        t2 = pd.drive(P, dopts(1), [(c, 70000) for c in rnd_chunks(frame, 7, 300000)])
        assert pd.joined(t2) == src and t2[-1][4] == 1


def test_two_threads(libs2, ref):
    P, _ = libs2
    srcs = [data(2 << 20, seed=51), data(2 << 20, seed=52)]
    frames = [ref.compress(np.frombuffer(s, np.uint8), level=3, block_size=64 * KB, checksum=1).tobytes() for s in srcs]
    res = [None] * 4

    def work(i):
        if i < 2:
            res[i] = pd.joined(pd.drive(P, dopts(1), [(c, 50000) for c in rnd_chunks(frames[i], i, 200000)]))
        else:
            res[i] = pd.joined(pd.drive(P, copts(3, 64 * KB, 1), [(c, 50000) for c in rnd_chunks(srcs[i - 2], i, 200000)]))

    th = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert res[0] == srcs[0] and res[1] == srcs[1]
    assert res[2] == frames[0] and res[3] == frames[1]


def test_python_wrapper(libs2, ref):
    import zxc_b200.stream as st
    src = data(1 << 20, seed=61)
    c = st.compressobj(level=3, block_size=64 * KB, checksum=True)
    frame = b"".join(c.compress(p) for p in rnd_chunks(src, 1, 200000)) + c.flush()
    assert frame == ref.compress(np.frombuffer(src, np.uint8), level=3, block_size=64 * KB, checksum=1).tobytes()
    d = st.decompressobj(checksum=True)
    out = b"".join(d.decompress(p) for p in rnd_chunks(frame + b"tail", 2, 100000))
    assert out == src and d.eof and d.unused_data == b"tail"
    assert d.decompress(b"more") == b"" and d.unused_data == b"tailmore"
    bad = bytearray(frame)
    bad[40] ^= 0x10
    d = st.decompressobj(checksum=True)
    with pytest.raises(st.ZxcError) as e:
        d.decompress(bytes(bad))
    tr = pd.drive(pd.bind(ref.lib), dopts(1), [(bytes(bad), pd.UNLIMITED)])
    assert e.value.code == tr[-1][0] < 0
    with pytest.raises(st.ZxcError) as e:
        st.decompressobj().decompress(b"not a zxc stream")
    assert e.value.code == -4
    with pytest.raises(ValueError):
        st.compressobj(block_size=1000)
