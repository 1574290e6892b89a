"""Push streaming (zxc_cstream_* / zxc_dstream_*) on paths that need no GPU: option checks, size hints, argument
checks, the empty stream, and every verdict reached before the first block is decoded.  Each test drives the product
and the reference through the same calls and compares the transcripts (tests/zxc_pstream_driver.py)."""
import ctypes as C
import os

import pytest

import zxc_ctypes as z
import zxc_pstream_driver as pd

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _read(*p):
    with open(os.path.join(GOLD, *p), "rb") as f:
        return f.read()


@pytest.fixture(scope="module")
def libs2(prod, ref):
    return pd.bind(prod.lib), pd.bind(ref.lib)


def _copts(**kw):
    return z.CompressOpts(**kw)


def _dopts(**kw):
    return z.DecompressOpts(**kw)


DICT = C.create_string_buffer(b"dictionary content" * 8)

C_OPTS = [
    None,
    dict(),
    dict(level=1), dict(level=7), dict(level=9), dict(level=-2), dict(level=100),
    dict(block_size=4096), dict(block_size=1 << 21), dict(block_size=65536, checksum_enabled=1),
    dict(block_size=1000), dict(block_size=4095), dict(block_size=3 << 12), dict(block_size=1 << 22),
    dict(block_size=2048), dict(block_size=1 << 63),
    dict(seekable=1), dict(n_threads=8), dict(progress_cb=1234),
    dict(dict=C.cast(DICT, C.c_void_p).value, dict_size=16), dict(dict_size=16), dict(dict_huf=C.cast(DICT, C.c_void_p).value),
]


@pytest.mark.parametrize("i", range(len(C_OPTS)))
def test_cstream_create_options(libs2, i):
    P, R = libs2
    kw = C_OPTS[i]
    o = None if kw is None else _copts(**kw)
    hp = P.zxc_cstream_create(C.byref(o) if o is not None else None)
    hr = R.zxc_cstream_create(C.byref(o) if o is not None else None)
    try:
        assert bool(hp) == bool(hr), kw
        if hp:
            assert P.zxc_cstream_in_size(hp) == R.zxc_cstream_in_size(hr)
            assert P.zxc_cstream_out_size(hp) == R.zxc_cstream_out_size(hr)
    finally:
        P.zxc_cstream_free(hp)
        R.zxc_cstream_free(hr)


D_OPTS = [None, dict(), dict(checksum_enabled=1), dict(n_threads=4), dict(dict=C.cast(DICT, C.c_void_p).value),
          dict(dict_size=3), dict(dict_huf=C.cast(DICT, C.c_void_p).value), dict(progress_cb=99)]


@pytest.mark.parametrize("i", range(len(D_OPTS)))
def test_dstream_create_options(libs2, i):
    P, R = libs2
    kw = D_OPTS[i]
    o = None if kw is None else _dopts(**kw)
    hp = P.zxc_dstream_create(C.byref(o) if o is not None else None)
    hr = R.zxc_dstream_create(C.byref(o) if o is not None else None)
    try:
        assert bool(hp) == bool(hr), kw
        if hp:
            assert P.zxc_dstream_in_size(hp) == R.zxc_dstream_in_size(hr)
            assert P.zxc_dstream_out_size(hp) == R.zxc_dstream_out_size(hr)
            assert P.zxc_dstream_finished(hp) == R.zxc_dstream_finished(hr) == 0
    finally:
        P.zxc_dstream_free(hp)
        R.zxc_dstream_free(hr)


def test_null_handles(libs2):
    for L in libs2:
        for k in ("c", "d"):
            assert getattr(L, f"zxc_{k}stream_in_size")(None) == 0
            assert getattr(L, f"zxc_{k}stream_out_size")(None) == 0
            getattr(L, f"zxc_{k}stream_free")(None)
        assert L.zxc_dstream_finished(None) == 0
    P, R = libs2
    ob, ib = pd.OutBuf(None, 0, 0), pd.InBuf(None, 0, 0)
    assert P.zxc_cstream_compress(None, C.byref(ob), C.byref(ib)) == R.zxc_cstream_compress(None, C.byref(ob), C.byref(ib))
    assert P.zxc_cstream_end(None, C.byref(ob)) == R.zxc_cstream_end(None, C.byref(ob))
    assert P.zxc_dstream_decompress(None, C.byref(ob), C.byref(ib)) == R.zxc_dstream_decompress(None, C.byref(ob), C.byref(ib))


@pytest.mark.parametrize("kind", ["c", "d"])
def test_argument_checks(libs2, kind):
    """NULL buffers, out-of-range positions and NULL pointers with room: the same verdict, in the same order, and no
    position moves."""
    frame = _read("valid", "text_1k.zxc")
    buf = C.create_string_buffer(frame, len(frame))
    dst = (C.c_uint8 * 64)()
    def cases():
        return [
            (None, pd.InBuf(C.cast(buf, C.c_void_p), len(frame), 0)),
            (pd.OutBuf(C.cast(dst, C.c_void_p), 64, 0), None),
            (pd.OutBuf(C.cast(dst, C.c_void_p), 64, 0), pd.InBuf(C.cast(buf, C.c_void_p), 4, 5)),
            (pd.OutBuf(C.cast(dst, C.c_void_p), 64, 65), pd.InBuf(C.cast(buf, C.c_void_p), 4, 0)),
            (pd.OutBuf(C.cast(dst, C.c_void_p), 64, 0), pd.InBuf(None, 4, 0)),
            (pd.OutBuf(None, 64, 0), pd.InBuf(C.cast(buf, C.c_void_p), 4, 0)),
            (pd.OutBuf(None, 64, 64), pd.InBuf(None, 4, 4)),  # NULL pointers with nothing left: accepted
        ]

    results = []
    for L in libs2:
        h = getattr(L, f"zxc_{kind}stream_create")(None)
        rs = []
        for ob, ib in cases():
            pob = C.byref(ob) if ob is not None else None
            pib = C.byref(ib) if ib is not None else None
            r = L.zxc_cstream_compress(h, pob, pib) if kind == "c" else L.zxc_dstream_decompress(h, pob, pib)
            rs.append((r, ob.pos if ob is not None else None, ib.pos if ib is not None else None))
        getattr(L, f"zxc_{kind}stream_free")(h)
        results.append(rs)
    assert results[0] == results[1]


@pytest.mark.parametrize("caps", [1, 5, 13, 16, "out_size", pd.UNLIMITED])
@pytest.mark.parametrize("checksum", [0, 1])
@pytest.mark.parametrize("block_size", [0, 4096, 1 << 21])
def test_cstream_empty(libs2, caps, checksum, block_size):
    """header + EOF block + footer, drained whole or a few bytes at a time, with and without a compress call first"""
    P, R = libs2
    o = _copts(level=3, block_size=block_size, checksum_enabled=checksum)
    for sched in ([], [(b"", caps)]):
        tp = pd.drive(P, ("c", o), sched, end_cap=caps)
        tr = pd.drive(R, ("c", o), sched, end_cap=caps)
        assert tp == tr
        assert pd.joined(tp) == pd.joined(tr)
    assert len(pd.joined(tp)) == 16 + 8 + 12


def test_cstream_after_done(libs2):
    """after the end: compress and end both return NULL_INPUT, like the reference"""
    res = []
    for L in libs2:
        h = L.zxc_cstream_create(None)
        dst = (C.c_uint8 * 64)()
        ob = pd.OutBuf(C.cast(dst, C.c_void_p), 64, 0)
        ib = pd.InBuf(None, 0, 0)
        r = [L.zxc_cstream_end(h, C.byref(ob)), ob.pos]
        r += [L.zxc_cstream_end(h, C.byref(ob)), L.zxc_cstream_compress(h, C.byref(ob), C.byref(ib))]
        L.zxc_cstream_free(h)
        res.append(r)
    assert res[0] == res[1]
    assert res[0][2] == -12


@pytest.mark.parametrize("sizes", [[1], [3, 7], [16], [20], [1 << 20]])
@pytest.mark.parametrize("checksum", [0, 1])
def test_dstream_empty_frame(libs2, sizes, checksum):
    """the empty frame up to DONE, with trailing garbage that must not be consumed"""
    P, R = libs2
    frame = _read("valid", "empty.zxc") + b"TRAILING GARBAGE"
    for cap in (0, 1, pd.UNLIMITED):
        sched = [(c, cap) for c in pd.chunks(frame, sizes)]
        tp = pd.drive(P, ("d", _dopts(checksum_enabled=checksum)), sched)
        tr = pd.drive(R, ("d", _dopts(checksum_enabled=checksum)), sched)
        assert tp == tr
    assert any(x[4] for x in tp)


@pytest.mark.parametrize("name", ["bad_magic", "bad_version", "bad_header_crc", "bad_checksum_algo",
                                  "bad_block_size_field", "too_short_4bytes", "zero_length", "all_0xff_garbage",
                                  "magic_then_zeros", "truncated_header_only"])
@pytest.mark.parametrize("sizes", [[1], [5], [1 << 20]])
def test_dstream_header_rejects(libs2, name, sizes):
    P, R = libs2
    frame = _read("invalid", name + ".zxc")
    sched = [(c, 1024) for c in pd.chunks(frame, sizes)] or [(b"", 1024)]
    tp = pd.drive(P, ("d", _dopts(checksum_enabled=1)), sched)
    tr = pd.drive(R, ("d", _dopts(checksum_enabled=1)), sched)
    assert tp == tr


@pytest.mark.parametrize("cut", range(0, 17))
def test_dstream_truncated_file_header(libs2, cut):
    """a stream cut inside its 16-byte file header: no verdict, nothing finished, the same hints"""
    P, R = libs2
    frame = _read("valid", "text_1k.zxc")[:cut]
    for sizes in ([1], [1 << 20]):
        sched = [(c, 4096) for c in pd.chunks(frame, sizes)] or [(b"", 4096)]
        tp = pd.drive(P, ("d", _dopts()), sched)
        tr = pd.drive(R, ("d", _dopts()), sched)
        assert tp == tr
        assert not any(x[4] for x in tp)


def test_dstream_hints_after_header(libs2):
    """in_size / out_size follow the block size of the parsed header (2 MiB frame: a different hint than the default)"""
    P, R = libs2
    frame = _read("valid", "text_64k_bs2m.zxc")
    for L_pair in ((P, R),):
        hs = []
        for L in L_pair:
            h = L.zxc_dstream_create(None)
            before = (L.zxc_dstream_in_size(h), L.zxc_dstream_out_size(h))
            buf = C.create_string_buffer(frame[:16], 16)
            ib = pd.InBuf(C.cast(buf, C.c_void_p), 16, 0)
            ob = pd.OutBuf(None, 0, 0)
            r = L.zxc_dstream_decompress(h, C.byref(ob), C.byref(ib))
            hs.append((before, r, ib.pos, L.zxc_dstream_in_size(h), L.zxc_dstream_out_size(h)))
            L.zxc_dstream_free(h)
        assert hs[0] == hs[1]
        assert hs[0][0] != hs[0][3:]


def test_no_device_latches_on_first_block(prod):
    """without a device, the first call that has to encode or decode a block latches ZXC_B200_ERROR_NO_DEVICE"""
    P = pd.bind(prod.lib)
    if P.zxc_b200_device_count() > 0:
        pytest.skip("a CUDA device is present")
    frame = _read("valid", "text_1k.zxc")
    t = pd.drive(P, ("d", _dopts()), [(frame, 1 << 16)])
    assert t[0][0] == -100 and t[-1][0] == -100
    t = pd.drive(P, ("c", _copts(block_size=4096)), [(b"x" * 5000, 1 << 16)])
    assert t[0][0] == -100
    t = pd.drive(P, ("c", _copts(block_size=4096)), [(b"x" * 100, 1 << 16)])
    assert t[0][0] == 0 and t[-1][0] == -100  # the header drains, the short last block needs the device
