"""Which transfer route a host-buffer decode takes (DESIGN.md section 4), observed through zxc_b200_launch_count().

Every route decodes the same bytes, so a regression in the routing rule would only show as a slower call.  The route
is visible in the launch count, though: without checksum verification every decode step is one lean launch plus one
general launch (zxc_gpu.cu launch_decode), and the routes cut a call into different numbers of such steps."""
import ctypes as C

import numpy as np
import pytest

import zxc_corpus as zc
import zxc_ctypes as z
from test_api_gpu import make_reader

pytestmark = pytest.mark.gpu

BS = 65536
LAUNCHES_PER_STEP = 2          # checksum-free: the lean instance, then the general one for what it deferred
PIPELINED_CHUNK = 64 << 20     # zxg_decode_pipelined: decoded bytes per pipeline stage
STAGED_CHUNK = 32 << 20        # zxg_decode_staged: decoded bytes per output slot (STAGE_OUT)
STREAM_MIN = 32 << 20          # zxc_api.c STREAM_MIN_BYTES: smaller calls take the in-HBM route


def pipelined(decoded):
    return LAUNCHES_PER_STEP * -(-decoded // PIPELINED_CHUNK)


def staged(decoded):
    # level-3 blocks of 64 KiB compress well below the 33 MiB input slot, so the output slot sets the chunk
    return LAUNCHES_PER_STEP * -(-decoded // STAGED_CHUNK)


IN_HBM = LAUNCHES_PER_STEP     # one decode step over all jobs


def covered(off, ln, total):
    """decoded bytes of the whole blocks a range touches"""
    return min(total, (off + ln - 1) // BS * BS + BS) - off // BS * BS


@pytest.fixture(scope="module")
def big(ref):
    data = zc.silesia_shaped(96 << 20, seed=5)
    return data, zc.compress_ref_mt(ref, data, level=3, block_size=BS)


@pytest.fixture
def one_device(monkeypatch):
    monkeypatch.delenv("ZXC_B200_DEVICES", raising=False)


def counted(L, call):
    L.zxc_b200_launch_count.restype = C.c_uint64
    n0 = L.zxc_b200_launch_count()
    r = call()
    return r, L.zxc_b200_launch_count() - n0


def test_frame_routes(prod, ref, big, one_device):
    torch = pytest.importorskip("torch")
    data, frame = big
    L = prod.lib
    assert data.size >= STREAM_MIN
    # pageable: staged
    (r, out), n = counted(L, lambda: prod.decompress(frame, data.size))
    assert r == data.size and np.array_equal(out, data)
    assert n == staged(data.size)
    # page-locked in and out: pipelined
    h_frame = torch.from_numpy(frame).pin_memory()
    h_out = torch.zeros(data.size, dtype=torch.uint8).pin_memory()
    r, n = counted(L, lambda: L.zxc_decompress(h_frame.data_ptr(), h_frame.numel(), h_out.data_ptr(), data.size, None))
    assert r == data.size and np.array_equal(h_out.numpy(), data)
    assert n == pipelined(data.size)
    # under STREAM_MIN decoded: in HBM
    small = data[:8 << 20]
    fs = zc.compress_ref_mt(ref, small, level=3, block_size=BS)
    (r, out), n = counted(L, lambda: prod.decompress(fs, small.size))
    assert r == small.size and np.array_equal(out, small)
    assert n == IN_HBM
    # in place, however large: in HBM (the whole frame is on the device before the first byte comes back)
    L.zxc_decompress_inplace_bound.restype = C.c_size_t
    L.zxc_decompress_inplace_bound.argtypes = [C.c_void_p, C.c_size_t]
    L.zxc_decompress_inplace.restype = C.c_int64
    L.zxc_decompress_inplace.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p]
    b = L.zxc_decompress_inplace_bound(frame.ctypes.data, frame.size)
    buf = np.zeros(b, np.uint8)
    buf[b - frame.size:] = frame
    r, n = counted(L, lambda: L.zxc_decompress_inplace(buf.ctypes.data, b, frame.size, None))
    assert r == data.size and np.array_equal(buf[:data.size], data)
    assert n == IN_HBM


def test_seekable_routes(prod, big, one_device):
    torch = pytest.importorskip("torch")
    data, frame = big
    L = prod.lib
    h_frame = torch.from_numpy(frame).pin_memory()
    hp = L.zxc_seekable_open(h_frame.data_ptr(), h_frame.numel())
    assert hp
    pout = torch.zeros(80 << 20, dtype=torch.uint8).pin_memory()
    # page-locked and block-aligned: pipelined
    off, ln = 16 * BS, 80 << 20
    r, n = counted(L, lambda: L.zxc_seekable_decompress_range(hp, pout.data_ptr(), ln, off, ln))
    assert r == ln and np.array_equal(pout.numpy()[:ln], data[off:off + ln])
    assert n == pipelined(covered(off, ln, data.size))
    # page-locked but ragged at both ends: staged
    off, ln = 16 * BS + 3, (80 << 20) - 5
    r, n = counted(L, lambda: L.zxc_seekable_decompress_range(hp, pout.data_ptr(), ln, off, ln))
    assert r == ln and np.array_equal(pout.numpy()[:ln], data[off:off + ln])
    assert n == staged(covered(off, ln, data.size))
    L.zxc_seekable_free(hp)
    # reader-backed
    calls = []
    rd, keep = make_reader(frame, calls)
    L.zxc_seekable_open_reader.restype = C.c_void_p
    L.zxc_seekable_open_reader.argtypes = [C.c_void_p]
    hr = L.zxc_seekable_open_reader(C.byref(rd))
    assert hr
    for off, ln in ((5 * BS + 1000, (70 << 20) + 3), (123457, 700001)):
        out = np.zeros(ln, np.uint8)
        r, n = counted(L, lambda: L.zxc_seekable_decompress_range(hr, out.ctypes.data, ln, off, ln))
        assert r == ln and np.array_equal(out, data[off:off + ln])
        dec = covered(off, ln, data.size)
        assert n == (staged(dec) if dec >= STREAM_MIN else IN_HBM), (off, ln)
    L.zxc_seekable_free(hr)


def test_failed_small_decodes_leave_the_destination_untouched(prod, ref, big, one_device):
    data, _ = big
    small = data[:3 << 20]
    L = prod.lib
    # a frame with block checksums and one flipped payload byte, decoded with checksum verification
    fc = zc.compress_ref_mt(ref, small, level=3, block_size=BS, checksum=1)
    fc[fc.size // 2] ^= 0x40
    r0, _ = ref.decompress(fc, small.size, checksum=1)
    assert r0 < 0
    out = np.full(small.size, 0xA5, np.uint8)
    o = z.DecompressOpts(checksum_enabled=1)
    assert L.zxc_decompress(fc.ctypes.data, fc.size, out.ctypes.data, out.size, C.byref(o)) == r0
    assert (out == 0xA5).all()
    # a seekable range never verifies checksums: a block header with a bad block type instead
    fs = zc.compress_ref_mt(ref, small, level=3, block_size=BS)
    h = L.zxc_seekable_open(fs.ctypes.data, fs.size)
    nb = L.zxc_seekable_get_num_blocks(h)
    k = nb // 2
    hdr = 16 + sum(L.zxc_seekable_get_block_comp_size(h, i) for i in range(k))  # past the file header
    L.zxc_seekable_free(h)
    fs[hdr] ^= 0x07
    off, ln = k * BS - 1000, 1 << 20
    for lib in (ref.lib, L):
        h = lib.zxc_seekable_open(fs.ctypes.data, fs.size)
        assert h
        out = np.full(ln, 0xA5, np.uint8)
        assert lib.zxc_seekable_decompress_range(h, out.ctypes.data, ln, off, ln) < 0
        lib.zxc_seekable_free(h)
    assert (out == 0xA5).all()  # the product's call


def test_launches_sum_over_device_stripes(prod, ref, monkeypatch):
    """ZXC_B200_DEVICES=all: contiguous block stripes, one per device, each through its own pipeline
    (zxc_api.c decode_multi)."""
    torch = pytest.importorskip("torch")
    L = prod.lib
    ndev = L.zxc_b200_device_count()
    if ndev < 2:
        pytest.skip("needs two devices")
    data = zc.silesia_shaped(192 << 20, seed=7)
    frame = zc.compress_ref_mt(ref, data, level=3, block_size=BS)
    monkeypatch.setenv("ZXC_B200_DEVICES", "all")
    n_blocks = -(-data.size // BS)
    d = min(ndev, 16, data.size >> 26)  # at least 64 MiB of output per stripe
    per = -(-n_blocks // d)
    stripes = [min(per, n_blocks - s) * BS for s in range(0, n_blocks, per)]
    (r, out), n = counted(L, lambda: prod.decompress(frame, data.size))
    assert r == data.size and np.array_equal(out, data)
    assert n == sum(staged(s) for s in stripes)
    h_frame = torch.from_numpy(frame).pin_memory()
    h_out = torch.zeros(data.size, dtype=torch.uint8).pin_memory()
    r, n = counted(L, lambda: L.zxc_decompress(h_frame.data_ptr(), h_frame.numel(), h_out.data_ptr(), data.size, None))
    assert r == data.size and np.array_equal(h_out.numpy(), data)
    assert n == sum(pipelined(s) for s in stripes)
