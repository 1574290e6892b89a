"""zxc_b200_decompress_inplace_device: a frame that lies flush-right in a device buffer decoded into the same buffer.

The oracle is this library's zxc_decompress_inplace on a host buffer with the same contents (pinned to the reference
by test_decode_gpu.py::test_dctx_and_inplace) for its own checks, and zxc_b200_decompress_device with the buffer as
output for everything after them; every valid frame is also compared with its input and, where the reference library
is built, with the reference's zxc_decompress_inplace.  Every call runs twice: with the smallest window (many rounds) and with a window of the
whole buffer (one round).  With more than one round the call has two limits of its own, both ZXC_ERROR_MEMORY; the
round-schedule hazard (limit (a)) is predicted here by a model of the rule written from the header's contract."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

import zxc_corpus as zc
import zxc_ctypes as z
from conftest import has_cuda
from test_decompress_device import _mutants, _stitched, dopts
from test_oracle import G, GC_DICT, INVALID, VALID, golden_dicts, make_case

HDR, FOOT = 16, 12
NULL_INPUT, DST_TOO_SMALL, DICT_BIG, MEMORY, NO_DEVICE = -12, -2, -17, -1, -100
UNIT = 4096
M64 = (1 << 64) - 1


def bind(L):
    L.zxc_b200_decompress_inplace_device_scratch_size.restype = C.c_size_t
    L.zxc_b200_decompress_inplace_device_scratch_size.argtypes = [C.c_uint64, C.c_uint32, C.c_uint64]
    L.zxc_b200_decompress_inplace_device_bound.restype = C.c_size_t
    L.zxc_b200_decompress_inplace_device_bound.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
    L.zxc_b200_decompress_inplace_device.restype = C.c_int
    L.zxc_b200_decompress_inplace_device.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p,
                                                     C.c_size_t, C.c_void_p, C.c_void_p]
    L.zxc_decompress_inplace_bound.restype = C.c_size_t
    L.zxc_decompress_inplace_bound.argtypes = [C.c_void_p, C.c_size_t]
    L.zxc_decompress_inplace.restype = C.c_int64
    L.zxc_decompress_inplace.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p]
    L.zxc_b200_launch_count.restype = C.c_uint64
    return L


def host_bound(L, frame):
    frame = np.ascontiguousarray(frame, np.uint8)
    return int(L.zxc_decompress_inplace_bound(frame.ctypes.data, frame.size))


def window_min(bs):
    return 4 * bs + UNIT


def window_whole(cap):
    return -(-cap // UNIT) * UNIT


def header_bs(frame):
    return 1 << int(frame[5]) if frame.size > 5 and 12 <= frame[5] <= 21 else 4096


def test_host_verdicts_without_a_device(prod):
    """The verdicts that need no buffer bytes come in order without a device; the size queries give 0."""
    if has_cuda():
        pytest.skip("only meaningful without a GPU")
    L = bind(prod.lib)
    fake = 1 << 40  # never dereferenced
    ip = L.zxc_b200_decompress_inplace_device
    big = C.byref(dopts(d=b"x" * 70000))
    assert ip(None, 1000, 100, None, fake, 1 << 20, fake, None) == NULL_INPUT
    assert ip(fake, 1000, 27, None, fake, 1 << 20, fake, None) == NULL_INPUT
    assert ip(fake, 100, 101, None, fake, 1 << 20, fake, None) == NULL_INPUT
    assert ip(fake, 1000, 100, None, None, 1 << 20, fake, None) == NULL_INPUT
    assert ip(fake, 1000, 100, None, fake, 1 << 20, None, None) == NULL_INPUT
    assert ip(fake, 1000, 27, big, fake, 1 << 20, fake, None) == NULL_INPUT
    assert ip(fake, 1000, 100, big, fake, 1 << 20, fake, None) == DICT_BIG
    assert ip(fake, 1000, 100, C.byref(dopts(1)), fake, 0, fake, None) == NO_DEVICE  # before the scratch check
    assert ip(fake, 28, 28, None, fake, 1 << 20, fake, None) == NO_DEVICE
    assert L.zxc_b200_decompress_inplace_device_scratch_size(1 << 20, 65536, 1 << 20) == 0
    assert L.zxc_b200_decompress_inplace_device_scratch_size(1 << 20, 5000, 0) == 0
    assert L.zxc_b200_decompress_inplace_device_bound(fake, 100, None) == 0
    assert L.zxc_b200_decompress_inplace_device_bound(None, 100, None) == 0


def test_python_bound_of_host_frames(prod):
    """device.inplace_bound on host bytes and arrays is zxc_decompress_inplace_bound (no device needed)"""
    from zxc_b200 import device as zd
    L = bind(prod.lib)
    for name in VALID[:6]:
        frame = np.fromfile(os.path.join(G, "valid", name + ".zxc"), np.uint8)
        b = host_bound(L, frame)
        assert b > frame.size
        assert zd.inplace_bound(frame.tobytes()) == b and zd.inplace_bound(frame) == b
        bad = frame.copy()
        bad[0] ^= 1
        assert zd.inplace_bound(bad) == 0


# ---------------------------------------------------------------------------------------------------------------
# a model of the round schedule's hazard rule (limit (a)), from the header's contract
# ---------------------------------------------------------------------------------------------------------------
def _le(b):
    return int.from_bytes(bytes(b), "little")


def _hash8(v):
    h = v ^ 0x9E3779B97F4A7C15
    h ^= (h << 13) & M64
    h ^= h >> 7
    h ^= (h << 17) & M64
    return ((h >> 32) ^ h) & 0xFF


def _walk(frame, bs, trailer):
    """(src_off, src_len) of every block ahead of the end of the block stream, as zxc_decompress walks it"""
    n, ip, jobs = frame.size, HDR, []
    while ip < n:
        rem = n - ip
        if rem < 8:
            break
        v = _le(frame[ip:ip + 8])
        if (v >> 56) != _hash8(v & ((1 << 56) - 1)):
            break
        typ, comp = v & 0xFF, (v >> 24) & 0xFFFFFFFF
        if typ == 255:
            break
        on_disk = 8 + comp + trailer
        jobs.append((ip, min(on_disk, rem)))
        if on_disk >= rem:
            break
        ip += on_disk
    return jobs


def probe_passes(L, frame, cap):
    """zxc_decompress_inplace's own checks ahead of the decode pass"""
    comp = frame.size
    b = host_bound(L, frame) if comp >= HDR + FOOT else 0
    if b == 0:
        return False
    dsize = _le(frame[comp - FOOT:comp - 4])
    return dsize <= cap and cap - dsize >= b - max(dsize, comp)


def predicts_hazard(L, frame, cap, W, B, d=None, h=None):
    """True where the call must give limit (a): the frame passes the checks that come before the plan
    (zxc_decompress_inplace's own, the dictionary id, a block size the scratch holds) and a placed job of the regular
    plan breaks the rule in a schedule of more than one round"""
    comp = frame.size
    if not probe_passes(L, frame, cap):
        return False
    dsize = _le(frame[comp - FOOT:comp - 4])
    bs = 1 << int(frame[5])
    if bs > B:
        return False
    if frame[6] & 0x40:
        did = _le(frame[7:11])
        if d is None or int(prod_dict_id(L, d, h)) != did:
            return False
    R = -(-comp // W)
    if R <= 1:
        return False
    trailer = 4 if frame[6] & 0x80 else 0
    jobs = _walk(frame, bs, trailer)
    n = len(jobs)
    if n == 0:
        return False
    last_start = (n - 1) * bs
    e = 0 if dsize <= last_start else min(bs, dsize - last_start)
    last = e or bs
    n_fit = min(cap // bs, n - 1) if cap // bs < n - 1 else n - 1 + (1 if (n - 1) * bs + last <= cap else 0)
    base, O = cap - comp, B + 12
    for i in range(n_fit):
        off, ln = jobs[i]
        k = off // W
        end = (i + 1) * bs if i + 1 < n else i * bs + last
        if off + ln > k * W + W + O and k * W + W + O + 8 < comp:
            return True
        if k + 1 < R and end + 8 > base + (k + 1) * W:
            return True
    return False


def prod_dict_id(L, d, h):
    L.zxc_dict_id.restype = C.c_uint32
    L.zxc_dict_id.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    return L.zxc_dict_id(bytes(d), len(d), bytes(h) if h is not None else None)


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
class Inplace:
    """zxc_b200_decompress_inplace_device through the C ABI with torch buffers and guard regions"""

    GUARD = 4096

    def __init__(self, prod):
        import torch
        from test_decompress_device import Dev
        self.torch = torch
        self.L = bind(prod.lib)
        self.dev = Dev(prod)

    def scratch_size(self, cap, bs, window):
        return int(self.L.zxc_b200_decompress_inplace_device_scratch_size(cap, bs, window))

    def oracle(self, frame, cap, cks=0, d=None, h=None):
        """zxc_decompress_inplace on a host buffer: (result, decoded bytes)"""
        buf = np.full(cap, 0x3C, np.uint8)
        buf[cap - frame.size:] = frame
        r = int(self.L.zxc_decompress_inplace(buf.ctypes.data, cap, frame.size, C.byref(dopts(cks, d, h))))
        return r, (buf[:r].copy() if r > 0 else np.zeros(0, np.uint8))

    def expected(self, frame, cap, cks=0, d=None, h=None):
        """the parity target: zxc_decompress_inplace's own checks, then what zxc_b200_decompress_device gives for the
        frame and the whole buffer as output (with its limits); on a valid frame both equal zxc_decompress_inplace"""
        r0, o0 = self.oracle(frame, cap, cks, d, h)
        if probe_passes(self.L, frame, cap):
            return self.dev.run(frame, cap, cks, d, h)
        return r0, o0

    def run(self, frame, cap, cks=0, d=None, h=None, window=0, bs=None, lead=0):
        """-> (result, the buffer after the call); guard bytes around the buffer and the scratch must stay as they
        were.  The buffer starts `lead` bytes into its tensor (any alignment)."""
        t, g = self.torch, self.GUARD
        frame = np.asarray(frame, np.uint8)
        bs = bs or header_bs(frame)
        ss = self.scratch_size(cap, bs, window)
        assert ss > 0
        host = np.full(lead + cap + g, 0xA5, np.uint8)
        host[lead:lead + cap] = 0x3C
        host[lead + cap - frame.size:lead + cap] = frame
        buf = t.from_numpy(host).cuda()
        scratch = t.full((ss + 2 * g,), 0x5A, dtype=t.uint8, device="cuda")
        result = t.full((1,), 12345, dtype=t.int64, device="cuda")
        rc = self.L.zxc_b200_decompress_inplace_device(buf.data_ptr() + lead, cap, frame.size,
                                                       C.byref(dopts(cks, d, h)), scratch.data_ptr() + g, ss,
                                                       result.data_ptr(), None)
        assert rc == 0, z.ERR.get(rc, rc)
        t.cuda.synchronize()
        out = buf.cpu().numpy()
        assert (out[:lead] == 0xA5).all() and (out[lead + cap:] == 0xA5).all(), "written outside the buffer"
        assert bool((scratch[:g] == 0x5A).all()) and bool((scratch[g + ss:] == 0x5A).all()), "written outside the scratch"
        return int(result.item()), out[lead:lead + cap]


@pytest.fixture(scope="module")
def ip(prod):
    return Inplace(prod)


def same(ip, frame, cap, cks=0, d=None, h=None, data=None, bs=None, lead=0, split_ok=False, what=None):
    """The call with the smallest and with the whole-buffer window against zxc_decompress_inplace.  With more than one
    round, ZXC_ERROR_MEMORY is accepted where the hazard model predicts it (the buffer is then unchanged), and, with
    split_ok, for a frame whose damage may need the general re-plan (limit (b)).  Returns the one-round result."""
    frame = np.asarray(frame, np.uint8)
    r0, o0 = ip.expected(frame, cap, cks, d, h)
    bs = bs or header_bs(frame)
    res = {}
    for name, window in (("min", 0), ("whole", cap)):
        r, out = ip.run(frame, cap, cks, d, h, window=window, bs=bs, lead=lead)
        W = window_min(bs) if name == "min" else window_whole(cap)
        rounds = -(-frame.size // W)
        if rounds > 1 and predicts_hazard(ip.L, frame, cap, W, bs, d, h):
            assert r == MEMORY, (what, name, z.ERR.get(r, r))
            assert out[cap - frame.size:].tobytes() == frame.tobytes(), (what, "the frame was touched")
        elif not (r == MEMORY and rounds > 1 and split_ok and r0 != MEMORY):
            assert r == r0, (what, name, rounds, z.ERR.get(r, r), z.ERR.get(r0, r0))
            if r0 > 0:
                assert np.array_equal(out[:r], o0), (what, name)
        if data is not None:
            assert r == data.size and np.array_equal(out[:r], data), (what, name)
        res[name] = r
    return res["whole"]


def _ref():
    return z.ZxcLib(z.REF_SO) if z.have_ref() else None


def ref_inplace(ref, frame, cap, cks=0):
    ref.lib.zxc_decompress_inplace.restype = C.c_int64
    ref.lib.zxc_decompress_inplace.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p]
    buf = np.zeros(cap, np.uint8)
    buf[cap - frame.size:] = frame
    r = int(ref.lib.zxc_decompress_inplace(buf.ctypes.data, cap, frame.size,
                                           C.byref(z.DecompressOpts(checksum_enabled=cks))))
    return r, buf[:max(r, 0)]


def _mixed(n, seed):
    """incompressible, all-zero and text runs back to back: both ends of the in-place margin in one frame"""
    rng = np.random.default_rng(seed)
    parts, k = [], 0
    while sum(p.size for p in parts) < n:
        m = int(rng.integers(20000, 90000))
        parts.append([zc.gen_random(m), np.zeros(m, np.uint8), zc.gen_text(m)][k % 3])
        k += 1
    return np.concatenate(parts)[:n]


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, 2, 3, 4, 5, 6, 7])
def test_valid_frames_at_the_bound(ip, prod, level):
    """every valid frame decodes at exactly the bound, with many rounds and with one; one byte less gives
    DST_TOO_SMALL"""
    ref = _ref()
    cases = [("random", zc.gen_random(150000)), ("zeros", np.zeros(300000, np.uint8)), ("mixed", _mixed(400000, 3))]
    every = ((0, 0), (1, 1), (1, 0), (0, 1))
    for kind, data in cases:
        for bs in (4096, 65536) + ((2 << 20,) if kind == "mixed" else ()):
            # every (checksum, seekable) pair at 64 KiB blocks, and one per level at the other sizes
            combos = every if bs == 65536 else (every[(level + len(kind)) % 4],)
            for cks, seek in combos:
                frame = prod.compress(data, level=level, block_size=bs, checksum=cks, seekable=seek)
                cap = host_bound(ip.L, frame)
                what = (kind, level, bs, cks, seek)
                assert same(ip, frame, cap, cks, data=data, what=what) == data.size
                if bs != 65536:
                    continue
                r = same(ip, frame, cap - 1, cks, what=what)
                dsize = data.size
                if dsize >= frame.size:  # the bound is the decoded size's, not the frame's: one byte less is short
                    assert r == DST_TOO_SMALL, what
                else:
                    assert r == dsize, what
                if ref is not None and kind != "zeros":
                    rr, orr = ref_inplace(ref, frame, cap, cks)
                    assert rr == data.size and np.array_equal(orr, data), (what, "reference")


@pytest.mark.gpu
def test_golden_vectors_and_dictionaries(ip, prod):
    dicts = golden_dicts()
    for name in VALID:
        frame = np.fromfile(os.path.join(G, "valid", name + ".zxc"), np.uint8)
        exp = np.frombuffer(open(os.path.join(G, "valid", name + ".expected"), "rb").read(), np.uint8)
        did = _le(frame[7:11]) if frame[6] & 0x40 else 0
        d, h = dicts.get(did, (None, None))
        cap = host_bound(ip.L, frame)
        for cks in (0, 1):
            assert same(ip, frame, cap, cks, d, h, data=exp, what=name) == exp.size
    for p in sorted(glob.glob(os.path.join(G, "format", "*.zxc"))):
        if os.path.basename(p).startswith("12_"):
            continue  # needs a trained literal table (test_decompress_device.py)
        frame = np.fromfile(p, np.uint8)
        same(ip, frame, host_bound(ip.L, frame), 1, GC_DICT if frame[6] & 0x40 else None, what=p)
    data = make_case("text", 150000)
    for d, h in dicts.values():
        for huf in (None, h):
            for bs, cks, seek in ((4096, 1, 1), (65536, 0, 0)):
                frame = prod.compress(data, level=6, block_size=bs, checksum=cks, seekable=seek, dict=d, dict_huf=huf)
                cap = host_bound(ip.L, frame)
                assert same(ip, frame, cap, 1, d, huf, data=data) == data.size
                same(ip, frame, cap, 1)  # DICT_REQUIRED
                same(ip, frame, cap, 1, d[:-1], huf)  # DICT_MISMATCH


@pytest.mark.gpu
def test_invalid_golden_vectors(ip, prod):
    for name in sorted(INVALID):
        frame = np.fromfile(os.path.join(G, "invalid", name + ".zxc"), np.uint8)
        if frame.size < 28:
            continue  # NULL_INPUT on the host: test_host_verdicts_without_a_device
        for cap in (max(host_bound(ip.L, frame), frame.size), frame.size + (1 << 20)):
            same(ip, frame, cap, 1, split_ok=True, what=(name, cap))


@pytest.mark.gpu
def test_mutations(ip, prod):
    d, h = next(iter(golden_dicts().values()))
    data = zc.silesia_shaped(1 << 20, seed=5)[:90000]
    frames = [
        ("lz", prod.compress(data, level=3, block_size=4096, checksum=1), None, None),
        ("huffman", prod.compress(make_case("text", 60000), level=6, block_size=4096, checksum=1), None, None),
        ("seekable", prod.compress(data, level=2, block_size=4096, checksum=1, seekable=1), None, None),
        ("dict", prod.compress(make_case("text", 40000), level=6, block_size=4096, checksum=1, seekable=1, dict=d,
                               dict_huf=h), d, h),
    ]
    for name, frame, dd, hh in frames:
        cap = host_bound(ip.L, frame)
        for k, m in _mutants(frame, 60, seed=len(name) + 100):
            same(ip, m, cap, 1, dd, hh, split_ok=True, what=(name, k))


@pytest.mark.gpu
def test_understated_footer_leaves_the_buffer_untouched(ip, prod):
    """a footer that claims a third of the true size: a buffer sized by it is too small for the blocks' planned
    spans, so with more than one round the call refuses before writing; with one round it gives the oracle's
    verdict"""
    for bs, n in ((4096, 300000), (65536, 3000000)):
        data = make_case("text", n)
        frame = prod.compress(data, level=3, block_size=bs)
        forged = frame.copy()
        forged[-FOOT:-4] = np.frombuffer((data.size // 3).to_bytes(8, "little"), np.uint8)
        cap = host_bound(ip.L, forged)
        assert predicts_hazard(ip.L, forged, cap, window_min(bs), bs), bs
        r, out = ip.run(forged, cap, window=0)
        assert r == MEMORY and out[cap - forged.size:].tobytes() == forged.tobytes()
        assert (out[:cap - forged.size] == 0x3C).all(), "the buffer in front of the frame was written"
        same(ip, forged, cap, what=("forged", bs))


@pytest.mark.gpu
def test_short_non_final_blocks(ip, prod):
    """frames that need the general re-plan: the oracle's verdict in one round, ZXC_ERROR_MEMORY in more"""
    data = zc.silesia_shaped(4 << 20, seed=21)[:2000000]
    for level in (1, 3):
        frame, _ = _stitched(prod, data, 65536, level, 4)
        cap = host_bound(ip.L, frame)
        r0 = ip.expected(frame, cap)[0]
        r1, out = ip.run(frame, cap, window=cap)
        assert r1 == r0 == data.size and np.array_equal(out[:r1], data), level
        assert ip.run(frame, cap, window=0)[0] == MEMORY, level


@pytest.mark.gpu
def test_unaligned_buffers_and_spare_room(ip, prod):
    data = make_case("text", 300000)
    for seek in (0, 1):
        frame = prod.compress(data, level=3, block_size=65536, checksum=1, seekable=seek)
        b = host_bound(ip.L, frame)
        for lead in (1, 7, 13, 4093):
            assert same(ip, frame, b, 1, lead=lead, data=data, what=lead) == data.size
        for cap in (b + 1, b + 100000, b - 1, b - 65536, frame.size):
            same(ip, frame, cap, 1, what=(seek, cap))


@pytest.mark.gpu
def test_frame_of_many_blocks(ip, prod):
    """more than 100 000 blocks of 4 KiB, decoded in place over thousands of rounds and in one"""
    t = ip.torch
    base = zc.silesia_shaped(8 << 20, seed=4)
    n = 100_003 * 4096 + 1234
    data = np.resize(base, n)
    data[::8191] ^= np.uint8(0x5A)  # no two copies of base alike
    frame = prod.compress(data, level=1, block_size=4096)
    cap = host_bound(ip.L, frame)
    expect = t.from_numpy(data).cuda()
    for window in (0, cap):
        ss = ip.scratch_size(cap, 4096, window)
        buf = t.empty(cap, dtype=t.uint8, device="cuda")
        buf[cap - frame.size:].copy_(t.from_numpy(frame))
        scratch = t.empty(ss, dtype=t.uint8, device="cuda")
        res = t.zeros(1, dtype=t.int64, device="cuda")
        assert ip.L.zxc_b200_decompress_inplace_device(buf.data_ptr(), cap, frame.size, None, scratch.data_ptr(), ss,
                                                       res.data_ptr(), None) == 0
        t.cuda.synchronize()
        assert int(res.item()) == n
        assert t.equal(buf[:n], expect), window
        del buf, scratch


@pytest.mark.gpu
def test_launch_count(ip, prod):
    """16 + R (1 + k (2 + c)): R = ceil(comp_size / W), k block sizes from 4 KiB to B, c = checksum verification"""
    t = ip.torch
    data = make_case("text", 300000)
    for bs in (4096, 65536):
        frame = prod.compress(data, level=3, block_size=bs, checksum=1)
        cap = host_bound(ip.L, frame)
        buf = t.empty(cap, dtype=t.uint8, device="cuda")
        res = t.zeros(1, dtype=t.int64, device="cuda")
        for window in (0, 3 * window_min(bs), cap):
            for cks in (0, 1):
                ss = ip.scratch_size(cap, bs, window)
                scratch = t.empty(ss, dtype=t.uint8, device="cuda")
                buf[cap - frame.size:].copy_(t.from_numpy(frame))
                t.cuda.synchronize()
                before = int(ip.L.zxc_b200_launch_count())
                assert ip.L.zxc_b200_decompress_inplace_device(buf.data_ptr(), cap, frame.size,
                                                               C.byref(dopts(cks)), scratch.data_ptr(), ss,
                                                               res.data_ptr(), None) == 0
                count = int(ip.L.zxc_b200_launch_count()) - before
                t.cuda.synchronize()
                assert int(res.item()) == data.size
                W = window_min(bs) if window == 0 else min(-(-window // UNIT) * UNIT, window_whole(cap))
                R = -(-frame.size // W)
                k = (bs // 4096).bit_length()
                assert count == 16 + R * (1 + k * (2 + cks)), (bs, window, cks, count, R)


@pytest.mark.gpu
def test_graph_replay_and_two_streams(ip, prod):
    """The call captured in a CUDA graph with the copy that restores the frame; replays with new frame bytes of the
    same size.  Then two calls on two streams at once."""
    t = ip.torch
    datas = [zc.gen_random(200000) for _ in range(3)]  # incompressible: frames of one size
    frames = [prod.compress(x, level=3, block_size=4096, checksum=1) for x in datas]
    assert len({f.size for f in frames}) == 1
    n = frames[0].size
    cap = host_bound(ip.L, frames[0])
    ss = ip.scratch_size(cap, 4096, 0)
    pristine = t.from_numpy(frames[0]).cuda()
    buf = t.empty(cap, dtype=t.uint8, device="cuda")
    scratch = t.empty(ss, dtype=t.uint8, device="cuda")
    res = t.zeros(1, dtype=t.int64, device="cuda")
    o = dopts(1)
    s = t.cuda.Stream()
    g = t.cuda.CUDAGraph()
    t.cuda.synchronize()
    with t.cuda.graph(g, stream=s):
        buf[cap - n:].copy_(pristine)
        assert ip.L.zxc_b200_decompress_inplace_device(buf.data_ptr(), cap, n, C.byref(o), scratch.data_ptr(), ss,
                                                       res.data_ptr(), s.cuda_stream) == 0
    for x, f in zip(datas, frames):
        pristine.copy_(t.from_numpy(f))
        g.replay()
        t.cuda.synchronize()
        assert int(res.item()) == x.size and np.array_equal(buf[:x.size].cpu().numpy(), x)
    bad = frames[1].copy()
    bad[HDR + 8 + 100] ^= 1  # a RAW payload byte: BAD_CHECKSUM
    pristine.copy_(t.from_numpy(bad))
    g.replay()
    t.cuda.synchronize()
    assert int(res.item()) == ip.oracle(bad, cap, 1)[0]
    del g
    streams = [t.cuda.Stream(), t.cuda.Stream()]
    bufs, scrs, rs = [], [], []
    for st, f in zip(streams, frames[:2]):
        b = t.empty(cap, dtype=t.uint8, device="cuda")
        b[cap - n:].copy_(t.from_numpy(f))
        bufs.append(b)
        scrs.append(t.empty(ss, dtype=t.uint8, device="cuda"))
        rs.append(t.zeros(1, dtype=t.int64, device="cuda"))
    t.cuda.synchronize()
    for st, b, sc, r in zip(streams, bufs, scrs, rs):
        assert ip.L.zxc_b200_decompress_inplace_device(b.data_ptr(), cap, n, None, sc.data_ptr(), ss, r.data_ptr(),
                                                       st.cuda_stream) == 0
    t.cuda.synchronize()
    for b, r, x in zip(bufs, rs, datas):
        assert int(r.item()) == x.size and np.array_equal(b[:x.size].cpu().numpy(), x)


@pytest.mark.gpu
def test_python_helpers(ip, prod):
    from zxc_b200 import device as zd
    t = ip.torch
    data = zc.silesia_shaped(4 << 20, seed=9)[:2000000]
    d, h = next(iter(golden_dicts().values()))
    for kw in ({}, {"checksum": True}):
        frame = prod.compress(data, level=3, block_size=65536, checksum=int(bool(kw)), seekable=1)
        b = host_bound(ip.L, frame)
        dev_frame = t.from_numpy(frame).cuda()
        assert zd.inplace_bound(dev_frame) == b == zd.inplace_bound(frame.tobytes())
        out = zd.load_frame(frame.tobytes(), **kw)
        assert out.is_cuda and np.array_equal(out.cpu().numpy(), data)
        for window in (None, 1, 1 << 20):  # 1: the smallest window, several rounds
            buf = t.empty(b, dtype=t.uint8, device="cuda")
            buf[b - frame.size:].copy_(dev_frame)
            out = zd.decompress_inplace(buf, frame.size, window=window, **kw)
            assert out.data_ptr() == buf.data_ptr() and np.array_equal(out.cpu().numpy(), data)
    text = make_case("text", 100000)
    fd = prod.compress(text, level=5, block_size=4096, dict=d, dict_huf=h)
    assert np.array_equal(zd.load_frame(fd, dict=d, dict_huf=h).cpu().numpy(), text)
    with pytest.raises(zd.ZxcError) as e:
        zd.load_frame(fd)
    assert e.value.code == ip.oracle(fd, host_bound(ip.L, fd))[0]
    bad = fd.copy()
    bad[0] ^= 1
    with pytest.raises(zd.ZxcError) as e:
        zd.load_frame(bad)
    assert e.value.code == ip.oracle(bad, bad.size)[0]
    small = t.from_numpy(fd).cuda()
    with pytest.raises(zd.ZxcError) as e:
        zd.decompress_inplace(small, fd.size, dict=d, dict_huf=h)
    assert e.value.code == DST_TOO_SMALL
