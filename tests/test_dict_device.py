"""Prepared device dictionaries: zxc_b200_dict_device_* and the seven _using_dict variants.

Each variant must give exactly its base call's results and bytes with the same dictionary as host bytes, stage
nothing (so it can be captured in a CUDA graph), launch no seeding kernel, and run in a scratch sized without a
dictionary.  Frame compress is also compared with the reference's zxc_compress where it is built."""
import ctypes as C

import numpy as np
import pytest

import zxc_corpus as zc
from conftest import has_cuda
from test_compress_device import opts
from test_dict_device_host import bind
from test_oracle import golden_dicts

pytestmark = pytest.mark.gpu

CORRUPT, NO_DEVICE, DICT_MISMATCH = -8, -100, -16
REC = 4096


@pytest.fixture(scope="module")
def env(prod):
    if not has_cuda():
        pytest.skip("needs a CUDA device")
    import torch
    import zxc_b200.device as D
    L = bind(prod.lib)
    L.zxc_b200_launch_count.restype = C.c_uint64
    for n in ("encode_scratch_size", "compress_device_batch_scratch_size", "compress_blocks_device_scratch_size",
              "decompress_device_scratch_size", "decompress_inplace_device_scratch_size",
              "decompress_device_batch_scratch_size", "decompress_blocks_device_scratch_size"):
        getattr(L, "zxc_b200_" + n).restype = C.c_size_t
    L.zxc_b200_encode_scratch_size.argtypes = [C.c_uint64, C.c_void_p]
    L.zxc_b200_compress_device_batch_scratch_size.argtypes = [C.c_uint32, C.c_uint64, C.c_void_p]
    L.zxc_b200_compress_blocks_device_scratch_size.argtypes = [C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p]
    L.zxc_b200_decompress_device_scratch_size.argtypes = [C.c_uint64, C.c_uint32]
    L.zxc_b200_decompress_inplace_device_scratch_size.argtypes = [C.c_uint64, C.c_uint32, C.c_uint64]
    L.zxc_b200_decompress_device_batch_scratch_size.argtypes = [C.c_uint32, C.c_uint64, C.c_uint32]
    L.zxc_b200_decompress_blocks_device_scratch_size.argtypes = [C.c_uint32, C.c_uint64]
    return torch, D, L


def train_huf(L, data, d):
    ns = data.size // REC
    ptrs = (C.c_void_p * ns)(*[data.ctypes.data + i * REC for i in range(ns)])
    sizes = (C.c_size_t * ns)(*([REC] * ns))
    huf = np.zeros(128, np.uint8)
    L.zxc_train_dict_huf.restype = C.c_int
    L.zxc_train_dict_huf.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    db = np.frombuffer(d, np.uint8).copy()
    assert L.zxc_train_dict_huf(ptrs, sizes, ns, db.ctypes.data, len(d), huf.ctypes.data) == 0
    return huf.tobytes()


@pytest.fixture(scope="module")
def corpus(libs, env):
    prod, _, ref = libs
    data = zc.records(512, REC)
    trained = zc.train_dict_ref(ref, data, REC, n_samples=512) if ref is not None else \
        zc.silesia_shaped(16384, seed=5).tobytes()
    text = zc.silesia_shaped(1 << 17, seed=6).tobytes()
    dicts = {"trained": (trained, None), "trained+huf": (trained, train_huf(prod.lib, data, trained))}
    for i, (c, h) in enumerate(sorted(golden_dicts().values())):
        dicts[f"golden{i}"] = (c, h)
    for k in (1, 2, 3, 4):
        dicts[f"{k}B"] = (text[:k], None)
    dicts["65535B"] = (text[:65535], None)
    src = np.ascontiguousarray(zc.records(48, REC, seed=11))
    return data, dicts, src


def same_error(f, g):
    """both raise ZxcError with one code, or both return equal tensors"""
    from zxc_b200.device import ZxcError
    try:
        a = f()
    except ZxcError as e:
        with pytest.raises(ZxcError) as e2:
            g()
        assert e2.value.code == e.code
        return e.code
    b = g()
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
    return a


# ---------------------------------------------------------------------------------------------------------------------
# 1. equivalence with the base calls (through the Python helpers, which call the base call for bytes and the variant
#    for a DeviceDict)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", range(1, 8))
def test_frame_compress_and_decode(env, libs, corpus, level):
    torch, D, L = env
    ref = libs[2]
    _, dicts, src = corpus
    s = torch.from_numpy(src).cuda()
    for name, (c, h) in dicts.items():
        with D.DeviceDict(c, h) as dd:
            assert dd.size == len(c) and dd.id == libs[0].lib.zxc_dict_id(c, len(c), h)
            for cks, seek, bs in ((0, 0, 4096), (1, 1, 65536), (1, 0, 4096), (0, 1, 65536)):
                kw = dict(level=level, block_size=bs, checksum=bool(cks), seekable=bool(seek))
                fb = D.compress(s, dict=c, dict_huf=h, **kw)
                fd = D.compress(s, dict=dd, **kw)
                key = (name, cks, seek, bs)
                assert torch.equal(fb.frame, fd.frame) and torch.equal(fb.jobs, fd.jobs), key
                assert fd.dict == c and fd.dict_huf == h
                if ref is not None:
                    want = ref.compress(src, level=level, block_size=bs, checksum=cks, seekable=seek, dict=c,
                                        dict_huf=h)
                    assert fd.frame.cpu().numpy().tobytes() == want.tobytes(), key
                out = same_error(lambda: D.decompress_frame(fb.frame, dict=c, dict_huf=h, checksum=bool(cks)),
                                 lambda: D.decompress_frame(fd.frame, dict=dd, checksum=bool(cks)))
                assert torch.equal(out, s), key
                assert torch.equal(D.decompress(fd), s), key
                buf = same_error(lambda: D.load_frame(fb.frame.cpu().numpy(), dict=c, dict_huf=h, checksum=bool(cks)),
                                 lambda: D.load_frame(fd.frame.cpu().numpy(), dict=dd, checksum=bool(cks)))
                assert torch.equal(buf, s), key


def test_decode_verdicts(env, corpus):
    """another dictionary's frame (DICT_MISMATCH), a frame without a dictionary id, a malformed table, no handle"""
    torch, D, L = env
    _, dicts, src = corpus
    s = torch.from_numpy(src).cuda()
    (c, h), (c2, h2) = dicts["trained+huf"], dicts["golden0"]
    bad = bytes([0xCC]) * 128  # every length 12: a malformed table for both checks
    plain = D.compress(s, level=3, block_size=4096)
    with D.DeviceDict(c, h) as dd, D.DeviceDict(c2, h2) as dd2, D.DeviceDict(c, bad) as dbad:
        other = D.compress(s, level=3, block_size=4096, dict=dd2)
        assert same_error(lambda: D.decompress_frame(other.frame, dict=c, dict_huf=h),
                          lambda: D.decompress_frame(other.frame, dict=dd)) == DICT_MISMATCH
        out = same_error(lambda: D.decompress_frame(plain.frame, dict=c, dict_huf=h),
                         lambda: D.decompress_frame(plain.frame, dict=dd))
        assert torch.equal(out, s)
        assert same_error(lambda: D.compress(s, dict=c, dict_huf=bad), lambda: D.compress(s, dict=dbad)) == CORRUPT
        code = same_error(lambda: D.decompress_frame(plain.frame, dict=c, dict_huf=bad),
                          lambda: D.decompress_frame(plain.frame, dict=dbad))
        assert code == CORRUPT
        same_error(lambda: D.load_frame(plain.frame.cpu().numpy(), dict=c, dict_huf=bad),
                   lambda: D.load_frame(plain.frame.cpu().numpy(), dict=dbad))
        with pytest.raises(ValueError):
            D.compress(s, dict=dd, dict_huf=h)
    with pytest.raises(ValueError):
        dd.handle  # closed


@pytest.mark.parametrize("level", (1, 3, 5, 6))
def test_batches_and_blocks(env, corpus, level):
    torch, D, L = env
    _, dicts, src = corpus
    srcs = [torch.from_numpy(src[i * 3000:i * 3000 + n].copy()).cuda() for i, n in enumerate((0, 1, 4095, 4096,
                                                                                             20000, 70000))]
    for name in ("trained", "trained+huf", "golden1", "3B", "65535B"):
        c, h = dicts[name]
        with D.DeviceDict(c, h) as dd:
            for cks, seek in ((0, 0), (1, 1)):
                kw = dict(level=level, block_size=4096, checksum=bool(cks), seekable=bool(seek))
                ob, rb = D.compress_frames(srcs, dict=c, dict_huf=h, **kw)
                od, rd = D.compress_frames(srcs, dict=dd, **kw)
                assert torch.equal(rb, rd), (name, cks)
                frames = [o[:r] for o, r in zip(od, rd.tolist())]
                for a, b, r in zip(ob, od, rd.tolist()):
                    assert torch.equal(a[:r], b[:r]), (name, cks)
                caps = [t.numel() for t in srcs]
                xb, yb = D.decompress_frames(frames, caps, dict=c, dict_huf=h, checksum=bool(cks))
                xd, yd = D.decompress_frames(frames, caps, dict=dd, checksum=bool(cks))
                assert torch.equal(yb, yd) and yd.tolist() == caps, (name, cks)
                for a, b in zip(xd, srcs):
                    assert torch.equal(a, b)
                bb, rbb = D.compress_blocks(srcs, level=level, checksum=bool(cks), dict=c)
                bd, rbd = D.compress_blocks(srcs, level=level, checksum=bool(cks), dict=dd)
                assert torch.equal(rbb, rbd), (name, cks)
                blocks = []
                for a, b, r in zip(bb, bd, rbd.tolist()):
                    if r > 0:
                        assert torch.equal(a[:r], b[:r])
                    blocks.append(torch.cat([b[:max(r, 0)], torch.zeros(8, dtype=torch.uint8, device="cuda")]))
                for safe in (False, True):
                    sizes = [max(t.numel(), 1) for t in srcs]
                    views = [b[:max(r, 0)] for b, r in zip(blocks, rbd.tolist())]
                    pb, qb = D.decompress_blocks(views, sizes, safe=safe, checksum=bool(cks), dict=c)
                    pd, qd = D.decompress_blocks(views, sizes, safe=safe, checksum=bool(cks), dict=dd)
                    assert torch.equal(qb, qd), (name, cks, safe)
                    for a, b, r in zip(pb, pd, qd.tolist()):
                        if r > 0:
                            assert torch.equal(a[:r], b[:r])


# ---------------------------------------------------------------------------------------------------------------------
# 2-4. graph capture, launch counts and scratch, through the C ABI
# ---------------------------------------------------------------------------------------------------------------------
def dopts(cks=0, d=None, h=None):
    import zxc_ctypes as z
    o = z.DecompressOpts(checksum_enabled=cks)
    o._keep = []
    if d is not None:
        o._keep = [bytes(d), bytes(h) if h is not None else None]
        o.dict, o.dict_size = C.cast(C.c_char_p(o._keep[0]), C.c_void_p), len(d)
        if h is not None:
            o.dict_huf = C.cast(C.c_char_p(o._keep[1]), C.c_void_p)
    return o


class Case:
    """One call on fixed buffers: fill(k) rewrites the inputs (and descriptors) for round k, run(variant, stream)
    enqueues it (the variant with the handle and a scratch sized without a dictionary, or the base call with the
    dictionary in opts and a scratch sized for it), outs() the tensors it writes."""

    def __init__(self, t, fill, run, outs):
        self.t, self.fill, self.run, self.outs = t, fill, run, outs

    def snapshot(self):
        return [o.cpu().numpy().tobytes() for o in self.outs()]

    def clear(self):
        for o in self.outs():
            o.fill_(0x5A)


def build_cases(env, corpus, dd, c, h, level=5, cks=1):
    torch, D, L = env
    t = torch
    _, _, src = corpus
    data = [np.ascontiguousarray(src[:65536 + 77]), np.ascontiguousarray(src[100000:100000 + 65536 + 77])]
    n_items = 5
    pieces = [[np.ascontiguousarray(x[i * 9000:i * 9000 + 3000 + 997 * i]) for i in range(n_items)] for x in data]
    co, cnone = opts(level, 4096, cks, 1, d=c, h=h), opts(level, 4096, cks, 1)
    do = dopts(cks, c, h)
    P = lambda x: t.from_numpy(x.copy()).cuda()  # noqa: E731
    ptr = lambda x: x.data_ptr()  # noqa: E731
    cases = {}

    def scr(size_dict, size_none):
        return t.empty(max(size_dict, size_none) + 256, dtype=t.uint8, device="cuda"), size_dict, size_none

    # compress_device: the input's bytes change between rounds
    N = data[0].size
    s_in = P(data[0])
    cap = 2 * N + 4096
    dst = t.empty(cap, dtype=t.uint8, device="cuda")
    res = t.empty(1, dtype=t.int64, device="cuda")
    nb = (N + 4095) // 4096
    jobs = t.empty(nb * 24, dtype=t.uint8, device="cuda")
    sc = scr(L.zxc_b200_encode_scratch_size(N, C.byref(co)), L.zxc_b200_encode_scratch_size(N, C.byref(cnone)))

    def run_cd(var, st):
        head = (ptr(s_in), N, ptr(dst), cap, C.byref(co))
        tail = (ptr(sc[0]), sc[2] if var else sc[1], ptr(res), ptr(jobs), st)
        return L.zxc_b200_compress_device_using_dict(*head, dd, *tail) if var else L.zxc_b200_compress_device(*head, *tail)
    cases["compress_device"] = Case(t, lambda k: s_in.copy_(P(data[k])), run_cd, lambda: [dst, res, jobs])

    # the batched calls: the items' bytes change and the descriptors are reversed between rounds
    ins = [[P(p) for p in ps] for ps in pieces]
    total = sum(p.size for p in pieces[0])
    bcap = [p.size + 4096 for p in pieces[0]]
    bdst = [t.empty(b, dtype=t.uint8, device="cuda") for b in bcap]
    bres = t.empty(n_items, dtype=t.int64, device="cuda")
    desc = t.empty((n_items, 4), dtype=t.int64, device="cuda")

    def fill_items(k, srcs, sizes, dsts, caps):
        order = list(range(n_items)) if k == 0 else list(reversed(range(n_items)))
        desc.copy_(t.tensor([[ptr(srcs[j]), sizes[j], ptr(dsts[i]), caps[i]] for i, j in enumerate(order)],
                            dtype=t.int64))

    sb = scr(L.zxc_b200_compress_device_batch_scratch_size(n_items, total + 4096, C.byref(co)),
             L.zxc_b200_compress_device_batch_scratch_size(n_items, total + 4096, C.byref(cnone)))

    def run_cb(var, st):
        tail = (ptr(sb[0]), sb[2] if var else sb[1], ptr(bres), st)
        if var:
            return L.zxc_b200_compress_device_batch_using_dict(ptr(desc), n_items, C.byref(co), dd, *tail)
        return L.zxc_b200_compress_device_batch(ptr(desc), n_items, C.byref(co), *tail)
    cases["compress_device_batch"] = Case(
        t, lambda k: fill_items(k, ins[k], [p.size for p in pieces[k]], bdst, bcap), run_cb, lambda: bdst + [bres])

    sk = scr(L.zxc_b200_compress_blocks_device_scratch_size(n_items, total + 4096, 8192, C.byref(co)),
             L.zxc_b200_compress_blocks_device_scratch_size(n_items, total + 4096, 8192, C.byref(cnone)))

    def run_ck(var, st):
        tail = (ptr(sk[0]), sk[2] if var else sk[1], ptr(bres), st)
        if var:
            return L.zxc_b200_compress_blocks_device_using_dict(ptr(desc), n_items, C.byref(co), dd, *tail)
        return L.zxc_b200_compress_blocks_device(ptr(desc), n_items, C.byref(co), *tail)
    cases["compress_blocks_device"] = Case(
        t, lambda k: fill_items(k, ins[k], [p.size for p in pieces[k]], bdst, bcap), run_ck, lambda: bdst + [bres])

    # the decodes: frames / blocks made with the dictionary by the host calls
    prod_lib = L

    def host_frame(x):
        o = opts(level, 4096, cks, 1, d=c, h=h)
        out = np.zeros(2 * x.size + 4096, np.uint8)
        prod_lib.zxc_compress.restype = C.c_int64
        prod_lib.zxc_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
        r = prod_lib.zxc_compress(x.ctypes.data, x.size, out.ctypes.data, out.size, C.byref(o))
        assert r > 0, r
        return out[:r].copy()

    frame = host_frame(data[0])
    f_in = P(frame)
    ddst = t.empty(N, dtype=t.uint8, device="cuda")
    sd = scr(L.zxc_b200_decompress_device_scratch_size(N, 4096), 0)

    def run_dd(var, st):
        head = (ptr(f_in), frame.size, ptr(ddst), N, C.byref(do))
        tail = (ptr(sd[0]), sd[1], ptr(res), st)
        return L.zxc_b200_decompress_device_using_dict(*head, dd, *tail) if var else L.zxc_b200_decompress_device(*head, *tail)
    cases["decompress_device"] = Case(t, lambda k: f_in.copy_(P(frame)), run_dd, lambda: [ddst, res])

    L.zxc_decompress_inplace_bound.restype = C.c_size_t
    L.zxc_decompress_inplace_bound.argtypes = [C.c_void_p, C.c_size_t]
    bound = int(L.zxc_decompress_inplace_bound(frame.ctypes.data, frame.size))
    assert bound > 0
    ibuf = t.empty(bound, dtype=t.uint8, device="cuda")
    si = scr(L.zxc_b200_decompress_inplace_device_scratch_size(bound, 4096, bound), 0)

    def fill_ip(k):
        ibuf.fill_(0)
        ibuf[bound - frame.size:].copy_(P(frame))

    def run_ip(var, st):
        head = (ptr(ibuf), bound, frame.size, C.byref(do))
        tail = (ptr(si[0]), si[1], ptr(res), st)
        if var:
            return L.zxc_b200_decompress_inplace_device_using_dict(*head, dd, *tail)
        return L.zxc_b200_decompress_inplace_device(*head, *tail)
    cases["decompress_inplace_device"] = Case(t, fill_ip, run_ip, lambda: [ibuf, res])

    frames = [[P(host_frame(p)) for p in ps] for ps in pieces]
    ocap = [p.size for p in pieces[0]]
    odst = [t.empty(x, dtype=t.uint8, device="cuda") for x in ocap]
    sf = scr(L.zxc_b200_decompress_device_batch_scratch_size(n_items, total + 4096, 4096), 0)

    def run_db(var, st):
        tail = (ptr(sf[0]), sf[1], ptr(bres), st)
        if var:
            return L.zxc_b200_decompress_device_batch_using_dict(ptr(desc), n_items, C.byref(do), dd, *tail)
        return L.zxc_b200_decompress_device_batch(ptr(desc), n_items, C.byref(do), *tail)
    cases["decompress_device_batch"] = Case(
        t, lambda k: fill_items(k, frames[k], [f.numel() for f in frames[k]], odst, [o.numel() for o in odst]),
        run_db, lambda: odst + [bres])

    def host_block(x):
        o = opts(level, 0, cks, d=c)
        prod_lib.zxc_create_cctx.restype = C.c_void_p
        prod_lib.zxc_free_cctx.argtypes = [C.c_void_p]
        prod_lib.zxc_compress_block.restype = C.c_int64
        prod_lib.zxc_compress_block.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                                C.c_void_p]
        cc = prod_lib.zxc_create_cctx(None)
        out = np.zeros(x.size + 4096, np.uint8)
        r = prod_lib.zxc_compress_block(cc, x.ctypes.data, x.size, out.ctypes.data, out.size, C.byref(o))
        prod_lib.zxc_free_cctx(cc)
        assert r > 0, r
        return np.concatenate([out[:r], np.zeros(8, np.uint8)])  # 8 readable bytes behind each block

    blocks = [[P(host_block(p)) for p in ps] for ps in pieces]
    sbd = scr(L.zxc_b200_decompress_blocks_device_scratch_size(n_items, max(ocap)), 0)

    def run_bd(var, st):
        tail = (ptr(sbd[0]), sbd[1], ptr(bres), st)
        if var:
            return L.zxc_b200_decompress_blocks_device_using_dict(ptr(desc), n_items, C.byref(do), dd, 0, *tail)
        return L.zxc_b200_decompress_blocks_device(ptr(desc), n_items, C.byref(do), 0, *tail)
    cases["decompress_blocks_device"] = Case(
        t, lambda k: fill_items(k, blocks[k], [b.numel() - 8 for b in blocks[k]], odst, [o.numel() for o in odst]),
        run_bd, lambda: odst + [bres])
    cases["_keep"] = (ins, frames, blocks, co, cnone, do)
    return cases


@pytest.mark.parametrize("which", ("trained+huf", "golden0"))
def test_graph_capture_launches_and_scratch(env, corpus, which):
    """Capture each variant once with the handle, replay it with rewritten inputs and descriptors, and compare with
    the base call run eagerly with the dictionary as host bytes (in its own, dictionary-sized scratch); the compress
    variants run in a scratch sized without a dictionary and launch as many kernels as a dictionary-free base call."""
    torch, D, L = env
    t = torch
    c, h = corpus[1][which]
    with D.DeviceDict(c, h) as ddict:
        dd = ddict.handle
        cases = build_cases(env, corpus, dd, c, h)
        keep = cases.pop("_keep")
        co, cnone = keep[3], keep[4]
        for name, cs in cases.items():
            # eager: variant, then base, on the same inputs
            cs.fill(0)
            cs.clear()
            c0 = L.zxc_b200_launch_count()
            assert cs.run(True, None) == 0, name
            n_var = L.zxc_b200_launch_count() - c0
            t.cuda.synchronize()
            got = cs.snapshot()
            cs.clear()
            c0 = L.zxc_b200_launch_count()
            assert cs.run(False, None) == 0, name
            n_base = L.zxc_b200_launch_count() - c0
            t.cuda.synchronize()
            want = cs.snapshot()
            assert got == want, name
            if name.startswith("compress"):
                assert n_var == n_base - 1, (name, n_var, n_base)  # no seeding kernel
            else:
                assert n_var == n_base, (name, n_var, n_base)
            # graph: captured on round 0, replayed on round 1, against the base call on round 1
            s = t.cuda.Stream()
            g = t.cuda.CUDAGraph()
            t.cuda.synchronize()
            with t.cuda.graph(g, stream=s):
                assert cs.run(True, s.cuda_stream) == 0, name
            cs.fill(1)
            cs.clear()
            g.replay()
            t.cuda.synchronize()
            got = cs.snapshot()
            cs.fill(1)
            cs.clear()
            assert cs.run(False, None) == 0, name
            t.cuda.synchronize()
            assert cs.snapshot() == got, (name, "graph")
            del g
        del keep, co, cnone


def test_null_handle_is_a_dictionary_free_call(env, corpus):
    torch, D, L = env
    t = torch
    _, dicts, src = corpus
    c, h = dicts["trained+huf"]
    s = t.from_numpy(src).cuda()
    n = src.size
    co, cnone = opts(5, 4096, 1, 1, d=c, h=h), opts(5, 4096, 1, 1)
    ss = int(L.zxc_b200_encode_scratch_size(n, C.byref(cnone)))
    outs = []
    for var in (True, False):
        dst = t.zeros(2 * n, dtype=t.uint8, device="cuda")
        scr = t.empty(ss, dtype=t.uint8, device="cuda")
        res = t.zeros(1, dtype=t.int64, device="cuda")
        if var:  # opts' dictionary is ignored
            rc = L.zxc_b200_compress_device_using_dict(s.data_ptr(), n, dst.data_ptr(), dst.numel(), C.byref(co),
                                                       None, scr.data_ptr(), ss, res.data_ptr(), None, None)
        else:
            rc = L.zxc_b200_compress_device(s.data_ptr(), n, dst.data_ptr(), dst.numel(), C.byref(cnone),
                                            scr.data_ptr(), ss, res.data_ptr(), None, None)
        assert rc == 0
        t.cuda.synchronize()
        r = int(res.item())
        assert r > 0
        outs.append(dst[:r].cpu().numpy().tobytes())
    assert outs[0] == outs[1]
    want = D.compress(s, level=5, block_size=4096, checksum=True, seekable=True)
    assert want.frame.cpu().numpy().tobytes() == outs[0]


# ---------------------------------------------------------------------------------------------------------------------
# 5-7. sharing, lifetime, wrong device
# ---------------------------------------------------------------------------------------------------------------------
def test_shared_by_two_streams_and_host_bytes_overwritten(env, corpus):
    torch, D, L = env
    t = torch
    _, dicts, src = corpus
    c, h = dicts["trained+huf"]
    cbuf, hbuf = np.frombuffer(c, np.uint8).copy(), np.frombuffer(h, np.uint8).copy()
    err = C.c_int(1)
    dd = L.zxc_b200_dict_device_create(cbuf.ctypes.data, cbuf.size, hbuf.ctypes.data, C.byref(err), None)
    assert dd and err.value == 0
    cbuf[:] = 0xEE  # the handle holds its own copy
    hbuf[:] = 0x11
    try:
        s = t.from_numpy(src).cuda()
        n = src.size
        base = D.compress(s, level=6, block_size=4096, checksum=True, dict=c, dict_huf=h)
        frame = base.frame.clone()
        o = opts(6, 4096, 1)
        do = dopts(1)
        s1, s2 = t.cuda.Stream(), t.cuda.Stream()
        ss = int(L.zxc_b200_encode_scratch_size(n, C.byref(o)))
        ds = int(L.zxc_b200_decompress_device_scratch_size(n, 4096))
        cdst, cscr = t.zeros(2 * n, dtype=t.uint8, device="cuda"), t.empty(ss, dtype=t.uint8, device="cuda")
        ddst, dscr = t.zeros(n, dtype=t.uint8, device="cuda"), t.empty(ds, dtype=t.uint8, device="cuda")
        r1, r2 = t.zeros(1, dtype=t.int64, device="cuda"), t.zeros(1, dtype=t.int64, device="cuda")
        t.cuda.synchronize()
        for _ in range(3):
            assert L.zxc_b200_compress_device_using_dict(s.data_ptr(), n, cdst.data_ptr(), cdst.numel(), C.byref(o), dd,
                                                         cscr.data_ptr(), ss, r1.data_ptr(), None, s1.cuda_stream) == 0
            assert L.zxc_b200_decompress_device_using_dict(frame.data_ptr(), frame.numel(), ddst.data_ptr(), n,
                                                           C.byref(do), dd, dscr.data_ptr(), ds, r2.data_ptr(),
                                                           s2.cuda_stream) == 0
        t.cuda.synchronize()
        assert int(r1.item()) == frame.numel() and torch.equal(cdst[:frame.numel()], frame)
        assert int(r2.item()) == n and torch.equal(ddst, s)
    finally:
        L.zxc_b200_dict_device_free(dd)


def test_wrong_device(env, corpus):
    torch, D, L = env
    t = torch
    if t.cuda.device_count() < 2:
        pytest.skip("needs two visible devices")
    _, dicts, src = corpus
    c, h = dicts["trained"]
    with t.cuda.device(0):
        dd = D.DeviceDict(c)
    with t.cuda.device(1):
        s = t.from_numpy(src).cuda()
        with pytest.raises(D.ZxcError) as e:
            D.compress(s, dict=dd)
        assert e.value.code == NO_DEVICE
        f = D.compress(s, dict=c)
        with pytest.raises(D.ZxcError) as e:
            D.decompress_frame(f.frame, dict=dd)
        assert e.value.code == NO_DEVICE
    dd.close()
