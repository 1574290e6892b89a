"""The two-launch decode route.  Without checksum verification a decode runs the lean kernel instance first: it decodes
RAW blocks and GLO blocks with raw tokens and raw or RLE literals, and defers every other block (GHI, Huffman literals,
Huffman tokens) to the general instance, which runs second.  One job table mixes all of these shapes; each job's
output and status must equal what the reference decodes -- on the warp emulator (CPU, tests/simt/simt_lean.cc) and
through the C ABI on the GPU, with and without a dictionary, and with more deferred jobs than the deferred-job list
holds.  The emulator also runs the reference differential and the damaged-block parity along this route."""
import ctypes as C
import os

import numpy as np
import pytest

import zxc_corpus as zc
import zxc_ctypes as z
import zxc_simt as zs
from zxc_simt import lean_emu  # noqa: F401  (fixture)
from test_oracle import CASES, G, make_case

BLOCK_CAP = 65536
DEFER_CAP = 1 << 16  # zxc_gpu.cu: deferred jobs the list holds; beyond that the general launch scans the status array


def plan_frame(prod, fb):
    """the job list the product's host code plans for the frame bytes `fb`"""
    prod.lib.zxc_b200_plan_frame.restype = C.c_int64
    prod.lib.zxc_b200_plan_frame.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    nb = prod.lib.zxc_b200_plan_frame(fb, len(fb), None, 0, None)
    assert nb >= 0, nb
    jobs = (zs.Job * max(nb, 1))()
    assert prod.lib.zxc_b200_plan_frame(fb, len(fb), jobs, nb, None) == nb
    return jobs[:nb]


def emu_decode(lib, src, jobs, total, dict_bytes=None, seed=1):
    """(status list, decoded bytes, stores outside the destination, jobs the lean instance deferred)"""
    nb = len(jobs)
    table = (zs.Job * max(nb, 1))(*jobs)
    out = np.zeros(max(total, 1), np.uint8)
    status = (C.c_int32 * max(nb, 1))()
    oob = C.c_int(0)
    s = np.frombuffer(src, np.uint8)
    d = np.frombuffer(dict_bytes, np.uint8) if dict_bytes else None
    lib.simt_decode_two_stage(s.ctypes.data, s.size, out.ctypes.data, total, table, nb, status,
                              d.ctypes.data if d is not None else None, d.size if d is not None else 0, None, BLOCK_CAP,
                              seed, C.byref(oob))
    return list(status)[:nb], out[:total], oob.value, C.c_uint32.in_dll(lib, "simt_lean_deferred").value


def _shape(fb, job):
    t = fb[job.src_off]
    if t == 1:
        lit, tok = fb[job.src_off + 8 + 8], fb[job.src_off + 8 + 9]
        return "glo-huf-tok" if tok == 2 else "glo-huf-lit" if lit >= 2 else "glo-rle" if lit == 1 else "glo-raw"
    return {0: "raw", 2: "ghi"}[t]


def _frames(ref, dict_bytes):
    """(frame, decoded bytes) pairs that between them hold every block shape"""
    sil = zc.silesia_shaped(1 << 20, seed=3)
    text = make_case("text", 300000)
    out = []
    for data, level, bs in ((text[:40000], 1, 4096),      # GHI
                            (sil[:300000], 3, 4096),      # GLO, raw literals, and RAW
                            (make_case("random", 9000), 3, 4096),  # RAW
                            (text[:60000], 6, 4096),      # Huffman literals
                            (sil[:200000], 7, 65536)):    # Huffman literals and tokens
        out.append((ref.compress(data, level=level, block_size=bs, dict=dict_bytes), data))
    rle = np.frombuffer(open(os.path.join(G, "format", "11_glo_rle.zxc"), "rb").read(), np.uint8)
    r, want = ref.decompress(rle)
    assert r > 0
    out.append((rle, want))
    return out


def mixed_table(prod, ref, dict_bytes=None, extra_deferred=0):
    """(src bytes, jobs, expected output, shape per job): the blocks of _frames() in one table, interleaved, plus
    `extra_deferred` more jobs that decode the first GHI block again into fresh output"""
    src, want, per_frame, base_s, base_d = [], [], [], 0, 0
    for frame, data in _frames(ref, dict_bytes):
        fb = frame.tobytes()
        jobs = plan_frame(prod, fb)
        assert sum(j.dst_cap for j in jobs) == data.size
        rows = []
        for j in jobs:
            rows.append((zs.Job(j.src_off + base_s, j.dst_off + base_d, j.src_len, j.dst_cap), _shape(fb, j)))
        per_frame.append(rows)
        src.append(fb)
        want.append(np.asarray(data, np.uint8))
        base_s += len(fb)
        base_d += data.size
    rows = []  # round robin over the frames: neighbouring jobs have different shapes
    for k in range(max(len(r) for r in per_frame)):
        rows += [r[k] for r in per_frame if k < len(r)]
    want = np.concatenate(want)
    if extra_deferred:
        g = next(j for j, s in rows if s == "ghi")
        first = want[g.dst_off:g.dst_off + g.dst_cap]
        rows += [(zs.Job(g.src_off, base_d + k * g.dst_cap, g.src_len, g.dst_cap), "ghi") for k in range(extra_deferred)]
        want = np.concatenate([want, np.tile(first, extra_deferred)])
    jobs = [j for j, _ in rows]
    shapes = [s for _, s in rows]
    assert set(shapes) == {"raw", "ghi", "glo-raw", "glo-rle", "glo-huf-lit", "glo-huf-tok"}, set(shapes)
    return b"".join(src), jobs, want, shapes


def _dictionary(ref):
    recs = zc.records(64, record_size=4096, seed=7)
    return zc.train_dict_ref(ref, recs, record_size=4096, n_samples=64, cap=16384)


def _expect(got_status, out, jobs, want):
    bad = [(k, z.ERR.get(s, s)) for k, (s, j) in enumerate(zip(got_status, jobs)) if s != j.dst_cap]
    assert not bad, bad[:5]
    assert np.array_equal(out, want)


@pytest.mark.parametrize("with_dict", [False, True], ids=["no-dict", "dict"])
def test_emulator_mixed_job_table(prod, ref, lean_emu, with_dict):
    d = _dictionary(ref) if with_dict else None
    src, jobs, want, shapes = mixed_table(prod, ref, d)
    st, out, oob, deferred = emu_decode(lean_emu, src, jobs, want.size, d, seed=7)
    assert oob == 0, "stores outside the destination"
    _expect(st, out, jobs, want)
    assert deferred == sum(s not in ("raw", "glo-raw", "glo-rle") for s in shapes)


@pytest.mark.parametrize("kind,n", [(k, min(n, 1 << 19)) for k, n in CASES])
def test_emulator_route_vs_reference(prod, ref, lean_emu, kind, n):
    data = make_case(kind, n)
    for level in (1, 3, 5, 7):
        for bs in (4096, 65536):
            fb = ref.compress(data, level=level, block_size=bs, seekable=1).tobytes()
            jobs = plan_frame(prod, fb)
            st, out, oob, _ = emu_decode(lean_emu, fb, jobs, data.size, seed=level * 31 + bs)
            assert oob == 0, "stores outside the destination"
            _expect(st, out, jobs, data)


def test_emulator_route_damaged_blocks_fail_like_the_reference(prod, ref, lean_emu):
    """single-byte damage inside the payloads of level-3 blocks, which the lean instance decodes: a block the reference
    rejects is rejected, a frame the reference still decodes gives the same bytes"""
    data = zc.silesia_shaped(3 * 65536, seed=5)
    fb = ref.compress(data, level=3, block_size=65536, checksum=0, seekable=0).tobytes()
    jobs = plan_frame(prod, fb)
    rng = np.random.default_rng(13)
    checked = 0
    for _ in range(60):
        b = bytearray(fb)
        j = jobs[int(rng.integers(0, len(jobs)))]
        b[int(rng.integers(j.src_off + 8 + 12, j.src_off + j.src_len))] ^= int(rng.integers(1, 256))
        r_ref, out_ref = ref.decompress(bytes(b), data.size)
        st, out, oob, deferred = emu_decode(lean_emu, bytes(b), jobs, data.size, seed=3)
        assert oob == 0
        bad = [s for s, jj in zip(st, jobs) if s != jj.dst_cap]
        if r_ref == data.size:
            assert not bad and np.array_equal(out, out_ref)
        else:
            assert bad, "the reference rejects, the kernel source accepts"
        checked += 1
    assert checked == 60


def _gpu_decode(prod, src, jobs, total, dict_bytes):
    import torch
    lib = prod.lib
    lib.zxc_b200_decode_scratch_size.restype = C.c_size_t
    lib.zxc_b200_decode_scratch_size.argtypes = [C.c_uint32]
    lib.zxc_b200_decode_blocks.restype = C.c_int
    lib.zxc_b200_decode_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                           C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_int, C.c_void_p]
    dev = torch.device("cuda", 0)
    table = (zs.Job * len(jobs))(*jobs)
    d_src = torch.from_numpy(np.frombuffer(src, np.uint8).copy()).to(dev)
    d_dst = torch.zeros(total, dtype=torch.uint8, device=dev)
    d_jobs = torch.from_numpy(np.frombuffer(bytes(table), np.uint8).copy()).to(dev)
    d_status = torch.zeros(len(jobs), dtype=torch.int32, device=dev)
    d_dict = torch.from_numpy(np.frombuffer(dict_bytes, np.uint8).copy()).to(dev) if dict_bytes else None
    ss = lib.zxc_b200_decode_scratch_size(BLOCK_CAP)
    d_scratch = torch.empty(ss, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev)
    rc = lib.zxc_b200_decode_blocks(d_src.data_ptr(), d_dst.data_ptr(), d_jobs.data_ptr(), len(jobs), d_status.data_ptr(),
                                    d_dict.data_ptr() if d_dict is not None else None,
                                    len(dict_bytes) if dict_bytes else 0, None, d_scratch.data_ptr(), ss, BLOCK_CAP, 0,
                                    stream.cuda_stream)
    assert rc == 0, z.ERR.get(rc, rc)
    torch.cuda.synchronize(dev)
    return list(d_status.cpu().numpy()), d_dst.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("with_dict,extra", [(False, 0), (True, 0), (False, DEFER_CAP + 100)],
                         ids=["no-dict", "dict", "deferred-list-overflow"])
def test_gpu_mixed_job_table(prod, ref, with_dict, extra):
    d = _dictionary(ref) if with_dict else None
    src, jobs, want, _ = mixed_table(prod, ref, d, extra_deferred=extra)
    st, out = _gpu_decode(prod, src, jobs, want.size, d)
    _expect(st, out, jobs, want)
