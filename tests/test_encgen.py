"""The block encoder on inputs shaped for its paths (tests/zxc_encgen.py): the window edge, chain slots recycled inside a
match-finder batch, inserts undone after a long match, hash-bucket pressure, the repeat-offset probe, length and
varint limits, section choices at their thresholds and dictionaries.  A general corpus reaches most of these only by
luck, and several (the saved chain slots, the undo, the repeat probe's arithmetic path) have no counterpart in the
reference, so a fault in them shows only on an input built for it.

Each case must give the reference encoder's frame, byte for byte:
  * on the CPU warp emulator (tests/simt/simt_encode.cc: the kernel source compiled with g++), block by block, under
    four lane schedules, with no store outside a block's slot or the warp's scratch, and with the counter of the path
    it targets non-zero (ZXC_STAT / ZXC_LANE_STAT); a subset also with every buffer against guard pages;
  * on the GPU through zxc_compress (and zxc_decompress gives the input back), and through zxc_compress_block for
    the single-block cases.
The emulator's scheduler itself is checked on partial masks, the way the optimal parser and the PivCo writer use them."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import zxc_ctypes as z
import zxc_encgen as eg
import zxc_simt as zs
from zxc_simt import enc_emu  # noqa: F401  (fixture)

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = eg.all_cases()
EMU = [c for c in CASES if c.emu]
IDS = [c.name for c in CASES]


def _stats(c):
    return c.stat if isinstance(c.stat, tuple) else (c.stat,) if c.stat is not None else ()


def _section(blk, k):
    """the part of a GLO / GHI / RAW block that byte k falls in"""
    if k < 8:
        return "block header"
    if blk[0] == 0:
        return "RAW payload"
    if k < 20:
        return "section header"
    lit_c, enc_lit = int.from_bytes(blk[12:16], "little"), blk[16]
    if blk[0] == 2:
        return "literals" if k < 20 + lit_c else "sequences / extras"
    desc = 20 + (4 if enc_lit else 0) + (4 if blk[17] else 0)
    if k < desc:
        return "section sizes"
    lit_end = desc + (int.from_bytes(blk[20:24], "little") if enc_lit else lit_c)
    return "literals (enc %d)" % enc_lit if k < lit_end else "tokens / offsets / extras"


def _compare(c, level, got, want):
    assert len(got) == len(want), (c.name, level, "block count", len(got), len(want))
    for j, (g, w) in enumerate(zip(got, want)):
        if g != w:
            k = next((i for i in range(min(len(g), len(w))) if g[i] != w[i]), min(len(g), len(w)))
            pytest.fail("%s L%d block %d: %d bytes, reference %d; first difference at byte %d (%s)"
                        % (c.name, level, j, len(g), len(w), k, _section(w, k)))


def _ref_blocks(ref, c, level):
    f = ref.compress(c.data, level=level, block_size=c.bs, checksum=c.checksum, dict=c.dict, dict_huf=c.dict_huf)
    assert not isinstance(f, int), (c.name, level, f)
    return zs.frame_blocks(f, c.checksum), f


def test_catalogue_covers_every_counter():
    assert len(CASES) >= 80 and all(c.doc for c in CASES)
    asserted = {s for c in EMU for s in _stats(c)}
    assert asserted >= set(eg.STAT_NAMES), sorted(set(eg.STAT_NAMES) - asserted)


# ------------------------------------------------------------------------------------------------------------------
# the kernel source on the CPU warp emulator
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", EMU, ids=[c.name for c in EMU])
def test_emulator_matches_reference(case, enc_emu, ref):
    """every level of the case on the emulator: the reference's blocks, nothing stored outside the slots or the
    scratch, the targeted counter non-zero; the highest level also under three more lane schedules (one of them lane
    order)"""
    k = IDS.index(case.name)
    stat = zs.encode_stats(enc_emu)
    C.memset(stat, 0, C.sizeof(stat))
    for level in case.levels:
        want, frame = _ref_blocks(ref, case, level)
        e = zs.encode_frame(enc_emu, case.data, level, case.bs, case.checksum, case.dict, case.dict_huf, seed=1)
        assert e.stray_slot == 0 and e.stray_scratch == 0, (case.name, level, e.stray_slot, e.stray_scratch)
        _compare(case, level, e.blocks, want)
        assert e.body == frame.tobytes()[16:16 + len(e.body)], (case.name, level, "compacted body")
        if hasattr(case, "lit_c"):
            assert int.from_bytes(want[0][12:16], "little") == case.lit_c, "the input no longer gives its literal count"
    hits = [stat[s] for s in _stats(case)]
    assert all(hits), ("targeted path not taken", case.name, [eg.STAT_NAMES[s] for s in _stats(case)], hits)
    level = max(case.levels)
    for seed in (0, 2 + k, 1000 + 7 * k):
        e = zs.encode_frame(enc_emu, case.data, level, case.bs, case.checksum, case.dict, case.dict_huf, seed=seed)
        assert e.stray_slot == 0 and e.stray_scratch == 0
        _compare(case, level, e.blocks, want)


def _corpus():
    from test_oracle import CASES as ORACLE_CASES, make_case
    return [(kind, make_case(kind, min(n, 1 << 17))) for kind, n in ORACLE_CASES]


@pytest.mark.parametrize("level", [1, 3, 5, 6, 7])
def test_emulator_corpus_smoke(level, enc_emu, ref):
    """test_encode_gpu.py's corpus (each input cut to 128 KiB) on the emulator at a fixed lane schedule"""
    for i, (kind, data) in enumerate(_corpus()):
        bs, cks = ((65536, 0), (4096, 1))[i & 1] if data.size <= 70000 else (65536, i & 1)
        c = eg.Case(kind, "", data, (level,), bs, cks)
        want, _ = _ref_blocks(ref, c, level)
        e = zs.encode_frame(enc_emu, data, level, bs, cks, seed=11 + i)
        assert e.stray_slot == 0 and e.stray_scratch == 0, kind
        _compare(c, level, e.blocks, want)


_GUARD_CHILD = r"""
import sys
sys.path.insert(0, %r)
import zxc_ctypes as z, zxc_encgen as eg, zxc_simt as zs
lib = zs.build_encoder(%r)
ref = z.ZxcLib(z.REF_SO)
names = %r
n = 0
for mode in (1, 2):
    lib.simt_enc_guard_pages(mode)
    for c in eg.all_cases():
        if c.name not in names:
            continue
        level = max(c.levels)
        f = ref.compress(c.data, level=level, block_size=c.bs, checksum=c.checksum, dict=c.dict, dict_huf=c.dict_huf)
        e = zs.encode_frame(lib, c.data, level, c.bs, c.checksum, c.dict, c.dict_huf, seed=3)
        assert e.blocks == zs.frame_blocks(f, c.checksum), (c.name, mode)
        assert e.stray_slot == 0 and e.stray_scratch == 0, c.name
        n += 1
print("guard ok", n)
"""
GUARD_CASES = ["tail-n1", "tail-n8", "tail-n13", "tail-2bs+13", "tail-1byte", "dict5-edge", "dict8-edge", "dict4096",
               "dict65535-edge", "huf-shared-800", "len-run65537", "off8-256", "window-d65536-bs128k"]


def test_emulator_loads_stay_inside_the_buffers(ref, tmp_path):
    """Short blocks, tails, dictionaries at both ends and the largest offsets with the source (its 64 bytes of tail
    included), the dictionary buffer, the scratch and the staging slots against PROT_NONE pages, flush with either
    end: a load outside them ends the child process with the faulting buffer+offset."""
    r = subprocess.run([sys.executable, "-c", _GUARD_CHILD % (HERE, str(tmp_path), GUARD_CASES)], capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0 and "guard ok %d" % (2 * len(GUARD_CASES)) in r.stdout, (r.returncode, r.stdout[-1500:],
                                                                                      r.stderr[-1500:])


# ------------------------------------------------------------------------------------------------------------------
# the emulator's scheduler on partial masks
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sched_so(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("simt_sched") / "libsimt_sched.so")
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I.", "-o", so, "simt_sched.cc",
                        "simt_rt.cc"], cwd=zs.SIMT_DIR, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    return so


def test_scheduler_partial_masks(sched_so):
    """disjoint groups shuffle, ballot and reduce at once; a masked match completes next to lanes at a full
    __syncwarp; both under lane order and random schedules"""
    lib = C.CDLL(sched_so)
    for f in (lib.sched_disjoint_groups, lib.sched_masked_match):
        f.argtypes = [C.c_uint64]
        for seed in (0, 1, 2, 99):
            assert f(seed) == 0, (f.__name__, seed)


@pytest.mark.parametrize("fn,msg", [("sched_bad_mask_without_self", "does not name it"),
                                    ("sched_bad_exited_lane", "have exited"),
                                    ("sched_bad_deadlock", "deadlock")])
def test_scheduler_rejects_undefined_behaviour(sched_so, fn, msg):
    """a mask without the calling lane, a mask naming exited lanes and a deadlock abort the (child) process"""
    r = subprocess.run([sys.executable, "-c", "import ctypes; ctypes.CDLL(%r).%s()" % (sched_so, fn)],
                       capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and msg in r.stderr, (r.returncode, r.stderr[-800:])


# ------------------------------------------------------------------------------------------------------------------
# the compiled sm_90a kernels
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_gpu_frames_identical_to_reference(case, prod, ref):
    for level in case.levels:
        a = ref.compress(case.data, level=level, block_size=case.bs, checksum=case.checksum, dict=case.dict,
                         dict_huf=case.dict_huf)
        b = prod.compress(case.data, level=level, block_size=case.bs, checksum=case.checksum, dict=case.dict,
                          dict_huf=case.dict_huf)
        assert not isinstance(b, int), (case.name, level, z.ERR.get(b, b))
        if a.size != b.size or not np.array_equal(a, b):
            _compare(case, level, zs.frame_blocks(b, case.checksum), zs.frame_blocks(a, case.checksum))
            assert a.tobytes() == b.tobytes(), (case.name, level, "frame trailer")
        r, out = prod.decompress(b, case.data.size, checksum=case.checksum, dict=case.dict, dict_huf=case.dict_huf)
        assert r == case.data.size and np.array_equal(out[:r], case.data), (case.name, level, r)


@pytest.mark.gpu
def test_gpu_block_api_identical_to_reference(prod, ref):
    """zxc_compress_block on every single-block case (dictionary attached, no shared table: the block API has none),
    one fresh context per case on either side"""
    n_cases = 0
    for c in CASES:
        if c.data.size == 0 or c.data.size > c.bs:
            continue
        src = np.ascontiguousarray(c.data)
        cap = int(ref.lib.zxc_compress_block_bound(src.size))
        keep = C.create_string_buffer(bytes(c.dict)) if c.dict else None
        rc_ref, rc_prod = ref.lib.zxc_create_cctx(None), prod.lib.zxc_create_cctx(None)
        try:
            for level in c.levels:
                o = z.CompressOpts(level=level, checksum_enabled=c.checksum)
                if c.dict:
                    o.dict, o.dict_size = C.cast(keep, C.c_void_p), len(c.dict)
                a, b = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
                ra = ref.lib.zxc_compress_block(rc_ref, src.ctypes.data, src.size, a.ctypes.data, cap, C.byref(o))
                rb = prod.lib.zxc_compress_block(rc_prod, src.ctypes.data, src.size, b.ctypes.data, cap, C.byref(o))
                assert ra == rb > 0, (c.name, level, ra, rb)
                assert np.array_equal(a[:ra], b[:rb]), (c.name, level)
                n_cases += 1
        finally:
            prod.lib.zxc_free_cctx(rc_prod)
            ref.lib.zxc_free_cctx(rc_ref)
    assert n_cases >= 100
