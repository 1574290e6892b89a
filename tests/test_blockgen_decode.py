"""The block decoder on synthetic sequence streams (tests/zxc_blockgen.py) built to reach each shape-dependent path of
decode_lz_block (zxc_b200/csrc/zxc_decode.cuh): short-offset period replication, the per-lane / balanced / byte copy
choices and their length, ring-wrap and near/far thresholds, partial batches with the escape ordinals re-based or the
varint cursor re-walked, giant sequences that bypass the ring, the sequence-order tail, dictionary sources at and
around the dictionary's ends, offset and varint limits, sequence counts, RLE runs and the first-failing-sequence
verdicts.  Reference-encoded frames rarely or never contain most of these shapes.

Each case must agree three ways: the generator's own byte loop, the oracle's zxo_decode_block, and the kernel -- on
the CPU warp emulator (both bodies, several lane schedules, the two-launch lean route, and with the buffers against
guard pages), and on the GPU through zxc_b200_decode_blocks, zxc_decompress and zxc_decompress_block.  On the
emulator each case also asserts that the path it targets was taken (the ZXC_STAT counters of tests/simt)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import zxc_blockgen as bg
import zxc_ctypes as z
import zxc_simt as zs
from zxc_blockgen import Block, Seq
from zxc_simt import lean_emu  # noqa: F401  (fixture)

BLOCK_CAP = 1 << 17  # launch block size: room for 65536-byte offsets inside one block
RING = 4096
RING_LIMIT = RING - 576
ROOM = {-2: -10}  # DST_TOO_SMALL where a frame driver reports what the kernel calls OVERFLOW

# ZXC_STAT counters of the emulator build (zxc_decode.cuh)
S_BATCH, S_LANE, S_LONG, S_TAIL = 0, 3, 4, 12
S_GIANT, S_PARTIAL, S_PARTIAL_WALK, S_REPL = 9, 10, 11, 15
S_DICT_BYTE, S_DICT_WORD, S_MATCH_BYTE, S_VERDICT, S_RING_WORD, S_GLOBAL_WORD = 16, 17, 18, 19, 20, 21


def _walk_pad():
    """extras-section padding that makes the escape values too many for the rank-table scratch (use_vals == false)"""
    cum = (11 * (((BLOCK_CAP + 255) & ~255) // 8) + 4 * 512 + 255) & ~255  # scr_cum_cap(BLOCK_CAP)
    return cum // 4 + 64


class Case:
    def __init__(self, name, block, stat):
        self.name, self.block, self.stat = name, block, stat  # stat: counter index that must be non-zero, or None

    def __repr__(self):
        return self.name


class Builder:
    """sequences at known absolute output positions; `src` (absolute, negative = dictionary) or `off` places a source"""

    def __init__(self, seed, dict_bytes=b""):
        self.rng = np.random.default_rng(seed)
        self.seqs, self.pos, self.dict_bytes = [], 0, bytes(dict_bytes)

    def add(self, ll, ml, off=None, src=None, **kw):
        mdst = self.pos + ll
        if src is not None:
            off = mdst - src
        s = Seq(self.rng.bytes(ll), ml, off, **kw)
        self.seqs.append(s)
        self.pos = mdst + ml
        return s

    def fill(self, n, **kw):
        for s in bg.fill_seqs(n, self.rng, start=self.pos, **kw):
            self.seqs.append(s)
        self.pos += n

    def batch(self, total, targets=None, n=32):
        """n sequences adding exactly `total` bytes: lane j is targets[j] = (ll, ml, dict(off= or src=, ...)) when
        given, the others are fillers (2 literals and a match from 64..1024 back) sharing the rest"""
        targets = targets or {}
        fixed = sum(t[0] + t[1] for t in targets.values())
        n_fill = n - len(targets)
        share = (total - fixed) // max(n_fill, 1)
        last_fill = max([j for j in range(n) if j not in targets], default=-1)
        for j in range(n):
            if j in targets:
                ll, ml, kw = targets[j]
                self.add(ll, ml, **kw)
            else:
                size = share + ((total - fixed) - share * n_fill if j == last_fill else 0)
                assert size >= 7, size
                self.add(2, size - 2, off=int(self.rng.integers(min(64, self.pos + 2), min(1024, self.pos + 2) + 1)))

    def block(self, tail=8, **kw):
        kw.setdefault("dict_bytes", self.dict_bytes)
        return Block(self.seqs, self.rng.bytes(tail), **kw)


# ------------------------------------------------------------------------------------------------------------------
# the catalogue
# ------------------------------------------------------------------------------------------------------------------
def _short_offsets():
    mls = [5, 6, 7, 8, 12, 13, 16, 17, 27, 28, 29, 31, 32, 33, 47, 64, 65, 100]
    for off in range(1, 34):
        b = Builder(100 + off)
        b.add(40, 5, off=min(off, 40))
        for cyc in range(5):
            for k, ml in enumerate(mls):
                b.add((k * 7 + cyc * 3) % 19, ml, off=off)
        kind = "ghi" if off % 4 == 0 else "glo"
        yield Case("short-off-%d" % off, b.block(kind=kind, enc_off=off % 2), S_REPL if off < 32 else S_TAIL)


def _thresholds():
    # literal and match lengths on either side of the per-lane limit (LIT_SHORT = MATCH_SHORT = 28)
    for ll, ml in ((28, 28), (29, 29), (28, 29), (29, 28), (27, 30)):
        for kind in ("glo", "ghi"):
            b = Builder(200 + ll * 3 + ml)
            b.add(64, 40, off=50)
            for k in range(70):
                b.add(ll, ml, off=int(b.rng.integers(ml, min(900, b.pos))))
            yield Case("len-ll%d-ml%d-%s" % (ll, ml, kind), b.block(kind=kind), S_LONG if max(ll, ml) > 28 else S_LANE)
    # destinations that wrap the ring: (mdst & 4095) + ml + 4 against 4096
    for ml in (8, 20, 28, 60):
        for delta in (-2, -1, 0, 1, 2):
            b = Builder(300 + ml * 7 + delta)
            b.fill(RING * 2 - ml - 4 + delta - 3)
            b.add(3, ml, off=3700)  # the source ends before the batch: the parallel pass copies it
            b.fill(200)
            yield Case("ring-wrap-ml%d-%+d" % (ml, delta), b.block(), S_MATCH_BYTE if delta > 0 else S_LANE if ml <= 28 else S_LONG)
    # ring sources at si 0..8 and around si + ml + 8 == 4096; the batch before is 2048 bytes, the match is lane 0
    for si in range(9):
        b = Builder(400 + si)
        for _ in range(4):
            b.batch(2176)
        b.batch(2048, {0: (0, 20, dict(src=8192 + si))})
        yield Case("ring-src-si%d" % si, b.block(), S_MATCH_BYTE if si < 8 else S_RING_WORD)
    for ml in (20, 60):
        for delta in (-1, 0, 1, 2):
            b = Builder(450 + ml + delta)
            for _ in range(4):
                b.batch(2176)
            b.batch(2048, {0: (0, ml, dict(src=8192 - ml - 8 + delta))})
            yield Case("ring-src-end-ml%d-%+d" % (ml, delta), b.block(), S_MATCH_BYTE if delta > 0 else S_RING_WORD)


def _near_far():
    # sources at near_lo - 1, near_lo, near_lo + 1 with near_lo = O + T - 4064 of the batch that holds the match
    for ml in (20, 100):
        for d in (-1, 0, 1):
            b = Builder(500 + ml + d)
            for _ in range(3):
                b.batch(3200)
            O, T = b.pos, 3200
            b.batch(T, {5: (3, ml, dict(src=O + T - (RING - 32) + d))})
            b.fill(300)
            yield Case("near-lo-ml%d-%+d" % (ml, d), b.block(kind="ghi" if d == 0 else "glo"),
                       S_MATCH_BYTE if d < 0 else S_RING_WORD)
    for off in (511, 512, 513, 4064, 4065, 4095, 4096, 4097):
        for ml in (20, 100):
            b = Builder(600 + off + ml)
            b.fill(9000)
            b.batch(3000, {j: (1 + j % 5, ml, dict(off=off)) for j in range(0, 32, 3)})
            b.fill(500)
            yield Case("off-%d-ml%d" % (off, ml), b.block(kind="glo" if ml == 20 else "ghi"), S_BATCH)


def _batch_heads():
    """lane 0 of every batch: no literals and a match that overlaps itself by 1..4 bytes (off = ml - 1 .. ml - 4), so
    its source ends at the batch's first byte and it goes in the parallel pass; only the byte path may copy it"""
    for kind, size in (("glo", 2000), ("ghi", 1500), ("glo", 1100)):
        b = Builder(650 + size)
        b.batch(size)
        for ml in (8, 12, 20, 28):
            for d in (1, 2, 3, 4):
                b.batch(size, {0: (0, ml, dict(off=ml - d))})
        yield Case("head-overlap-%s-%d" % (kind, size), b.block(kind=kind), S_REPL)


def _partial_batches():
    """the batch's running output crosses RING_LIMIT at lane k; escapes just before, at and after the cut, sources
    just below the batch's first byte; the sequences after it carry escapes as well"""
    for walk in (False, True):
        for k in range(32):
            b = Builder(700 + k + 100 * walk)
            for _ in range(3):
                b.batch(3200)
            O = b.pos
            ghi = k % 4 == 3
            esc_ll = 255 + 10 if ghi else 17
            pre = RING_LIMIT - 100  # output of lanes 0..k-1
            sizes = [pre // k] * k if k else []
            if k:
                sizes[-1] += pre - sum(sizes)
            for j, size in enumerate(sizes):
                ll = esc_ll if j == k - 1 and size > esc_ll + 10 else 1 + j % 3
                b.add(ll, size - ll, src=O - 100 - 11 * j)
            b.add(esc_ll, 400 if k else RING_LIMIT + 100, src=O - 300)  # lane k: crosses the limit (lane 0: a giant)
            b.add(esc_ll, 30, src=O - 40)
            for j in range(40):
                b.add(1 + j % 20, 5 + j % 40, off=int(b.rng.integers(64, 2000)))
            blk = b.block(kind="ghi" if ghi else "glo", extra_pad=_walk_pad() if walk else 0)
            stat = S_GIANT if k == 0 else S_PARTIAL_WALK if walk else S_PARTIAL
            yield Case("partial-lane%d%s" % (k, "-walk" if walk else ""), blk, stat)


def _giants(dict65k):
    for what in ("lit", "match"):
        for off in (1, 7, 31, 32, 64, 4096, 65536):
            b = Builder(800 + off + (what == "lit"))
            b.fill(max(off, 200) + (off % 13) + 5)
            if what == "lit":
                b.add(RING_LIMIT + 100 + off % 7, 10, off=off)
            else:
                b.add(17, RING_LIMIT + 500, off=off)
            b.add(3, 6, off=2)  # lane 1 without escapes
            for o in range(1, 129, 3):
                b.add(o % 17, 5 + o % 23, off=o)
            yield Case("giant-%s-off%d" % (what, off), b.block(kind="ghi" if off == 65536 and what == "lit" else "glo"), S_GIANT)
    for what, src in (("match", -60000), ("match", -500), ("lit-then-dict", -40)):
        b = Builder(900 - src, dict65k)
        if what == "match":
            b.add(5, RING_LIMIT + 700, src=src)
        else:
            b.add(RING_LIMIT + 300, 30, src=src)
        for o in range(1, 129, 5):
            b.add(o % 19, 20 + o % 9, off=o)
        yield Case("giant-dict%d-%s" % (src, what), b.block(), S_GIANT)


def _dependency_tail():
    for kind in ("glo", "ghi"):
        for mode in ("chain", "chain-overlap", "mixed", "mixed-overlap"):
            b = Builder(1000 + len(mode) + (kind == "ghi"))
            b.batch(2500)
            b.batch(2500)
            for j in range(32):
                ll = j % 3
                ml = 12 + j % 20
                if mode.startswith("mixed") and j % 2:
                    b.add(ll, ml, off=int(b.rng.integers(300, 3000)))  # independent
                elif mode.endswith("overlap"):
                    b.add(ll, ml, off=1 + j % 9)  # reads its own output
                else:
                    b.add(ll, ml, off=ll + ml + (j % 4))  # reads the sequence just before
            b.fill(600)
            yield Case("tail-%s-%s" % (mode, kind), b.block(kind=kind), S_TAIL)


def _dictionary(dicts):
    for size, d in dicts.items():
        def mk(tag, seqspecs, stat, seed):
            b = Builder(seed, d)
            for ll, ml, src in seqspecs:
                b.add(ll, ml, off=min(b.pos + ll - src, 65536))  # the largest dictionary: as close as an offset reaches
            b.fill(300, ll=3)
            return Case("dict%d-%s" % (size, tag), b.block(), stat)

        lo = [(1 + k % 4, ml, -size + k) for k in range(10) for ml in (5, 12, 28, 40) if k + ml <= size]
        if lo:
            yield mk("from-start", lo, S_DICT_BYTE, size * 3)
        hi = [(1 + e % 4, ml, -e - ml) for e in range(10) for ml in (5, 12, 28, 40) if e + ml <= size]
        if hi:
            yield mk("from-end", hi, S_DICT_BYTE, size * 3 + 1)
        mid = [(1 + k % 4, ml, -size + 8 + k) for k in range(6) for ml in (5, 20, 28, 100) if 8 + k + ml + 8 <= size]
        if mid:
            yield mk("inside", mid, S_DICT_WORD, size * 3 + 2)
        # straddling the end into the output: the first sequence's literals are the output it reaches
        st = [(12, ml, -min(size, s)) for s in (1, 3, 8) for ml in (6, 20, 40)]
        yield mk("straddle", st, S_DICT_BYTE, size * 3 + 5)
        # off = mdst + dict_size: the dictionary's first byte; one more is out of reach
        if size + 40 < 65536:
            yield mk("first-byte", [(3, 5 + j, -size) for j in range(6)], S_DICT_BYTE, size * 3 + 6)
        else:  # only the first sequence of a block reaches that far back
            for k in (0, 1, 5, 9):
                yield mk("first-byte+%d" % k, [(1, 12, -size + k)], S_DICT_BYTE if k < 8 else S_DICT_WORD, size * 3 + 20 + k)
        b = Builder(size * 3 + 7, d)
        b.add(0, 9, off=size + 1)
        b.fill(100)
        yield Case("dict%d-beyond" % size, b.block(), S_VERDICT)


def _offset_limits():
    b = Builder(1100)
    b.fill(65600, off_hi=4000, ml=200)
    for j in range(20):
        b.add(2, 20 + j, off=65536)
    yield Case("off-65536-glo16", b.block(), S_GLOBAL_WORD)
    b = Builder(1101)
    b.fill(65600, off_hi=4000, ml=200)
    for j in range(20):
        b.add(2, 30 + j, off=65536)
    yield Case("off-65536-ghi", b.block(kind="ghi"), S_GLOBAL_WORD)
    b = Builder(1102)
    b.fill(2000, off_hi=256)
    for j in range(40):
        b.add(1 + j % 3, 5 + j, off=256 - j % 2)
    yield Case("off-256-glo8", b.block(enc_off=1), S_BATCH)


def _varints():
    def one(tag, seqs_fn, stat, **kw):
        b = Builder(1200 + len(tag))
        b.fill(4000)
        seqs_fn(b)
        b.fill(200)
        return Case("varint-" + tag, b.block(**kw), stat)

    yield one("ll-127-128", lambda b: [b.add(15 + v, 10, off=100) for v in (126, 127, 128, 129)], S_LONG)
    yield one("ml-127-128", lambda b: [b.add(3, 20 + v, off=3800) for v in (126, 127, 128, 129)], S_LONG)
    yield one("ml-16383-16384", lambda b: [b.add(3, 20 + v, off=200) for v in (16383, 16384)], S_GIANT)
    yield one("ghi-boundaries", lambda b: [b.add(255 + v, 260 + v, off=333) for v in (0, 1, 127, 128)], S_LONG, kind="ghi")
    yield one("non-minimal", lambda b: [b.add(15 + v % 5, 20 + v, off=90, ll_form=2 + v % 2, ml_form=3 - v % 2)
                                        for v in range(12)], S_LANE)
    yield one("non-minimal-ghi", lambda b: [b.add(255 + v, 260, off=90, ll_form=3, ml_form=2) for v in range(3)], S_LONG,
              kind="ghi")
    b = Builder(1250)
    b.fill(300)
    b.add(3, 20 + (1 << 21) - 1, off=50)  # 2^21 - 1: no block holds it
    yield Case("varint-2^21-1", b.block(cap=BLOCK_CAP), S_GIANT)
    # escapes read past the end of the extras section, as 0: 64 sequences leave no slack padding
    for walk in (False, True):
        b = Builder(1260 + walk)
        b.fill(400)
        for j in range(64):
            last = j >= 56
            b.add(15 if last else 1 + j % 14, 20 if last else 5 + j % 14, off=64 + j,
                  ll_form="omit" if last else None, ml_form="omit" if last else None)
        yield Case("varint-past-end" + ("-walk" if walk else ""), b.block(extra_pad=_walk_pad() if walk else 0), S_LANE)
    # a 0xE0 prefix jams the cursor: it and every later escape read 0
    b = Builder(1270)
    b.fill(400)
    for j in range(50):
        jam = j == 20
        after = j > 20 and j % 3 == 0
        b.add(15 if (jam or after) else 2, 20 if jam else 5 + j % 9, off=70 + j,
              ll_form="jam" if jam else "omit" if after else None, ml_form="omit" if jam else None)
    yield Case("varint-jammed", b.block(), S_LANE)


def _counts():
    for n in (0, 1, 31, 32, 33, 63, 64, 65):
        b = Builder(1300 + n)
        if n:
            b.add(40, 10, off=30)
        for j in range(max(n - 1, 0)):
            b.add(j % 4, 5 + j % 30, off=1 + j % 40)
        yield Case("n-seq-%d" % n, b.block(tail=17), S_BATCH if n else None)
    d = np.random.default_rng(1310).bytes(16)
    b = Builder(1311, d)
    for j in range(40):
        b.add(0, 5 + j % 11, src=-16 + j % 3)
    yield Case("n-lit-0", b.block(tail=0), S_DICT_BYTE)
    b = Builder(1312)
    b.fill(3000)
    yield Case("no-trailing-literals", b.block(tail=0), S_BATCH)


def _rle():
    plans = {
        "rep4-raw1": [("rep", 4), ("raw", 1)] * 40,
        "rep131-raw128": [("rep", 131), ("raw", 128)] * 6,
        "rep131": [("rep", 131)] * 8,
        "raw1": [("raw", 1)] * 200,
    }
    for name, plan in plans.items():
        rng = np.random.default_rng(len(name))
        lits = bytearray()
        for kind, n in plan:
            if kind == "rep":
                lits += bytes([int(rng.integers(0, 256))]) * n
            else:
                v = rng.integers(0, 256, n).astype(np.uint8)
                v[1:][v[1:] == v[:-1]] ^= 0x55  # no accidental runs
                lits += v.tobytes()
        for enc_off in (0, 1):
            b = Builder(1400 + len(name) + enc_off)
            seqs, p, pos = [], 0, 0
            while p < len(lits) - 40:
                n = int(b.rng.integers(1, 40))
                seqs.append(Seq(lits[p:p + n], 5 + n % 13, 1 + (pos + n) % min(pos + n, 200) if pos + n > 1 else 1))
                pos += n + seqs[-1].ml
                p += n
            blk = Block(seqs, lits[p:], enc_lit=1, enc_off=enc_off, rle_plan=plan)
            yield Case("rle-%s-off%d" % (name, 8 if enc_off else 16), blk, S_BATCH)


def _verdicts():
    def mk(tag, fn, stat, **kw):
        b = Builder(1500 + len(tag))
        fn(b)
        return Case("verdict-" + tag, b.block(**kw), stat)

    def bad_at(lane, batch=0):
        def f(b):
            for _ in range(batch):
                b.batch(2000)
            b.batch(2000, {lane: (3, 10, dict(off=b.pos + 3 + 10 + 40 * lane + 5000))})
        return f

    for lane, batch in ((0, 1), (31, 0), (0, 2), (17, 1)):
        yield mk("bad-offset-lane%d-batch%d" % (lane, batch), bad_at(lane, batch), S_VERDICT)

    b = Builder(1550)
    b.batch(2000)
    start = b.pos
    b.batch(2000)
    yield Case("verdict-overflow-batch1-lane31", b.block(tail=0, cap=start + 2000 - 1), S_VERDICT)
    # overflow and bad offset in one sequence: overflow wins
    b = Builder(1560)
    b.fill(500)
    b.add(10, 100, off=650)
    yield Case("verdict-overflow-beats-bad-offset", b.block(tail=0, cap=560), S_VERDICT)
    # a literal run past the declared literal count
    b = Builder(1561)
    b.fill(600)
    for j in range(10):
        b.add(9, 8, off=33)
    yield Case("verdict-literals-past-n-lit", b.block(tail=0, n_lit=sum(len(s.lit) for s in b.seqs) - 5), S_VERDICT)
    # dst_cap one byte short of the output (trailing literals do not fit)
    b = Builder(1562)
    b.fill(3000)
    blk = b.block(tail=20)
    yield Case("verdict-cap-one-short", Block(blk.seqs, blk.tail, cap=blk.cap - 1), S_BATCH)
    # inside a partial batch: the crossing lane has a bad offset (the next round fails at its lane 0)
    b = Builder(1563)
    b.batch(3200)
    b.batch(3300, n=20)
    b.add(2, 500, off=b.pos + 2 + 10)
    b.fill(300)
    yield Case("verdict-partial-batch", b.block(), S_PARTIAL)
    # on the giant path: bad offset, and a giant that overflows the output
    b = Builder(1564)
    b.fill(300)
    b.add(2, RING_LIMIT + 50, off=b.pos + 2 + 1)
    yield Case("verdict-giant-bad-offset", b.block(), S_GIANT)
    b = Builder(1565)
    b.fill(300)
    b.add(2, RING_LIMIT + 50, off=40)
    blk = b.block(tail=0)
    yield Case("verdict-giant-overflow", Block(blk.seqs, b"", cap=blk.cap - 1), S_GIANT)
    b = Builder(1566)
    b.fill(300)
    b.add(RING_LIMIT + 50, 10, off=40)
    blk = b.block(tail=0)
    yield Case("verdict-giant-literals-past-n-lit", Block(blk.seqs, b"", n_lit=len(b"".join(s.lit for s in blk.seqs)) - 1),
               S_GIANT)


def _dicts():
    rng = np.random.default_rng(77)
    return {s: rng.bytes(s) for s in (1, 5, 7, 8, 9, 16, 4096, 65535)}


_CAT = None


def catalogue():
    global _CAT
    if _CAT is None:
        dicts = _dicts()
        cases = []
        for gen in (_short_offsets(), _thresholds(), _near_far(), _batch_heads(), _partial_batches(), _giants(dicts[65535]),
                    _dependency_tail(), _dictionary(dicts), _offset_limits(), _varints(), _counts(), _rle(), _verdicts()):
            cases += [c for c in gen if c is not None]
        names = [c.name for c in cases]
        assert len(set(names)) == len(names), "case names are unique"
        _CAT = cases
    return _CAT


CASES = catalogue()
IDS = [c.name for c in CASES]


def _same_verdict(got, want):
    return ROOM.get(got, got) == ROOM.get(want, want)


def _oracle_block(orc, blk, raw=None, verify=0):
    raw = blk.raw if raw is None else raw
    out = np.zeros(max(blk.cap, 1), np.uint8)
    d = blk.dict_bytes
    r = orc.lib.zxo_decode_block(raw, len(raw), out.ctypes.data, blk.cap, d if d else None, len(d), None, verify)
    return r, out[:max(r, 0)]


def _expect(st, out, blk, what):
    """status and bytes of one decoded block against the generator's"""
    if blk.status >= 0:
        assert st == blk.status, (what, z.ERR.get(st, st))
        assert out[:st].tobytes() == blk.want, (what, "first wrong byte at %d" % int(np.argmax(out[:st] != np.frombuffer(blk.want, np.uint8))))
    else:
        assert _same_verdict(st, blk.status), (what, z.ERR.get(st, st), z.ERR.get(blk.status))


def _emu(blocks, units=0, seed=1, src_res=0, dst_res=0, lean=None, dict_bytes=None):
    """decode `blocks` as one job table on the emulator: (status list, output bytes, per-job slices, stray stores)"""
    src, rows, total = bg.job_table(blocks, src_res, dst_res)
    jobs = (zs.Job * len(rows))(*[zs.Job(*r) for r in rows])
    out = np.zeros(max(total, 1), np.uint8)
    status = (C.c_int32 * len(rows))()
    oob = C.c_int(0)
    s = np.frombuffer(src, np.uint8)
    d = blocks[0].dict_bytes if dict_bytes is None else dict_bytes
    dp = np.frombuffer(d, np.uint8).ctypes.data if d else None
    if lean is None:
        zs.lib().simt_decode_blocks(s.ctypes.data, s.size, out.ctypes.data, total, jobs, len(rows), status, dp, len(d),
                                    None, BLOCK_CAP, 0, units, seed, C.byref(oob))
    else:
        lean.simt_decode_two_stage(s.ctypes.data, s.size, out.ctypes.data, total, jobs, len(rows), status, dp, len(d),
                                   None, BLOCK_CAP, seed, C.byref(oob))
    return list(status), out, [(r[1], r[3]) for r in rows], oob.value


def _stats(lib):
    return (C.c_uint64 * 32).in_dll(lib, "simt_stat")


def test_catalogue_covers_every_family():
    fams = {}
    for c in CASES:
        fams.setdefault(c.name.split("-")[0], []).append(c)
    assert len(CASES) >= 100
    assert set(fams) >= {"short", "len", "ring", "near", "off", "head", "partial", "giant", "tail", "dict1", "dict5", "dict7",
                         "dict8", "dict9", "dict16", "dict4096", "dict65535", "varint", "n", "rle", "verdict"}, set(fams)
    assert sum(c.block.status < 0 for c in CASES) >= 15


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_generator_agrees_with_oracle(orc, case):
    """the generator's byte loop and the oracle's block decoder: same verdict, same bytes"""
    r, out = _oracle_block(orc, case.block)
    _expect(r, out, case.block, "oracle")
    r, out = _oracle_block(orc, case.block, raw=bg.block_bytes(case.block.raw[0], case.block.payload, True), verify=1)
    _expect(r, out, case.block, "oracle, checksum verified")


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_emulator_sequence_body(case):
    """the production body under three lane schedules at a 16-byte residue of its own; the targeted path is taken"""
    k = IDS.index(case.name)
    lib = zs.lib()
    stat = _stats(lib)
    for seed in (0, 1 + k, 1000 + k):
        C.memset(stat, 0, C.sizeof(stat))
        st, out, spans, oob = _emu([case.block], units=0, seed=seed, src_res=k % 16, dst_res=(7 * k + seed) % 16)
        assert oob == 0, "stores outside the destination"
        _expect(st[0], out[spans[0][0]:], case.block, "emulator seed %d" % seed)
        if case.stat is None:
            assert stat[S_BATCH] == 0
        else:
            assert stat[case.stat] > 0, ("targeted path not taken", case.stat, list(stat))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_emulator_unit_walk_and_lean_route(case, lean_emu):
    """the output-centric body, and the two-launch route (lean instance, then the general one for what it defers)"""
    k = IDS.index(case.name)
    st, out, spans, oob = _emu([case.block], units=1, seed=5 + k, src_res=(k + 3) % 16, dst_res=(k + 9) % 16)
    assert oob == 0
    _expect(st[0], out[spans[0][0]:], case.block, "unit walk")
    st, out, spans, oob = _emu([case.block], seed=9 + k, src_res=(k + 5) % 16, dst_res=(3 * k) % 16, lean=lean_emu)
    assert oob == 0
    _expect(st[0], out[spans[0][0]:], case.block, "lean route")


def test_emulator_whole_catalogue_in_one_table():
    """every case without a dictionary as one job table: neighbouring jobs share the source and destination buffers"""
    blocks = [c.block for c in CASES if not c.block.dict_bytes]
    st, out, spans, oob = _emu(blocks, seed=77, src_res=3, dst_res=11)
    assert oob == 0
    for s, (d0, cap), blk in zip(st, spans, blocks):
        _expect(s, out[d0:d0 + cap], blk, "table")


_GUARD_CHILD = r"""
import sys
sys.path.insert(0, %r)
import numpy as np
import test_blockgen_decode as t
import zxc_simt as zs
lib = zs.lib()
n = 0
for mode in (1, 2):
    lib.simt_guard_pages(mode)
    for c in t.CASES:
        if not c.block.dict_bytes and not c.name.startswith(("giant", "off-65536", "verdict")):
            continue
        for src_res, dst_res in ((0, 0), (5, 13)):
            st, out, spans, oob = t._emu([c.block], seed=3, src_res=src_res, dst_res=dst_res)
            assert oob == 0, c.name
            t._expect(st[0], out[spans[0][0]:], c.block, c.name)
            n += 1
print("guard ok", n)
"""


def test_emulator_loads_stay_inside_the_buffers():
    """The dictionary, giant, far-offset and verdict cases with the source, destination and dictionary (dictionary_size
    + 128 bytes, as the product allocates it) placed against PROT_NONE pages, flush with either end: a load outside
    the kernel's documented reach ends the child process with the faulting buffer+offset."""
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _GUARD_CHILD % here], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "guard ok" in r.stdout, (r.returncode, r.stdout[-1500:], r.stderr[-1500:])


# ------------------------------------------------------------------------------------------------------------------
# the compiled sm_90a kernels
# ------------------------------------------------------------------------------------------------------------------
class _Signed:
    """a block as it sits in a frame with checksums: the payload's checksum behind it"""

    def __init__(self, blk):
        self.raw, self.cap = bg.block_bytes(blk.raw[0], blk.payload, True), blk.cap


def _groups():
    """cases by dictionary: one launch each"""
    g = {}
    for c in CASES:
        g.setdefault(c.block.dict_bytes, []).append(c.block)
    return g


def _gpu_table(prod, blocks, dict_bytes, verify, src_res, dst_res):
    import torch
    lib = prod.lib
    lib.zxc_b200_decode_scratch_size.restype = C.c_size_t
    lib.zxc_b200_decode_scratch_size.argtypes = [C.c_uint32]
    lib.zxc_b200_decode_blocks.restype = C.c_int
    lib.zxc_b200_decode_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                           C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_int, C.c_void_p]
    src, rows, total = bg.job_table([_Signed(b) for b in blocks] if verify else blocks, src_res, dst_res)
    dev = torch.device("cuda", 0)
    table = (zs.Job * len(rows))(*[zs.Job(*r) for r in rows])
    d_src = torch.from_numpy(np.frombuffer(src, np.uint8).copy()).to(dev)
    d_dst = torch.zeros(total, dtype=torch.uint8, device=dev)
    d_jobs = torch.from_numpy(np.frombuffer(bytes(table), np.uint8).copy()).to(dev)
    d_status = torch.zeros(len(rows), dtype=torch.int32, device=dev)
    d_dict = torch.from_numpy(np.frombuffer(dict_bytes + bytes(128), np.uint8).copy()).to(dev) if dict_bytes else None
    ss = lib.zxc_b200_decode_scratch_size(BLOCK_CAP)
    d_scratch = torch.empty(ss, dtype=torch.uint8, device=dev)
    rc = lib.zxc_b200_decode_blocks(d_src.data_ptr(), d_dst.data_ptr(), d_jobs.data_ptr(), len(rows), d_status.data_ptr(),
                                    d_dict.data_ptr() if d_dict is not None else None, len(dict_bytes), None,
                                    d_scratch.data_ptr(), ss, BLOCK_CAP, verify, torch.cuda.current_stream(dev).cuda_stream)
    assert rc == 0, z.ERR.get(rc, rc)
    torch.cuda.synchronize(dev)
    return list(d_status.cpu().numpy()), d_dst.cpu().numpy(), [(r[1], r[3]) for r in rows]


@pytest.mark.gpu
@pytest.mark.parametrize("verify", [0, 1], ids=["lean-then-general", "general-verified"])
def test_gpu_job_tables_at_every_residue(prod, verify):
    """every case through zxc_b200_decode_blocks, one launch per dictionary, at source and destination offsets of every
    residue mod 16; without verification the lean instance runs first, with it the general instance alone on blocks
    that carry checksums.  The cases without a dictionary run once more with a 4096-byte dictionary present."""
    groups = _groups()
    d4k = _dicts()[4096]
    launches = 0
    for dict_bytes, blocks in list(groups.items()) + [(d4k, [b for b in groups[b""] if b.status >= 0])]:
        for r in range(16):
            st, out, spans = _gpu_table(prod, blocks, dict_bytes, verify, r, (5 * r + 3) % 16)
            for s, (d0, cap), blk in zip(st, spans, blocks):
                _expect(int(s), out[d0:d0 + cap], blk, ("residue", r, len(dict_bytes)))
            launches += 1
    assert launches == 16 * (len(groups) + 1)


def _frame_of(blk, checksum):
    block_size = max(4096, 1 << (blk.cap - 1).bit_length())
    did = _oracle_lib().dict_id(blk.dict_bytes) if blk.dict_bytes else 0
    total = blk.status if blk.status >= 0 else blk.cap
    return bg.frame([(blk.payload, blk.raw[0])], block_size, checksum=checksum, dict_id=did, total=total), total


def _oracle_lib():
    return bg._oracle()


@pytest.mark.gpu
@pytest.mark.parametrize("checksum", [0, 1])
def test_gpu_frames_and_block_api(prod, orc, libs, checksum):
    """every case as a one-block frame through zxc_decompress, judged by the oracle's frame decoder (and the reference
    library where it is built), and as a bare block through zxc_decompress_block"""
    ref = libs[2]
    dctx = prod.lib.zxc_create_dctx()
    try:
        for c in CASES:
            blk = c.block
            d = blk.dict_bytes or None
            fr, total = _frame_of(blk, checksum)
            r0, o0 = orc.decompress(fr, total, checksum=checksum, dict=d)
            if blk.status >= 0:
                assert r0 == blk.status and o0.tobytes() == blk.want, (c.name, r0)
            r1, o1 = prod.decompress(fr, total, checksum=checksum, dict=d)
            assert _same_verdict(r1, r0), (c.name, z.ERR.get(r1, r1), z.ERR.get(r0, r0))
            if r0 >= 0:
                assert np.array_equal(o1, o0), c.name
            if ref is not None:
                r2, o2 = ref.decompress(fr, total, checksum=checksum, dict=d)
                assert _same_verdict(r2, r0) and (r0 < 0 or np.array_equal(o2, o0)), (c.name, r2, r0)
            raw = _Signed(blk).raw if checksum else blk.raw
            out = np.zeros(blk.cap, np.uint8)
            o = z.DecompressOpts(checksum_enabled=checksum)
            keep = np.frombuffer(blk.dict_bytes, np.uint8) if d else None
            if d:
                o.dict, o.dict_size = keep.ctypes.data, keep.size
            r3 = prod.lib.zxc_decompress_block(dctx, raw, len(raw), out.ctypes.data, blk.cap, C.byref(o))
            _expect(int(r3), out, blk, (c.name, "zxc_decompress_block"))
    finally:
        prod.lib.zxc_free_dctx(dctx)


_ALT_CHILD = r"""
import sys
sys.path.insert(0, %r)
import numpy as np
import test_blockgen_decode as t
import zxc_ctypes as z
prod, orc = z.ZxcLib(z.PRODUCT_SO), z.Oracle()
n = 0
for c in t.CASES:
    blk = c.block
    d = blk.dict_bytes or None
    for cks in (0, 1):
        fr, total = t._frame_of(blk, cks)
        r0, o0 = orc.decompress(fr, total, checksum=cks, dict=d)
        r1, o1 = prod.decompress(fr, total, checksum=cks, dict=d)
        assert t._same_verdict(r1, r0) and (r0 < 0 or np.array_equal(o1, o0)), (c.name, cks, r0, r1)
        n += 1
print("alt ok", n)
"""


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{"ZXC_B200_UNITS": "1"}], ids=["unit-walk-forced"])
def test_gpu_alternative_bodies_on_the_catalogue(env):
    """the output-centric body, selected per process by an environment variable"""
    e = dict(os.environ)
    e.update(env)
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _ALT_CHILD % here], env=e, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "alt ok" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
