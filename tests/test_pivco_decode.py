"""The PivCo Huffman section decoder (pivco_decode, zxc_b200/csrc/zxc_huffman.cuh) on synthetic code tables and runs.

Reference-encoded frames only ever carry the tables the level 6-7 package-merge happens to build.  Here
tests/zxc_blockgen.py writes the sections from chosen code lengths and symbol strings (or takes malformed tables and
runs as they are) into GLO blocks: Huffman literals (enc_lit = 2), literals under the dictionary's table (enc_lit = 3)
and Huffman tokens (enc_tok = 2), combined with raw, RLE or Huffman literals, 8/16-bit offsets, escapes and dictionary
sources.  The catalogue reaches the decoder's trouble spots: flat roots of every depth at every level, the
single-symbol code, rank words at 32-bit boundaries and the last word's padding, zero-count subtrees, the run-area
bounds, the reads at the end of the last run, and the section checks around the decoder (the token limit of
block_size / 5 + 16, empty token sections, lit_comp / tok_comp bounds).

Each case must agree with the generator's own tree-walking decoder, the oracle's block decoder and the unmodified
reference library, which decides every verdict; then with the kernel on the CPU warp emulator (general instance under
three lane schedules, the two-launch lean route, guard pages) and on the GPU (zxc_b200_decode_blocks, zxc_decompress,
zxc_decompress_block, the unit-walk body).  On the emulator each case also asserts that the
decoder path it targets was taken (ZXC_STAT counters of tests/simt)."""
import ctypes as C
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

import zxc_blockgen as bg
import zxc_ctypes as z
import zxc_simt as zs
from zxc_blockgen import Block, Huf, Seq
from zxc_simt import lean_emu  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFI_SO = os.path.join(ROOT, "oracle", "_ref", "libzxc_ref_internals.so")
ROOM = {-2: -10}  # DST_TOO_SMALL where a frame driver reports what the kernel calls OVERFLOW

# ZXC_STAT counters of zxc_huffman.cuh in the emulator build
S_SINGLE, S_BITMAP, S_RANK, S_VERDICT, S_FLAT = 32, 33, 34, 35, 40  # S_FLAT + D: symbols read from a depth-D flat root


class Case:
    """`stat`: the counter that must be non-zero on the emulator, or None for a verdict raised before the decoder runs
    (then the decoder's counters must stay zero).  `emu`: small enough for the emulator."""

    def __init__(self, name, block, stat, emu=True, frame_status=None):
        self.name, self.block, self.stat, self.emu = name, block, stat, emu
        self.frame_status = frame_status  # the verdict of a frame when the frame decides it before the block

    def __repr__(self):
        return self.name


# ------------------------------------------------------------------------------------------------------------------
# code tables
# ------------------------------------------------------------------------------------------------------------------
def lens_of(counts, rng, syms=None):
    """256 code lengths with counts[l] symbols of length l, the symbols drawn at random (or `syms` in order)"""
    syms = list(rng.permutation(256)) if syms is None else list(syms)
    lens, k = [0] * 256, 0
    for l, c in sorted(counts.items()):
        for _ in range(c):
            lens[int(syms[k])] = l
            k += 1
    return lens


def chain(L, rng):
    """lengths 1, 2, ..., L - 1, L, L: a leaf pair at the bottom, one leaf beside every internal node above"""
    c = {l: 1 for l in range(1, L)}
    c[L] = c.get(L, 0) + 2 if L > 1 else 2
    return lens_of(c, rng)


def flat_at(D, p, rng, beside="leaf"):
    """a flat root of depth D at depth p: a chain of leaves down to it (beside = "leaf"), or a bitmap subtree beside it
    (beside = "bitmap": its sibling holds a leaf at p + 1 and two at p + 2)"""
    if p == 0:
        return lens_of({D: 1 << D}, rng)
    if beside == "leaf":
        c = {l: 1 for l in range(1, p + 1)}
    else:
        c = {l: 1 for l in range(1, p)}
        c[p + 1] = c.get(p + 1, 0) + 1
        c[p + 2] = c.get(p + 2, 0) + 2
    c[p + D] = c.get(p + D, 0) + (1 << D)
    return lens_of(c, rng)


def random_code(maxlen, n_sym, rng):
    """a Kraft-complete code of n_sym symbols and maximum length `maxlen`, by random leaf splits"""
    while True:
        leaves = [0]
        while len(leaves) < n_sym:
            cand = [i for i, d in enumerate(leaves) if d < maxlen]
            i = cand[int(rng.integers(len(cand)))]
            d = leaves.pop(i)
            leaves += [d + 1, d + 1]
        if max(leaves) == maxlen:
            syms = rng.permutation(256)[:n_sym]
            lens = [0] * 256
            for s, d in zip(syms, leaves):
                lens[int(s)] = d
            return lens


def one_symbol(s, L=1):
    lens = [0] * 256
    lens[s] = L
    return lens


def stream(lens, n, rng, how="uniform", pick=None):
    """n symbols out of the code's symbols: uniform, skewed (geometric over the symbols), alternating between two,
    or one symbol `pick` only"""
    present = np.array([s for s in range(256) if lens[s]], np.uint8)
    if how == "one":
        return bytes([pick if pick is not None else int(present[-1])]) * n
    if how == "alt":
        return bytes(present[np.arange(n) % min(2, present.size)])
    if how == "skew":
        w = 0.6 ** np.arange(present.size)
        return bytes(rng.choice(present, n, p=w / w.sum()))
    return bytes(rng.choice(present, n))


# ------------------------------------------------------------------------------------------------------------------
# blocks
# ------------------------------------------------------------------------------------------------------------------
def lit_block(lits, huf, rng, enc_lit=2, n_seq=3, **kw):
    """Huffman literals `lits` (all of them trailing literals after n_seq sequences that copy from the dictionary or
    the output so far, so that every literal is used)"""
    lits = bytes(lits)
    seqs = []
    if n_seq and len(lits) > 16:
        cut = sorted(rng.choice(np.arange(8, len(lits)), min(n_seq, len(lits) - 8), replace=False).tolist())
        prev = 0
        for c in cut:
            seqs.append(Seq(lits[prev:c], 5 + c % 11, 1 + c % max(1, min(c, 250))))
            prev = c
        tail = lits[prev:]
    else:
        tail = lits
    return Block(seqs, tail, enc_lit=enc_lit, lit_huf=huf, **kw)


def tok_lens(seqs, rng, how="chain"):
    """a code for the tokens of `seqs`: every token value present, the rest by `how`"""
    toks = sorted({(min(len(s.lit), 15) << 4) | min(s.ml - bg.MIN_MATCH, 15) for s in seqs})
    n = len(toks)
    if n == 1:
        lens = [0] * 256
        lens[toks[0]] = 1
        return lens
    # Kraft-complete over exactly these symbols
    if how == "chain" and n <= 12:
        c = {l: 1 for l in range(1, n - 1)}
        c[n - 1] = c.get(n - 1, 0) + 2
    else:
        L = max(1, (n - 1).bit_length())
        short = (1 << L) - n  # symbols one level up
        c = {L - 1: short, L: n - short} if short else {L: n}
    return lens_of(c, rng, syms=list(rng.permutation(toks)))


def tok_block(seqs, tail, rng, tok_how="chain", enc_lit=0, lit_huf=None, **kw):
    return Block(seqs, tail, tok_huf=Huf(tok_lens(seqs, rng, tok_how)), enc_lit=enc_lit, lit_huf=lit_huf, **kw)


def target(blk):
    """the counter the block's sections are sure to move: the deepest flat root any symbol reaches, else the
    single-symbol path, else the rank-word fill"""
    flats, single = [], False
    for lens, syms in blk.decoded:
        if bg.PivcoTree(lens).single:
            single = True
            continue
        sizes = []
        bg.pivco_runs(lens, syms, sizes)
        flats += [k for _, k, c, _ in sizes if k != "bitmap" and c]
    return S_FLAT + max(flats) if flats else S_SINGLE if single else S_RANK


def _tables(rng):
    """(name, lengths, stat-if-fixed)"""
    out = []
    for L in range(1, 12):
        out.append(("chain%d" % L, chain(L, rng)))
        if L >= 2:
            out.append(("random-max%d" % L, random_code(L, min(1 << L, 3 + 23 * L) if L > 1 else 2, rng)))
    for s in (0, 1, 254, 255):
        out.append(("single%d" % s, one_symbol(s)))
    out.append(("two", lens_of({1: 2}, rng)))
    out.append(("all256-len8", [8] * 256))
    for D in range(2, 9):
        for p in range(0, 12 - D):
            if p + (1 << D) > 256 or (p and p + 2 + (1 << D) > 256):
                continue
            out.append(("flat-d%d-at%d" % (D, p), flat_at(D, p, rng)))
            if p >= 1 and p + 1 + (1 << D) <= 256 and p + D <= 11:
                out.append(("flat-d%d-at%d-by-bitmap" % (D, p), flat_at(D, p, rng, "bitmap")))
    out.append(("mixed256", random_code(11, 256, rng)))
    return out


def _table_cases():
    rng = np.random.default_rng(2026)
    for name, lens in _tables(rng):
        t = bg.PivcoTree(lens)
        assert t.error is None, name
        if name.startswith("flat-d"):
            D, p = int(name.split("-")[1][1:]), int(name.split("-")[2][2:])
            assert any(t.kind[n] == D and n[0] == p for n in t.emitting()), (name, t.flat_depths())
        n = 700 + len(name) * 13  # counts that are not a multiple of 8 or 32
        how = ("uniform", "skew", "alt")[len(name) % 3]
        lits = stream(lens, n, rng, how)
        yield Case("lit-%s-%s" % (name, how), lit_block(lits, Huf(lens), rng, enc_off=len(name) % 2), None)
    # a single symbol out of a wide table: zero counts and zero-length runs everywhere else
    for name, lens in (("chain11", chain(11, rng)), ("mixed256", random_code(11, 256, rng)), ("flat-d3-at5", flat_at(3, 5, rng))):
        deepest = max(range(256), key=lambda s: (lens[s], s))
        shallow = min((s for s in range(256) if lens[s]), key=lambda s: (lens[s], s))
        for tag, s in (("deepest", deepest), ("shallowest", shallow)):
            yield Case("lit-%s-only-%s" % (name, tag), lit_block(stream(lens, 300, rng, "one", s), Huf(lens), rng), None)


def _count_cases():
    rng = np.random.default_rng(7)
    c11 = chain(11, rng)
    two = lens_of({1: 2}, rng)
    f3 = flat_at(3, 2, rng)
    for n in (1, 7, 8, 9, 31, 32, 33, 63, 64, 65, 255, 256, 257):
        yield Case("count-%d-chain11" % n, lit_block(stream(c11, n, rng, "skew"), Huf(c11), rng, n_seq=0), None)
        yield Case("count-%d-flat3" % n, lit_block(stream(f3, n, rng), Huf(f3), rng, n_seq=0), None)
    # the depth-1 internal node of a two-leaf-then-chain table sees k*32 +- 1 symbols; the root sees more
    c4 = chain(4, rng)
    right = [s for s in range(256) if c4[s] > 1]
    left = [s for s in range(256) if c4[s] == 1][0]
    for k in (1, 2, 5):
        for d in (-1, 0, 1):
            m = 32 * k + d
            syms = np.array([left] * 45 + list(rng.choice(right, m)), np.uint8)
            rng.shuffle(syms)
            yield Case("count-node-%d" % m, lit_block(bytes(syms), Huf(c4), rng, n_seq=0), None)
    # the last flat path straddles a byte: c * D not a multiple of 8
    for D in (3, 5, 6, 7):
        fl = flat_at(D, 0, rng)
        for n in (1, 3, 5, 9, 13):
            yield Case("count-flat%d-%d" % (D, n), lit_block(stream(fl, n, rng), Huf(fl), rng, n_seq=0), None)
    # up to the block size
    for bs, n, lens, emu in ((4096, 4096, [8] * 256, True), (65536, 65536, c11, True), (1 << 21, 1 << 21, two, False)):
        yield Case("count-lit-%d" % n, lit_block(stream(lens, n, rng, "skew"), Huf(lens), rng, n_seq=0, block_size=bs), None,
                   emu=emu)


def _token_cases(dict_bytes, dict_lens):
    rng = np.random.default_rng(11)

    def seqs_for(n, short=False, esc=False, dict_src=False):
        out, pos = [], 0
        for j in range(n):
            ll = (15 + j % 40) if esc and j % 3 == 0 else j % 6
            ml = (20 + j % 300) if esc and j % 4 == 1 else 5 + j % 9
            lit = rng.bytes(ll)
            room = pos + ll
            if dict_src and j % 2 == 0:
                off = min(room + 1 + j % len(dict_bytes), room + len(dict_bytes))
            elif short:
                off = 1 + j % 8 if room else 1
                off = min(off, room) if room else 1
            else:
                off = 1 + int(rng.integers(0, max(1, min(room, 255))))
            if not dict_src and room == 0:
                lit, ll, room = rng.bytes(8), 8, pos + 8
                off = min(off, room)
            out.append(Seq(lit, ml, off))
            pos = room + ml
        return out

    for n in (1, 7, 8, 9, 31, 32, 33, 63, 64, 65, 255, 256, 257):
        s = seqs_for(n)
        yield Case("tok-n%d-raw-lits" % n, tok_block(s, rng.bytes(9), rng, enc_off=n % 2), None)
    s = seqs_for(120, short=True)
    yield Case("tok-short-offsets-off8", tok_block(s, b"", rng, enc_off=1), None)
    s = seqs_for(90, esc=True)
    yield Case("tok-escapes", tok_block(s, rng.bytes(3), rng, tok_how="wide"), None)
    s = seqs_for(70, dict_src=True)
    yield Case("tok-dict-sources", tok_block(s, b"", rng, dict_bytes=dict_bytes), None)
    # with RLE and Huffman literals
    s = [Seq(bytes([65 + j % 3]) * (4 + j % 20), 5 + j % 7, 1 + j % 4) for j in range(60)]
    yield Case("tok-rle-lits", tok_block(s, b"x" * 30, rng, enc_lit=1), None)
    ll = chain(9, rng)
    s = [Seq(stream(ll, 1 + j % 30, rng, "skew"), 5 + j % 12, 1 + j % 16) for j in range(80)]
    yield Case("tok-huf-lits", tok_block(s, stream(ll, 5, rng), rng, enc_lit=2, lit_huf=Huf(ll)), None)
    s = [Seq(stream(dict_lens, 1 + j % 30, rng), 5 + j % 12, 1 + j % 16) for j in range(80)]
    yield Case("tok-dict-table-lits", tok_block(s, b"", rng, enc_lit=3, lit_huf=Huf(dict_lens), dict_bytes=dict_bytes,
                                                dict_huf=bg.pack_lengths(dict_lens)), None)
    # a single token value: the single-symbol code
    s = [Seq(b"ab", 7, 2) for _ in range(40)]
    yield Case("tok-single-symbol", tok_block(s, b"", rng), None)
    # the end of the last run 1..3 bytes before the payload end: only the 8-bit offsets follow the token section
    for n in (1, 2, 3):
        s = [Seq(rng.bytes(3 + j), 6 + j, 2) for j in range(n)]
        yield Case("tok-runs-end-%d-before-payload-end" % n, tok_block(s, b"", rng, tok_how="wide", enc_off=1), None)
    for n in (1, 2, 3):  # ... with a flat root last in the run area
        s = [Seq(rng.bytes(4), 5 + j % 4, 4) for j in range(4 * n)]
        blk = Block(s, b"", enc_off=1, tok_huf=Huf(lens_of({2: 4}, rng, syms=sorted({(4 << 4) | j for j in range(4)}))))
        yield Case("tok-flat-runs-end-%d" % n, blk, None)


def _block_size_cases():
    """n_lit and n_seq at the block-size limits"""
    rng = np.random.default_rng(13)
    two = lens_of({1: 2}, rng)
    for n in (4095, 4096, 4097):
        yield Case("n-lit-bs4096%+d" % (n - 4096), lit_block(stream(two, n, rng), Huf(two), rng, n_seq=0, block_size=4096,
                                                              cap=n + 64), None)
    for bs in (4096, 65536, 1 << 21):
        lim = bs // 5 + 16
        for d in (0, 1):
            n = lim + d
            s = [Seq(b"", 5, 1) for _ in range(n)]
            s[0] = Seq(b"Q", 5, 1)
            blk = tok_block(s, b"", rng, block_size=bs)
            yield Case("n-seq-bs%d-limit%+d" % (bs, d), blk, None, emu=bs <= 65536 or d == 1)


def _verdict_cases(dict_bytes, dict_lens):
    rng = np.random.default_rng(17)
    c11 = chain(11, rng)
    lits = stream(c11, 500, rng, "skew")

    def lb(tag, huf, lits=lits, **kw):
        return Case("verdict-" + tag, lit_block(lits, huf, rng, n_seq=0, **kw), None)

    for nib in range(12, 16):
        for half in (0, 1):
            tab = bytearray(bg.pack_lengths(c11))
            tab[40] = (tab[40] & (0xF0 if half == 0 else 0x0F)) | (nib << (4 * half))
            yield lb("nibble%d-%s" % (nib, "low" if half == 0 else "high"), Huf(c11, table=bytes(tab), runs=bg.pivco_runs(c11, lits)))
    # Kraft one length-11 unit over / under: one more symbol at 11, or one of the pair at 11 dropped
    over = list(c11)
    over[next(s for s in range(256) if not c11[s])] = 11
    under = list(c11)
    under[max(range(256), key=lambda s: (c11[s], s))] = 0
    for tag, bad in (("kraft-over", over), ("kraft-under", under)):
        yield lb(tag, Huf(c11, table=bg.pack_lengths(bad), runs=bg.pivco_runs(c11, lits)))
    yield lb("no-symbols", Huf(c11, table=bytes(128), runs=bg.pivco_runs(c11, lits)))
    for L in (2, 3, 11):
        yield lb("lone-symbol-length%d" % L, Huf(one_symbol(9), table=bg.pack_lengths(one_symbol(9, L)), runs=bytes(100)),
                 lits=b"\x09" * 500)
    # the run area one byte short at the first, a middle, the last and a flat node
    f5 = flat_at(3, 5, rng)
    l5 = stream(f5, 600, rng)
    for tag, lens, ll in (("chain11", c11, lits), ("flat3", f5, l5)):
        sizes = []
        runs = bg.pivco_runs(lens, ll, sizes)
        ends = np.cumsum([sz for *_, sz in sizes])
        picks = {"first": 0, "middle": len(sizes) // 2, "last": len(sizes) - 1}
        flats = [i for i, (_, k, c, sz) in enumerate(sizes) if k != "bitmap" and sz]
        if flats:
            picks["flat"] = flats[0]
        for where, i in picks.items():
            if sizes[i][3] == 0:
                continue
            yield lb("%s-runs-short-at-%s" % (tag, where), Huf(lens, runs=runs[:int(ends[i]) - 1]), lits=ll)
    # single-symbol runs: a set bit inside n is rejected, set padding bits beyond n are not
    for n in (1, 7, 9, 33):
        for bit in sorted({0, n - 1}):
            r = bytearray((n + 7) // 8)
            r[bit >> 3] |= 1 << (bit & 7)
            yield lb("single-bit%d-of-%d" % (bit, n), Huf(one_symbol(200), runs=bytes(r)), lits=b"\xc8" * n)
        if n % 8:
            r = bytearray((n + 7) // 8)
            r[-1] = 0xFF & ~((1 << (n % 8)) - 1)
            yield Case("pad-single-%d" % n, lit_block(b"\xc8" * n, Huf(one_symbol(200), runs=bytes(r)), rng, n_seq=0), None)
    # padding bits set in every run's last byte (bitmap words and flat paths): accepted
    for tag, lens, n in (("chain11", c11, 289), ("flat3", f5, 333), ("two", lens_of({1: 2}, rng), 97)):
        ll = stream(lens, n, rng)
        sizes = []
        runs = bytearray(bg.pivco_runs(lens, ll, sizes))
        end = 0
        for _, k, c, sz in sizes:
            end += sz
            used = c * (1 if k == "bitmap" else k)
            if sz and used % 8:
                runs[end - 1] |= 0xFF & ~((1 << (used % 8)) - 1)
        yield Case("pad-%s" % tag, lit_block(ll, Huf(lens, runs=bytes(runs)), rng, n_seq=0), None)
    # extra bytes after the runs: accepted
    yield Case("extra-after-runs", lit_block(lits, Huf(c11, extra=b"\xff" * 13), rng, n_seq=0), None)
    s = [Seq(b"k", 5 + j % 3, 1) for j in range(20)]
    yield Case("tok-extra-after-runs", Block(s, b"", tok_huf=Huf(tok_lens(s, rng), extra=b"\x5a" * 7)), None)
    # section sizes
    runs = bg.pivco_runs(c11, lits)
    yield lb("lit-comp-127", Huf(c11, comp=127))
    yield lb("lit-comp-past-avail", Huf(c11, comp=128 + len(runs) + 5000))
    s = [Seq(b"k", 5 + j % 3, 1) for j in range(20)]
    yield Case("verdict-tok-comp-127", Block(s, b"", tok_huf=Huf(tok_lens(s, rng), comp=127)), None)
    # enc_lit = 3: no table, a table that fails Kraft, an all-zero table
    dl = stream(dict_lens, 300, rng)
    yield Case("verdict-dict-table-missing", lit_block(dl, Huf(dict_lens), rng, enc_lit=3, n_seq=0, dict_bytes=dict_bytes),
               None)
    yield Case("dict-table", lit_block(dl, Huf(dict_lens), rng, enc_lit=3, n_seq=0, dict_bytes=dict_bytes,
                                       dict_huf=bg.pack_lengths(dict_lens)), None)
    # a table that fails Kraft fails the frame when the reference attaches it (CORRUPT_DATA, as the block decoder says);
    # an all-zero one is no table at all there (DICT_REQUIRED) and a table without symbols to the block decoder
    bad = list(dict_lens)
    bad[max(range(256), key=lambda s: (dict_lens[s], s))] = 0
    yield Case("verdict-dict-table-kraft", lit_block(dl, Huf(dict_lens), rng, enc_lit=3, n_seq=0, dict_bytes=dict_bytes,
                                                     dict_huf=bg.pack_lengths(bad)), None)
    yield Case("verdict-dict-table-zero", lit_block(dl, Huf(dict_lens), rng, enc_lit=3, n_seq=0, dict_bytes=dict_bytes,
                                                    dict_huf=bytes(128)), None, frame_status=bg.DICT_REQUIRED)
    # enc_tok = 2 with no sequences
    two = lens_of({1: 2}, rng)
    yield Case("verdict-tok-n-seq-0-valid-table", Block([], rng.bytes(11), tok_huf=Huf(two)), None)
    yield Case("verdict-tok-n-seq-0-zero-table", Block([], rng.bytes(11), tok_huf=Huf(two, table=bytes(128))), None)


def _dict():
    rng = np.random.default_rng(99)
    return rng.bytes(3000), chain(10, rng)


_CAT = None


def catalogue():
    global _CAT
    if _CAT is None:
        d, dl = _dict()
        cases = []
        for gen in (_table_cases(), _count_cases(), _token_cases(d, dl), _block_size_cases(), _verdict_cases(d, dl)):
            cases += list(gen)
        for c in cases:  # the decoder counter each case must move
            if c.block.pivco_verdict:
                c.stat = S_VERDICT
            elif c.block.decoded:
                c.stat = target(c.block)
        names = [c.name for c in cases]
        assert len(set(names)) == len(names), "case names are unique"
        _CAT = cases
    return _CAT


CASES = catalogue()
IDS = [c.name for c in CASES]


# ------------------------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------------------------
def _same_verdict(got, want):
    return ROOM.get(got, got) == ROOM.get(want, want)


def _expect(st, out, blk, what):
    if blk.status >= 0:
        assert st == blk.status, (what, z.ERR.get(st, st))
        got = np.asarray(out[:st], np.uint8).tobytes()
        assert got == blk.want, (what, "first wrong byte at %d" % next(i for i in range(st) if got[i] != blk.want[i]))
    else:
        assert _same_verdict(st, blk.status), (what, z.ERR.get(st, st), z.ERR.get(blk.status))


def _frame_expect(c):
    """the block as a frame decodes to what the block does, unless the frame decides first"""
    if c.frame_status is None:
        return c.block

    class V:
        status, want = c.frame_status, b""
    return V


def _block_api_expect(blk):
    """the block API attaches no dictionary table: a Huffman literal section under it needs one"""
    if blk.payload[8] == 3 and struct.unpack_from("<I", blk.payload, 4)[0]:  # (its other checks pass in this catalogue)

        class V:
            status, want = bg.DICT_REQUIRED, b""
        return V
    return blk


def _dict_id(orc, blk):
    if not blk.dict_bytes:
        return 0
    return orc.lib.zxo_dict_id(blk.dict_bytes, len(blk.dict_bytes), blk.dict_huf)


def _frame(orc, blk, checksum=0):
    total = blk.status if blk.status >= 0 else blk.cap
    return bg.frame([(blk.payload, 1)], blk.block_size, checksum=checksum, dict_id=_dict_id(orc, blk), total=total), total


def _in_frame(blk):
    """a frame block decodes to at most the block size; larger outputs are another issue (test_frame_block_over_size)"""
    return blk.status <= blk.block_size


def _stats(lib):
    return (C.c_uint64 * 64).in_dll(lib, "simt_stat")


def _emu(blk, units=0, seed=1, src_res=0, dst_res=0, lean=None, with_dict=None):
    src, rows, total = bg.job_table([blk], src_res, dst_res)
    jobs = (zs.Job * 1)(zs.Job(*rows[0]))
    out = np.zeros(max(total, 1), np.uint8)
    status = (C.c_int32 * 1)()
    oob = C.c_int(0)
    s = np.frombuffer(src, np.uint8)
    d = blk.dict_bytes if with_dict is None else with_dict
    dp = np.frombuffer(d, np.uint8).ctypes.data if d else None
    hp = blk.dict_huf
    if lean is None:
        zs.lib().simt_decode_blocks(s.ctypes.data, s.size, out.ctypes.data, total, jobs, 1, status, dp, len(d), hp,
                                    blk.block_size, 0, units, seed, C.byref(oob))
    else:
        lean.simt_decode_two_stage(s.ctypes.data, s.size, out.ctypes.data, total, jobs, 1, status, dp, len(d), hp,
                                   blk.block_size, seed, C.byref(oob))
    return status[0], out[rows[0][1]:], oob.value


# ------------------------------------------------------------------------------------------------------------------
# CPU: generator, oracle, reference
# ------------------------------------------------------------------------------------------------------------------
def test_catalogue_covers_the_decoder():
    names = " ".join(IDS)
    for L in range(1, 12):
        assert "lit-chain%d-" % L in names
    for D in range(2, 9):
        assert "flat-d%d-" % D in names
    assert sum(c.block.status < 0 for c in CASES) >= 35
    assert {c.stat for c in CASES} >= {S_SINGLE, S_RANK, S_VERDICT, None} | {S_FLAT + D for D in range(2, 9)}


@pytest.fixture(scope="module")
def refi():
    if not os.path.exists(REFI_SO):
        pytest.skip("oracle/_ref/libzxc_ref_internals.so not built (reference sources absent)")
    r = C.CDLL(REFI_SO)
    r.zxri_encode_section.restype = C.c_int
    r.zxri_encode_section.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    return r


def test_writer_matches_the_reference_encoder(refi):
    """every section the writer builds from code lengths and symbols is byte-identical to the reference's encoder"""
    n = 0
    for c in CASES:
        for lens, syms, sec in c.block.written_sections:
            s = np.frombuffer(syms, np.uint8)
            if not s.size:
                continue
            f = np.bincount(s, minlength=256).astype(np.uint32)
            cl = np.array(lens, np.uint8)
            dst = np.zeros(len(sec) + 4096, np.uint8)
            r = refi.zxri_encode_section(s.ctypes.data, s.size, f.ctypes.data, cl.ctypes.data, dst.ctypes.data, dst.size)
            assert r == len(sec) and dst[:r].tobytes() == sec, (c.name, r, len(sec))
            n += 1
    assert n >= 150


def test_tree_decoder_reads_back_the_writer():
    rng = np.random.default_rng(5)
    for name, lens in _tables(rng):
        for n in (1, 33, 1000):
            syms = stream(lens, n, rng, "skew")
            sec = bg.pivco_section(lens, syms)
            assert bg.pivco_decode(sec[:128], sec[128:], n) == (n, syms), name


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_generator_agrees_with_oracle(orc, case):
    blk = case.block
    out = np.zeros(max(blk.cap, 1), np.uint8)
    d = blk.dict_bytes
    r = orc.lib.zxo_decode_block_bs(blk.raw, len(blk.raw), out.ctypes.data, blk.cap, d or None, len(d), blk.dict_huf, 0,
                                    blk.block_size)
    _expect(r, out, blk, "oracle")


def test_reference_decides_every_verdict(ref, orc):
    """each case as a one-block frame through the unmodified reference: the generator's verdict and bytes are its"""
    for c in CASES:
        blk = c.block
        if not _in_frame(blk):
            continue
        fr, total = _frame(orc, blk)
        r, o = ref.decompress(fr, total, dict=blk.dict_bytes or None, dict_huf=blk.dict_huf)
        _expect(r, o, _frame_expect(c), (c.name, "reference"))
        r, o = orc.decompress(fr, total, dict=blk.dict_bytes or None, dict_huf=blk.dict_huf)
        _expect(r, o, _frame_expect(c), (c.name, "oracle frame"))


def test_reference_block_api_agrees(ref, orc):
    """zxc_decompress_block takes the block size from dst_capacity; where that is the case's block size the verdict is
    the generator's (the token limit cases above 4 KiB included)"""
    dctx = ref.lib.zxc_create_dctx()
    try:
        for c in CASES:
            blk = c.block
            if max(4096, 1 << (blk.cap - 1).bit_length()) != blk.block_size:
                continue
            out = np.zeros(blk.cap, np.uint8)
            o = z.DecompressOpts()
            keep = np.frombuffer(blk.dict_bytes, np.uint8) if blk.dict_bytes else None
            if keep is not None:
                o.dict, o.dict_size = keep.ctypes.data, keep.size
                o.dict_huf = C.cast(C.c_char_p(blk.dict_huf), C.c_void_p) if blk.dict_huf else None
            r = ref.lib.zxc_decompress_block(dctx, blk.raw, len(blk.raw), out.ctypes.data, blk.cap, C.byref(o))
            _expect(int(r), out, _block_api_expect(blk), (c.name, "reference block API"))
    finally:
        ref.lib.zxc_free_dctx(dctx)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the kernel on the warp emulator
# ------------------------------------------------------------------------------------------------------------------
EMU = [c for c in CASES if c.emu]
EMU_IDS = [c.name for c in EMU]


@pytest.mark.parametrize("case", EMU, ids=EMU_IDS)
def test_emulator_general_instance(case):
    k = EMU_IDS.index(case.name)
    stat = _stats(zs.lib())
    for seed in (0, 1 + k, 1000 + k):
        C.memset(stat, 0, C.sizeof(stat))
        st, out, oob = _emu(case.block, seed=seed, src_res=k % 16, dst_res=(7 * k + seed) % 16)
        assert oob == 0
        _expect(st, out, case.block, "emulator seed %d" % seed)
        if case.stat is None:
            assert stat[S_RANK] == stat[S_SINGLE] == stat[S_VERDICT] == 0, "the decoder ran"
        else:
            assert stat[case.stat] > 0, ("targeted path not taken", case.stat, list(stat)[32:])


def test_emulator_lean_route_defers_every_case(lean_emu):
    """the lean instance defers every Huffman block before it reads the counts; the general one decodes it"""
    for k, c in enumerate(EMU):
        st, out, oob = _emu(c.block, seed=9 + k, src_res=(k + 5) % 16, dst_res=(3 * k) % 16, lean=lean_emu)
        assert oob == 0
        assert C.c_uint32.in_dll(lean_emu, "simt_lean_deferred").value == 1, c.name
        _expect(st, out, c.block, (c.name, "lean route"))


_GUARD_CHILD = r"""
import sys
sys.path.insert(0, %r)
import test_pivco_decode as t
import zxc_simt as zs
lib = zs.lib()
n = 0
for mode in (1, 2):
    lib.simt_guard_pages(mode)
    for c in t.EMU:
        if c.block.block_size > 65536:
            continue
        for src_res, dst_res in ((0, 0), (5, 13)):
            st, out, oob = t._emu(c.block, seed=3, src_res=src_res, dst_res=dst_res)
            assert oob == 0, c.name
            t._expect(st, out, c.block, c.name)
            n += 1
print("guard ok", n)
"""


def test_emulator_loads_stay_inside_the_buffers():
    """every emulated case with the source, destination and dictionary (+ its 128-byte table) against PROT_NONE
    pages, flush with either end.  The token-section cases whose last run ends 1..3 bytes before the payload (and, in
    mode 2, the source) ends are the ones where a 4-byte bitmap word or a 3-byte flat path would read past it."""
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _GUARD_CHILD % here], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "guard ok" in r.stdout, (r.returncode, r.stdout[-1500:], r.stderr[-1500:])


# ------------------------------------------------------------------------------------------------------------------
# the frame planning divergence (not PivCo)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.xfail(reason="frame planning: a block that decodes to more than the frame's block size is given only the "
                          "block size of room; the reference decodes it into block_size + its tail padding", strict=False)
def test_frame_block_over_size(ref, orc, prod):
    s = [Seq(b"Q" if j == 0 else b"", 5, 1) for j in range(835)]
    blk = Block(s, b"", block_size=4096)
    fr, total = _frame(orc, blk)
    r0, o0 = ref.decompress(fr, total)
    assert r0 == blk.status
    st, out = zs.decode_frame(prod, fr)[:2]
    assert st[0] == r0


# ------------------------------------------------------------------------------------------------------------------
# the compiled sm_90a kernels
# ------------------------------------------------------------------------------------------------------------------
def _groups():
    g = {}
    for c in CASES:
        b = c.block
        g.setdefault((b.block_size, b.dict_bytes, b.dict_huf), []).append(b)
    return g


def _gpu_table(prod, blocks, block_size, dict_bytes, dict_huf, verify, src_res, dst_res):
    import torch
    lib = prod.lib
    lib.zxc_b200_decode_scratch_size.restype = C.c_size_t
    lib.zxc_b200_decode_scratch_size.argtypes = [C.c_uint32]
    lib.zxc_b200_decode_blocks.restype = C.c_int
    lib.zxc_b200_decode_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                           C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_int, C.c_void_p]

    class Signed:
        def __init__(self, b):
            self.raw, self.cap = bg.block_bytes(1, b.payload, True), b.cap

    src, rows, total = bg.job_table([Signed(b) for b in blocks] if verify else blocks, src_res, dst_res)
    dev = torch.device("cuda", 0)
    table = (zs.Job * len(rows))(*[zs.Job(*r) for r in rows])
    d_src = torch.from_numpy(np.frombuffer(src, np.uint8).copy()).to(dev)
    d_dst = torch.zeros(total, dtype=torch.uint8, device=dev)
    d_jobs = torch.from_numpy(np.frombuffer(bytes(table), np.uint8).copy()).to(dev)
    d_status = torch.zeros(len(rows), dtype=torch.int32, device=dev)
    dd = (dict_bytes or b"") + (dict_huf or bytes(128))
    d_dict = torch.from_numpy(np.frombuffer(dd, np.uint8).copy()).to(dev) if (dict_bytes or dict_huf) else None
    ss = lib.zxc_b200_decode_scratch_size(block_size)
    d_scratch = torch.empty(ss, dtype=torch.uint8, device=dev)
    rc = lib.zxc_b200_decode_blocks(d_src.data_ptr(), d_dst.data_ptr(), d_jobs.data_ptr(), len(rows), d_status.data_ptr(),
                                    d_dict.data_ptr() if dict_bytes else None, len(dict_bytes),
                                    d_dict.data_ptr() + len(dict_bytes) if dict_huf else None,
                                    d_scratch.data_ptr(), ss, block_size, verify, torch.cuda.current_stream(dev).cuda_stream)
    assert rc == 0, z.ERR.get(rc, rc)
    torch.cuda.synchronize(dev)
    return list(d_status.cpu().numpy()), d_dst.cpu().numpy(), [(r[1], r[3]) for r in rows]


@pytest.mark.gpu
@pytest.mark.parametrize("verify", [0, 1], ids=["lean-then-general", "general-verified"])
def test_gpu_job_tables_at_every_residue(prod, verify):
    """every case through zxc_b200_decode_blocks, one launch per (block size, dictionary, table) at source and
    destination offsets of every residue mod 16; the cases without a dictionary once more with one present"""
    groups = _groups()
    d = _dict()[0]
    extra = [((4096, d, None), [b for b in groups.get((4096, b"", None), []) if b.status >= 0])]
    for (bs, dict_bytes, dict_huf), blocks in list(groups.items()) + extra:
        for r in range(16) if bs < (1 << 21) else (0, 7):
            st, out, spans = _gpu_table(prod, blocks, bs, dict_bytes, dict_huf, verify, r, (5 * r + 3) % 16)
            for s, (d0, cap), blk in zip(st, spans, blocks):
                _expect(int(s), out[d0:d0 + cap], blk, ("residue", r, bs, len(dict_bytes)))


@pytest.mark.gpu
@pytest.mark.parametrize("checksum", [0, 1])
def test_gpu_frames_and_block_api(prod, orc, checksum):
    dctx = prod.lib.zxc_create_dctx()
    try:
        for c in CASES:
            blk = c.block
            d = blk.dict_bytes or None
            if _in_frame(blk):
                fr, total = _frame(orc, blk, checksum)
                r1, o1 = prod.decompress(fr, total, checksum=checksum, dict=d, dict_huf=blk.dict_huf)
                _expect(r1, o1, _frame_expect(c), (c.name, "zxc_decompress"))
            if max(4096, 1 << (blk.cap - 1).bit_length()) != blk.block_size:
                continue
            raw = bg.block_bytes(1, blk.payload, True) if checksum else blk.raw
            out = np.zeros(blk.cap, np.uint8)
            o = z.DecompressOpts(checksum_enabled=checksum)
            keep = np.frombuffer(blk.dict_bytes, np.uint8) if d else None
            if d:
                o.dict, o.dict_size = keep.ctypes.data, keep.size
                o.dict_huf = C.cast(C.c_char_p(blk.dict_huf), C.c_void_p) if blk.dict_huf else None
            r3 = prod.lib.zxc_decompress_block(dctx, raw, len(raw), out.ctypes.data, blk.cap, C.byref(o))
            _expect(int(r3), out, _block_api_expect(blk), (c.name, "zxc_decompress_block"))
    finally:
        prod.lib.zxc_free_dctx(dctx)


_ALT_CHILD = r"""
import sys
sys.path.insert(0, %r)
import test_pivco_decode as t
import zxc_ctypes as z
prod, orc = z.ZxcLib(z.PRODUCT_SO), z.Oracle()
n = 0
for c in t.CASES:
    blk = c.block
    if not t._in_frame(blk):
        continue
    for cks in (0, 1):
        fr, total = t._frame(orc, blk, cks)
        r, o = prod.decompress(fr, total, checksum=cks, dict=blk.dict_bytes or None, dict_huf=blk.dict_huf)
        t._expect(r, o, t._frame_expect(c), (c.name, cks))
        n += 1
print("alt ok", n)
"""


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{"ZXC_B200_UNITS": "1"}], ids=["unit-walk-forced"])
def test_gpu_alternative_bodies_on_the_catalogue(env):
    e = dict(os.environ)
    e.update(env)
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _ALT_CHILD % here], env=e, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "alt ok" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
