"""TEST INFRASTRUCTURE: a catalogue of encoder inputs, each shaped to reach one path of the block encoder
(zxc_b200/csrc/zxc_encode.cuh, levels 1-5, and zxc_encode_opt.cuh, levels 6-7) that a general corpus reaches only by
luck: the window edge, chain slots recycled inside a match-finder batch, inserts undone after a long match, hash-bucket
pressure, the repeat-offset probe, length / count / varint limits, section choices at their thresholds and
dictionaries.  Every input is deterministic.  A case names the counter of the emulator build (ZXC_STAT /
ZXC_LANE_STAT, S_* below) that must be non-zero when it is encoded, so a case that stops reaching its path fails."""
import numpy as np

# encoder event counters of the emulator build (tests/simt/simt_encode.cc: simt_stat[64..])
S_BATCH, S_TRUNC, S_UNDO_HEAD, S_UNDO = 64, 65, 66, 67
S_RDCHAIN_OLD, S_FIXUP_OLD, S_INSERT_GROUP = 68, 69, 70
S_REP_ARITH, S_REP_SPEC, S_REP_LOAD, S_REP_TIE = 71, 72, 73, 74
S_DP_FAR, S_LMAX_CAP, S_FAR_OPT, S_FAR = 75, 76, 77, 78
S_LAZY, S_STEP, S_BACK, S_L5_INSERT = 79, 80, 81, 82
S_RAW, S_RLE, S_HUF, S_HUF_DICT, S_TOK_HUF, S_OFF8 = 83, 84, 85, 86, 87, 88
S_FLAT_ROOT, S_SLOT_GROUP, S_DICT_SEED, S_SKIP_HEAD, S_HUF_BUILT = 89, 90, 91, 92, 93

STAT_NAMES = {
    S_BATCH: "batches", S_TRUNC: "truncated batches", S_UNDO_HEAD: "undo: head restored", S_UNDO: "undone inserts",
    S_RDCHAIN_OLD: "skip-head link from oldc", S_FIXUP_OLD: "walk link from oldc", S_INSERT_GROUP: "insert groups > 1",
    S_REP_ARITH: "repeat probe: arithmetic", S_REP_SPEC: "repeat probe: speculative", S_REP_LOAD: "repeat probe: loaded",
    S_REP_TIE: "repeat offset wins a tie", S_DP_FAR: "DP past the register front", S_LMAX_CAP: "L_max capped",
    S_FAR_OPT: "candidates past the window (6-7)", S_FAR: "candidates past the window (1-5)", S_LAZY: "lazy replacements",
    S_STEP: "step skips > 1", S_BACK: "backtracked starts", S_L5_INSERT: "level-5 match_end-2 inserts",
    S_RAW: "RAW blocks", S_RLE: "RLE literals", S_HUF: "HUF literals", S_HUF_DICT: "shared-table literals",
    S_TOK_HUF: "HUF tokens", S_OFF8: "8-bit offsets", S_FLAT_ROOT: "PivCo flat-root writes",
    S_SLOT_GROUP: "PivCo same-node slot groups", S_DICT_SEED: "per-block dictionary seed", S_SKIP_HEAD: "skip_head",
    S_HUF_BUILT: "literal Huffman code built",
}

M64 = (1 << 64) - 1


def hash5(v):
    """enc_hash(v, true) of the 8 little-endian bytes at a position (levels 3-7)"""
    return (((v & 0xFFFFFFFFFF) * 0x2545F4914F6CDD1D) & M64) >> 49


def tag(v):
    """enc_tag of the first 4 bytes"""
    v &= 0xFFFFFFFF
    return (v ^ (v >> 16)) & 0xFF


def le(b):
    return int.from_bytes(bytes(b[:8]).ljust(8, b"\0"), "little")


class Case:
    """one input: `levels` it is encoded at, block size `bs` (0: the default), `stat` the counter that must be non-zero
    on the emulator (summed over its levels), `emu` False for inputs too large for the CPU emulator"""

    def __init__(self, name, doc, data, levels, bs=65536, checksum=0, stat=None, dict=None, dict_huf=None, emu=True,
                 guard=False):
        self.name, self.doc, self.levels, self.bs, self.checksum, self.stat = name, doc, tuple(levels), bs, checksum, stat
        self.data = np.frombuffer(bytes(data), np.uint8) if not isinstance(data, np.ndarray) else data
        self.dict, self.dict_huf, self.emu, self.guard = dict, dict_huf, emu, guard

    def __repr__(self):
        return self.name


def _rand(seed, n):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def _rand64(seed, n):
    """random bytes from a 64-letter alphabet: few chance matches, but literals that still compress (the block is not
    stored RAW, so the parse shows in the output)"""
    return np.random.default_rng(seed).integers(32, 96, n, dtype=np.uint8)


# ------------------------------------------------------------------------------------------------------------------
def window_edge():
    """A 64-byte motif repeated at distances 65 534..65 537 over a zero filler: the candidate at 65 536 or more must be
    dropped by the ENC_MAX_DIST test in the chain walk (levels 1-5: find_best_match, 6-7: the lane walks)."""
    for bs, emu in ((131072, True), (524288, False), (2 << 20, False)):
        for d in (65534, 65535, 65536, 65537):
            data = np.zeros(bs, np.uint8)
            motif = _rand(d, 64)
            a = 3000
            data[a:a + 64] = motif
            data[a + d:a + d + 64] = motif
            data[a + d + 64:a + d + 80] = _rand(d + 1, 16)  # the copy ends differently from the original
            far = d > 65535
            yield Case("window-d%d-bs%dk" % (d, bs >> 10), window_edge.__doc__, data, range(1, 8), bs,
                       stat=((S_FAR, S_FAR_OPT, S_BACK) if far else None), emu=emu, checksum=d & 1)
    for k in (1, 13, 100):
        """the block is 65 536 + k bytes: position p and p - 65 536 share a chain slot"""
        base = _rand64(100 + k, 65536 + k)
        base[65536:] = base[:k]
        base[30000:30200] = base[100:300]
        yield Case("window-n65536+%d" % k, "A block of 65 536 + k bytes whose tail repeats its head: positions p and "
                   "p - 65 536 share a chain slot, the head candidate is exactly 65 536 back.", base, (1, 3, 6, 7), 131072,
                   stat=None)


def _recycled(i, j, seed, with_far):
    """Position X (batch index i) looks for motif A: a 12-byte prefix of it at Q, whose chain slot the batch's own index
    j overwrites (X - Q = 65 536 - (j - i)); 24 bytes of it at Z = Q - 26, reachable only through Q's saved link (oldc);
    with_far: 36 bytes at exactly 65 536 back, which the distance filter must drop."""
    n = 98304
    data = _rand64(seed, n)
    X = 128 * 560 + i
    Q = X + (j - i) - 65536
    Z = Q - 26
    assert X - Z <= 65535
    A = _rand(seed + 1, 64)
    data[Z:Z + 24] = A[:24]
    data[Q:Q + 12] = A[:12]
    data[X:X + 24] = A[:24]
    if with_far:
        Z2 = X - 65536
        assert Z2 + 36 <= Z
        data[Z2:Z2 + 36] = A[:36]
        data[X:X + 36] = A[:36]
    return data


def _hashes(data):
    """hash5 of every position of data (zero bytes past its end)"""
    d = np.concatenate([data, np.zeros(8, np.uint8)]).astype(np.uint64)
    v = d[:-8] | d[1:-7] << np.uint64(8) | d[2:-6] << np.uint64(16) | d[3:-5] << np.uint64(24) | d[4:-4] << np.uint64(32)
    return (v * np.uint64(0x2545F4914F6CDD1D)) >> np.uint64(49)


def _clear_bucket(data, h, lo, hi, keep):
    """changes unprotected bytes until no position in [lo, hi) hashes to bucket h"""
    for _ in range(100):
        bad = np.nonzero(_hashes(data)[lo:hi] == h)[0] + lo
        if bad.size == 0:
            return
        for p in bad:
            q = next(q for q in range(p, p + 5) if not keep[q])
            data[q] ^= 0x5A
    raise AssertionError("bucket not cleared")


def recycled_slots():
    """Level 6-7, block over 64 KiB: the current batch overwrites chain slots that a lane walking 65 536 - 128 .. 65 536
    positions back still needs; the walk must read the saved copy (oldc), and the distance filter decides the rest."""
    for i, j, far in ((10, 90, True), (40, 120, True), (70, 100, False), (100, 127, False), (0, 31, False)):
        yield Case("recycled-i%d-j%d" % (i, j), recycled_slots.__doc__, _recycled(i, j, 700 + i, far), (6, 7), 131072,
                   stat=S_FIXUP_OLD)
    # the head candidate itself is recycled and its tag differs: the skip_head link (OPT_RDCHAIN) reads oldc
    data = _rand64(790, 98304)
    v, w = _bucket_pair(1234, same_tag=False)
    X = 128 * 560 + 20
    Q = X + 60 - 65536
    A = _rand(791, 40)
    A[:8] = np.frombuffer(v.to_bytes(8, "little"), np.uint8)
    data[Q - 30:Q - 30 + 40] = A  # the real candidate, linked from Q's old slot
    data[Q:Q + 8] = np.frombuffer(w.to_bytes(8, "little"), np.uint8)  # same bucket, other tag: the head, skipped
    data[X:X + 40] = A
    keep = np.zeros(data.size, bool)
    keep[Q - 30:Q + 10] = keep[X:X + 40] = True
    _clear_bucket(data, hash5(v), Q + 1, X, keep)  # nothing between Q and X takes over the head
    yield Case("recycled-skip-head", "Level 6-7: the head of X's bucket is a recycled slot whose tag differs from X's, "
               "so the skip_head step reads the displaced link (OPT_RDCHAIN from oldc).", data, (6, 7), 131072,
               stat=S_RDCHAIN_OLD)


def long_match_undo():
    """A match of 300 bytes starting mid-batch at index i (rows k = 0..3, lanes 0 and 31): the batch's later inserts are
    undone.  The undone positions share hashes with positions before the batch and with a lower position of the same
    batch, and the same bytes come again later, so a head restored wrongly changes a later match."""
    for i in (0, 31, 37, 69, 101, 127):
        data = _rand64(800 + i, 65536)
        C = _rand(900 + i, 300)
        S0 = 5000
        data[S0:S0 + 300] = C
        X = 128 * 200 + i
        data[X:X + 300] = C
        data[X - 1] = data[S0 - 1] ^ 0x5A  # the match starts exactly at X
        if i >= 12:
            data[X - 10:X - 2] = C[20:28]  # a lower position of the batch with the hash of undone position X + 20
        Y = 50000
        data[Y:Y + 40] = C[20:60]
        data[Y + 40:Y + 48] = C[20:28]
        # at index 127 the match is the batch's last position: nothing is left to undo
        yield Case("undo-i%d" % i, long_match_undo.__doc__, data, (6, 7), 65536,
                   stat=(S_UNDO_HEAD, S_UNDO, S_TRUNC) if i < 127 else S_BATCH)


def _bucket_values(seed, count=4000000):
    """random 8-byte values and their hash5 buckets"""
    rng = np.random.default_rng(seed)
    vals = rng.integers(0, 1 << 63, count, dtype=np.uint64) | (rng.integers(0, 2, count, dtype=np.uint64) << 63)
    h = ((vals & np.uint64(0xFFFFFFFFFF)) * np.uint64(0x2545F4914F6CDD1D)) >> np.uint64(49)
    return vals, h


def _bucket_pair(seed, same_tag):
    vals, h = _bucket_values(seed, 200000)
    order = np.argsort(h, kind="stable")
    hs = h[order]
    for a in range(len(hs) - 1):
        if hs[a] == hs[a + 1]:
            v, w = int(vals[order[a]]), int(vals[order[a + 1]])
            if (tag(v) == tag(w)) == same_tag and (v & 0xFFFFFFFF) != (w & 0xFFFFFFFF):
                return v, w
    raise AssertionError("no pair")


def bucket_pressure():
    """Many distinct values in one 15-bit hash bucket (levels 3-7), with different tags and with equal tags: skip_head,
    chains that run out of attempts; and runs of 6..36 equal bytes, whose positions form __match_any_sync insert groups
    of 2..32 lanes."""
    vals, h = _bucket_values(77, 1000000)
    counts = np.bincount(h.astype(np.int64), minlength=1 << 15)
    b = int(np.argmax(counts))
    members = [int(v) for v in vals[h == b]]
    rng = np.random.default_rng(78)
    out = []
    for r in range(12):
        for v in rng.permutation(members):
            out.append(int(v).to_bytes(8, "little")[:5])
            out.append(rng.bytes(int(rng.integers(0, 4))))
    yield Case("bucket-tags", bucket_pressure.__doc__, b"".join(out)[:60000], (3, 5, 6, 7), 65536,
               stat=(S_SKIP_HEAD, S_L5_INSERT))
    parts = []
    for g in list(range(2, 33)) * 3:
        parts.append(bytes([int(rng.integers(0, 256))]) * (g + 4))
        parts.append(rng.bytes(int(rng.integers(5, 40))))
    yield Case("bucket-groups", bucket_pressure.__doc__, b"".join(parts), (6, 7), 65536, stat=S_INSERT_GROUP)


def repeat_offsets():
    """The repeat-offset probe: a chain match tied by the repeat offset (which wins the tie), segments alternating
    between two offsets (speculative and loaded probes) and a stretch longer than one batch at one offset (the
    arithmetic path)."""
    rng = np.random.default_rng(61)
    data = bytearray(rng.bytes(40000))
    for t in range(60):  # ties: X-1 matches P1-1 (31 bytes), X finds the closer P2 (30 bytes) first
        P1, P2, X = 2000 + 400 * t, 2200 + 400 * t, 30000 + 150 * t
        S = rng.bytes(30)
        data[P1 - 1:P1 + 30] = bytes([data[X - 1]]) + S
        data[P2:P2 + 30] = S
        data[P2 - 1] = data[X - 1] ^ 1
        data[X:X + 30] = S
    yield Case("repeat-tie", repeat_offsets.__doc__, bytes(data), (6, 7), 65536, stat=S_REP_TIE)
    src = rng.bytes(3000)
    out = bytearray(src)
    for t in range(200):
        off = (1000, 1723)[t & 1]
        for _ in range(int(rng.integers(12, 40))):
            out.append(out[-off])
        out += rng.bytes(int(rng.integers(1, 3)))
    yield Case("repeat-alternating", repeat_offsets.__doc__, bytes(out), (6, 7), 65536, stat=(S_REP_LOAD, S_REP_SPEC))
    body = bytearray(rng.bytes(2000))
    for _ in range(6000):
        body.append(body[-777])
    body += rng.bytes(100)
    yield Case("repeat-stretch", repeat_offsets.__doc__, bytes(body), (6, 7), 65536, stat=S_REP_ARITH)


def _lit_match(ll_list, ml_list, seed):
    """literal runs of the given lengths (fresh random bytes) each followed by a match of the given length copied from an
    early random pool, whose next byte differs"""
    rng = np.random.default_rng(seed)
    pool = rng.bytes(20000)
    out = bytearray(pool)
    for ll, ml in zip(ll_list, ml_list):
        out += rng.bytes(ll)
        s = int(rng.integers(0, len(pool) - ml - 1)) if ml < len(pool) - 1 else 0
        out += pool[s:s + ml] if ml < len(pool) else (pool * (ml // len(pool) + 1))[:ml]
        out.append(pool[s + ml] ^ 0xFF if s + ml < len(pool) else 0x55)
    return bytes(out)


def length_limits():
    """Literal runs and match lengths at the token nibble (14/15/16), and the varint byte counts (15 + 127/128,
    15 + 16 383/16 384); GHI's 8-bit fields (254/255/256); matches of 65 535 and 65 536+ bytes at levels 6-7 (the L_max
    cap); literal-only tails: n < 9 blocks, the last 8 bytes, k * bs + 1..13 and a 1-byte last block of 4 KiB blocks."""
    for tag_, lens, lv in (("nibble", (14, 15, 16, 19, 20, 21), range(1, 8)), ("var1", (141, 142, 143, 144), range(1, 8)),
                           ("var2", (16397, 16398, 16399, 16400), (1, 3, 6)), ("ghi", (258, 259, 260, 261, 262), (1, 2))):
        ll = [x for x in lens for _ in range(2)]
        ml = [x for x in reversed(lens) for _ in range(2)]
        yield Case("len-%s" % tag_, length_limits.__doc__, _lit_match(ll, ml, 40 + len(tag_)), lv, 131072,
                   stat=S_DP_FAR if tag_ == "var1" else None, checksum=1)
    for n in (65536, 65537, 65836):
        data = np.zeros(n + 2000, np.uint8)
        data[:1000] = _rand(n, 1000)
        data[1000 + n:] = _rand(n + 1, 1000)
        yield Case("len-run%d" % n, "A zero run of %d bytes: a match of run - 1 bytes at offset 1, capped at 65 535 by "
                   "L_max from 65 536 up." % n, data, (6, 7), 131072, stat=S_LMAX_CAP if n > 65536 else S_DP_FAR)
    text = np.frombuffer(b"abcdefghij" * 2000, np.uint8)
    for n in range(1, 14):
        yield Case("tail-n%d" % n, "A block of n < 14 bytes: literal-only (n < 9) or a match-free last 8 bytes.",
                   text[:n], range(1, 8), 4096, stat=None, checksum=n & 1)
    for extra in (1, 5, 9, 13):
        yield Case("tail-2bs+%d" % extra, "Two full blocks and a last block of 1..13 bytes.", text[:2 * 4096 + extra],
                   (1, 3, 6, 7), 4096, stat=None)
    yield Case("tail-1byte", "A 1-byte last block of 4 KiB blocks.", text[:3 * 4096 + 1], (2, 5, 7), 4096, checksum=1)


def _offset_case(off, seed):
    """a random period of `off` bytes, repeated: every match is at offset `off` (max_off = off - 1)"""
    return np.tile(_rand(seed, off), 8000 // off + 1)


def sections():
    """The section choice: 8-bit offsets at largest offsets of 256 / 257 (max_off 255 / 256), RLE against RAW
    literals, Huffman literal sections at levels 6-7 (one- and two-symbol alphabets, 11-bit codes at level 7), token
    Huffman at level 7 and the RAW fallback of a block that does not shrink."""
    for off in (255, 256, 257, 258):
        yield Case("off8-%d" % off, sections.__doc__, _offset_case(off, off), range(1, 8), 65536,
                   stat=(S_OFF8 if off <= 256 else None))
    rng = np.random.default_rng(5)
    runs = bytearray()
    while len(runs) < 30000:
        runs += bytes([int(rng.integers(0, 256))]) * int(rng.integers(1, 9))
    yield Case("rle", sections.__doc__, bytes(runs), (3, 5, 6), 65536, stat=(S_RLE, S_LAZY))
    two = np.where(rng.random(20000) < 0.8, 97, 98).astype(np.uint8)
    yield Case("huf-2sym", sections.__doc__, two, (6, 7), 65536, stat=(S_HUF, S_SLOT_GROUP))
    u = rng.random(30000)
    wide = (np.minimum(-np.log2(u + 1e-12) * 6, 255)).astype(np.uint8)
    yield Case("huf-wide", sections.__doc__, wide, (6, 7), 65536, stat=S_FLAT_ROOT)
    toks = bytearray(rng.bytes(300))
    for _ in range(3000):
        toks += rng.bytes(int(rng.choice([0, 1, 2, 3], p=[.6, .2, .1, .1])))
        o = int(rng.integers(5, 250))
        for _ in range(int(rng.choice([5, 6, 7, 9]))):
            toks.append(toks[-o])
    yield Case("huf-tokens", sections.__doc__, bytes(toks), (6, 7), 65536, stat=S_TOK_HUF)
    yield Case("raw-random", sections.__doc__, _rand(9, 70000), (1, 3, 6, 7), 65536, stat=(S_RAW, S_STEP), checksum=1)
    for lit in (136, 138, 139, 140):
        d = bytearray(_rand(lit, lit - 1))  # m random bytes, then zeros: the first zero is literal m + 1
        d += bytes(4000)
        c = Case("huf-min-lit%d" % lit, "Literal counts around HUF_MIN_LITERALS (139): the literal Huffman code is "
                 "built only from 139 literals up.", bytes(d), (6, 7), 65536, stat=(S_HUF_BUILT if lit >= 139 else None))
        c.lit_c = lit
        yield c
    # the dictionary's shared literal table: 5-bit codes for 16 letters, 8 and 9 bits for the rest; a block of fewer
    # than 1 024 such literals is cheaper with it than with its own 4-bit code and 128-byte header, a longer one is not
    lens = np.full(256, 9, np.uint8)
    lens[97:113] = 5
    lens[0:16] = 8
    packed = (lens[0::2] | (lens[1::2] << 4)).astype(np.uint8).tobytes()
    d = _rand(3, 4096).tobytes()
    for n, st in ((800, S_HUF_DICT), (3000, S_HUF)):
        lit = (97 + np.random.default_rng(n).integers(0, 16, n)).astype(np.uint8)
        yield Case("huf-shared-%d" % n, "The dictionary's shared literal table against the block's own Huffman code.",
                   lit, (6, 7), 65536, dict=d, dict_huf=packed, stat=st)


def dictionaries():
    """Dictionaries of 5, 6, 8, 4 096 and 65 535 bytes; matches starting in the dictionary's first and last 8 bytes; the
    one per-block seeded position whose hash window reaches into the block (levels 1-2: 6-byte window, 3+: 5 bytes)."""
    rng = np.random.default_rng(31)
    for size in (5, 6, 8, 4096, 65535):
        d = rng.bytes(size)
        parts = [rng.bytes(50)]
        for k in range(40):
            a = (0, max(0, size - 8), max(0, size - 3))[k % 3]
            parts.append(d[a:a + 24] + bytes(d[:min(size, 8)][::-1]))
            parts.append(rng.bytes(int(rng.integers(3, 30))))
        data = b"".join(parts) * 3
        levels = (1, 2, 3, 5, 6, 7) if size < 65535 else (1, 3, 6)
        yield Case("dict%d" % size, dictionaries.__doc__, data, levels, 4096 if size < 4096 else 65536, checksum=1,
                   dict=d, stat=S_DICT_SEED)
        # the block starts with the bytes that complete the dictionary's last positions
        yield Case("dict%d-edge" % size, dictionaries.__doc__, d[-4:] + d[:60] + rng.bytes(20) + d[-30:] * 4,
                   (1, 2, 3, 6), 4096, dict=d, stat=S_DICT_SEED)


def all_cases():
    cases = []
    for g in (window_edge, recycled_slots, long_match_undo, bucket_pressure, repeat_offsets, length_limits, sections,
              dictionaries):
        cases.extend(g())
    names = [c.name for c in cases]
    assert len(names) == len(set(names)), names
    return cases
