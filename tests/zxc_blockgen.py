"""TEST INFRASTRUCTURE: a sequence-level writer of ZXC blocks and frames.

The input is a list of sequences -- (literal bytes, match length, offset) -- plus trailing literals; the writer lays
them out as a GLO block (16-bit or 8-bit offsets, raw or RLE literal section) or a GHI block (32-bit sequence words),
with the length escapes as prefix varints in their 1-, 2- or 3-byte forms, and the 32-byte literal slack the format
asks for.  A varint may be written in a longer form than needed, or left out or jammed on purpose to build the
damaged inputs the decoder is specified to reject or to read as 0.  Blocks go into frames (file header, block headers
and checksums, end-of-frame block, footer with the global hash) or into raw job tables at chosen 16-byte residues of
their source and destination offsets.

Every block carries what it is meant to decode to, computed here by a plain byte loop over the sequences (the
reference's lz_emit semantics, dictionary reads included): the decoded bytes, or the error code of the first sequence
that cannot be emitted.  Huffman sections are not written; reference-encoded frames cover them.

The header hashes and block checksums come from the test oracle (oracle/libzxc_oracle.so)."""
import struct

import numpy as np

MIN_MATCH = 5
SLACK = 32
OVERFLOW, BAD_OFFSET = -10, -9

_orc = None


def _oracle():
    global _orc
    if _orc is None:
        import zxc_ctypes as z
        _orc = z.Oracle()
    return _orc


def varint(v, form=None):
    """prefix varint of v: form 1 (< 2^7), 2 (< 2^14) or 3 (< 2^21); None = the shortest"""
    if form is None:
        form = 1 if v < (1 << 7) else 2 if v < (1 << 14) else 3
    assert 0 <= v < (1 << (7 * form)), (v, form)
    if form == 1:
        return bytes([v])
    if form == 2:
        return bytes([0x80 | (v & 0x3F), v >> 6])
    return bytes([0xC0 | (v & 0x1F), (v >> 5) & 0xFF, v >> 13])


class Seq:
    """One sequence.  `ll_form` / `ml_form` choose how an escaped length's remainder is written: None = shortest varint,
    1/2/3 = that form, "omit" = no bytes (the remainder must be 0: the reader finds zeros or the section's end),
    "jam" = a 0xE0 prefix, which reads as 0 and moves the cursor to the section's end."""

    def __init__(self, lit=b"", ml=MIN_MATCH, off=1, ll_form=None, ml_form=None):
        self.lit = bytes(lit)
        self.ml = ml
        self.off = off
        self.ll_form = ll_form
        self.ml_form = ml_form

    def __repr__(self):
        return "Seq(ll=%d, ml=%d, off=%d)" % (len(self.lit), self.ml, self.off)


def rle_encode(data, plan=None):
    """RLE literal section (oracle rle_expand): a token t < 0x80 is followed by t + 1 raw bytes, t >= 0x80 repeats the
    next byte (t & 0x7F) + 4 times.  `plan` is a list of ("raw" | "rep", length) runs covering `data`; by default runs
    of 4..131 equal bytes repeat and everything else goes raw in pieces of up to 128."""
    data = bytes(data)
    if plan is None:
        plan, i = [], 0
        while i < len(data):
            j = i
            while j < len(data) and j - i < 131 and data[j] == data[i]:
                j += 1
            if j - i >= 4:
                plan.append(("rep", j - i))
                i = j
                continue
            k = i  # raw run: up to the next run of four equal bytes
            while k < len(data) and k - i < 128 and not (k + 3 < len(data) and data[k] == data[k + 1] == data[k + 2] == data[k + 3]):
                k += 1
            plan.append(("raw", max(k - i, 1)))
            i += max(k - i, 1)
    out, i = bytearray(), 0
    for kind, n in plan:
        if kind == "rep":
            assert 4 <= n <= 131 and data[i:i + n] == bytes([data[i]]) * n
            out += bytes([0x80 | (n - 4), data[i]])
        else:
            assert 1 <= n <= 128
            out += bytes([n - 1]) + data[i:i + n]
        i += n
    assert i == len(data)
    return bytes(out), plan


def lz_decode(seqs, tail, cap, dict_bytes=b"", n_lit=None, lits=None):
    """(status, bytes) of the reference's sequence loop: literals then match per sequence, a match byte at distance
    `off` read from the output or, before its start, from the end of the dictionary; then the trailing literals.
    `n_lit` (default: all literals present) is the literal count the block declares, `lits` the literal section when
    it is not the sequences' literals and the tail."""
    if lits is None:
        lits = b"".join(s.lit for s in seqs) + bytes(tail)
    if n_lit is None:
        n_lit = len(lits)
    out = bytearray()
    lpos = 0
    ds = len(dict_bytes)
    for s in seqs:
        ll = len(s.lit)
        if ll + s.ml > cap - len(out) or ll > n_lit - lpos:
            return OVERFLOW, bytes(out)
        out += lits[lpos:lpos + ll]
        lpos += ll
        o = len(out)
        if o + ds < s.off:
            return BAD_OFFSET, bytes(out)
        for k in range(s.ml):
            p = o + k
            out.append(out[p - s.off] if p >= s.off else dict_bytes[ds - (s.off - p)])
    rem = n_lit - lpos
    if rem > cap - len(out):
        return OVERFLOW, bytes(out)
    out += lits[lpos:lpos + rem]
    return len(out), bytes(out)


def _escapes(seqs, esc):
    """the extras section: per sequence the ll remainder, then the ml remainder, in the forms asked for"""
    ext = bytearray()
    ended = False  # a jam or an omitted varint: everything after must read as 0 from zeros or the end
    for s in seqs:
        for v, form in ((len(s.lit) - esc, s.ll_form), (s.ml - MIN_MATCH - esc, s.ml_form)):
            if v < 0:
                continue
            if form in ("omit", "jam"):
                assert v == 0, "an omitted or jammed varint reads as 0"
                if form == "jam" and not ended:
                    ext.append(0xE0)
                ended = True
                continue
            assert not ended, "a varint after a jammed or omitted one is never read"
            ext += varint(v, form)
    return bytes(ext), ended


class Block:
    """A GLO or GHI block: `raw` is the on-disk block (8-byte header + payload [+ checksum]), `want` the status and
    bytes it decodes to with `dict_bytes` into `cap` bytes."""

    def __init__(self, seqs, tail=b"", kind="glo", enc_off=0, enc_lit=0, rle_plan=None, dict_bytes=b"", cap=None,
                 extra_pad=0, checksum=False, n_lit=None):
        self.seqs, self.tail, self.kind = list(seqs), bytes(tail), kind
        self.dict_bytes = bytes(dict_bytes)
        lits = b"".join(s.lit for s in self.seqs) + self.tail
        n_lit_decl = len(lits) if n_lit is None else n_lit
        lits = (lits + bytes(max(0, n_lit_decl - len(lits))))[:n_lit_decl]  # a section holds what the header declares
        esc = 15 if kind == "glo" else 255
        omax = (256 if enc_off else 65536) if kind == "glo" else 65536
        for s in self.seqs:
            assert 1 <= s.off <= omax and s.ml >= MIN_MATCH, s
        ext, _ = _escapes(self.seqs, esc)
        if kind == "glo":
            tok = bytes((min(len(s.lit), 15) << 4) | min(s.ml - MIN_MATCH, 15) for s in self.seqs)
            offs = b"".join(bytes([s.off - 1]) if enc_off else struct.pack("<H", s.off - 1) for s in self.seqs)
            if enc_lit == 1:
                lsec, self.rle_plan = rle_encode(lits, rle_plan)
                desc = struct.pack("<I", len(lsec))
            else:
                lsec, desc = lits, b""
            body = tok + offs + ext
            hdr = struct.pack("<IIBBBB", len(self.seqs), n_lit_decl, enc_lit, 0, 0, enc_off) + desc
        else:
            words = b"".join(struct.pack("<I", (min(len(s.lit), 255) << 24) | (min(s.ml - MIN_MATCH, 255) << 16) | (s.off - 1))
                             for s in self.seqs)
            lsec, hdr = lits, struct.pack("<IIBBBB", len(self.seqs), n_lit_decl, 0, 0, 0, 0)
            body = words + ext
        pad = max(0, SLACK - len(body)) + extra_pad  # zeros: read as varint 0 where an escape reaches them
        self.ext_end = len(ext) + pad
        self.payload = hdr + lsec + body + bytes(pad)
        self.cap = cap
        out_len = len(lits) + sum(s.ml for s in self.seqs)
        if self.cap is None:
            self.cap = out_len
        self.status, self.want = lz_decode(self.seqs, self.tail, self.cap, self.dict_bytes, n_lit_decl, lits)
        self.checksum = checksum
        self.raw = block_bytes(1 if kind == "glo" else 2, self.payload, checksum)


def block_bytes(btype, payload, checksum):
    h = bytearray(struct.pack("<BBBI", btype, 0, 0, len(payload)) + b"\0")
    h[7] = _oracle().lib.zxo_hash8(bytes(h))
    out = bytes(h) + payload
    if checksum:
        out += struct.pack("<I", _oracle().lib.zxo_checksum(payload, len(payload)))
    return out


def frame(blocks, block_size, checksum=False, dict_id=0, total=None):
    """a frame of `blocks` (payload bytes, btype) with the header, EOF block and footer; the global hash is the
    reference's rotate-and-xor of the block checksums"""
    orc = _oracle().lib
    log2 = block_size.bit_length() - 1
    assert 1 << log2 == block_size
    hdr = bytearray(struct.pack("<IBBB", 0x9CB02EF5, 8, log2, (0x80 if checksum else 0) | (0x40 if dict_id else 0)))
    hdr += struct.pack("<I", dict_id) + bytes(5)
    struct.pack_into("<H", hdr, 14, orc.zxo_hash16(bytes(hdr)))
    out = bytearray(hdr)
    ghash = 0
    for payload, btype in blocks:
        out += block_bytes(btype, payload, checksum)
        if checksum:
            c = orc.zxo_checksum(payload, len(payload))
            ghash = (((ghash << 1) | (ghash >> 31)) & 0xFFFFFFFF) ^ c
    out += block_bytes(255, b"", False)
    out += struct.pack("<QI", total, ghash if checksum else 0)
    return bytes(out)


def job_table(blocks, src_res=0, dst_res=0, gap=0):
    """(source bytes, list of (src_off, dst_off, src_len, dst_cap)) with every block's src_off = src_res and dst_off =
    dst_res mod 16 and `gap` spare bytes between neighbours"""
    src, jobs, s, d = bytearray(), [], 0, 0
    for b in blocks:
        s = (s + 15 - src_res) // 16 * 16 + src_res if s % 16 != src_res else s
        d = (d + 15 - dst_res) // 16 * 16 + dst_res if d % 16 != dst_res else d
        src += bytes(s - len(src))
        src += b.raw
        jobs.append((s, d, len(b.raw), b.cap))
        s = len(src) + gap
        d += b.cap + gap
    return bytes(src), jobs, d


def fill_seqs(n, rng, off_lo=64, off_hi=1024, ml=60, ll=4, start=0):
    """sequences that add exactly n output bytes (n = 0 or n >= ll + 5, ll >= 1 when start == 0) after `start` bytes of
    output: each `ll` random literals then a match of about `ml` bytes from a random distance in [off_lo, off_hi]
    that the output so far covers"""
    seqs, made = [], 0
    while made < n:
        left = n - made
        if left < ll + MIN_MATCH:
            seqs[-1].ml += left
            break
        m = left - ll if left - ll < ml + ll + MIN_MATCH else ml
        pos = start + made + ll
        off = int(rng.integers(min(off_lo, pos), min(off_hi, pos) + 1))
        seqs.append(Seq(rng.bytes(ll), m, off))
        made += ll + m
    return seqs


def out_len(seqs):
    return sum(len(s.lit) + s.ml for s in seqs)
