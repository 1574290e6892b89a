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
that cannot be emitted.

GLO literal and token sections may also be PivCo Huffman sections (docs/FORMAT.md, PivCo): a 128-byte table of code
lengths, then one run per emitting tree node in BFS order.  pivco_runs() writes them from 256 code lengths and a symbol
string; pivco_decode() reads them back by walking the explicit code tree one branch at a time, with no rank tables.
A caller may also hand in the table and the run bytes as they are, to build malformed sections.

The header hashes and block checksums come from the test oracle (oracle/libzxc_oracle.so)."""
import struct

import numpy as np

MIN_MATCH = 5
SLACK = 32
OVERFLOW, BAD_OFFSET = -10, -9
DST_TOO_SMALL, CORRUPT, DICT_REQUIRED = -2, -8, -15
HUF_MAXLEN = 11

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


# ------------------------------------------------------------------------------------------------------------------
# PivCo sections
# ------------------------------------------------------------------------------------------------------------------
def pack_lengths(lens):
    """the 128-byte table: symbol 2i in the low nibble of byte i, 2i + 1 in the high one"""
    lens = list(lens) + [0] * (256 - len(lens))
    assert all(0 <= v <= 15 for v in lens)
    return bytes(lens[2 * i] | (lens[2 * i + 1] << 4) for i in range(128))


def unpack_lengths(table):
    return [(table[s >> 1] >> (4 * (s & 1))) & 15 for s in range(256)]


class PivcoTree:
    """The explicit canonical code tree of 256 code lengths.  A node is (depth, prefix); `kind[node]` is "leaf",
    "bitmap", a flat-root depth D >= 2 (every leaf below it sits D levels down) or "covered" (below a flat root).
    `error` is set, and nothing else, when the lengths do not make a code the format accepts."""

    def __init__(self, lens):
        self.lens = list(lens)
        self.error = None
        present = [s for s in range(256) if self.lens[s]]
        if any(v > HUF_MAXLEN for v in self.lens) or not present:
            self.error = CORRUPT
            return
        kraft = sum(1 << (HUF_MAXLEN - self.lens[s]) for s in present)
        self.single = len(present) == 1 and self.lens[present[0]] == 1
        if kraft != 1 << HUF_MAXLEN and not self.single:
            self.error = CORRUPT
            return
        self.code = [0] * 256
        code = 0
        prev = 0
        for s in sorted(present, key=lambda s: (self.lens[s], s)):  # canonical: by (length, symbol)
            code <<= self.lens[s] - prev
            prev = self.lens[s]
            self.code[s] = code
            code += 1
        self.leaf = {(self.lens[s], self.code[s]): s for s in present}
        internal = set()
        for d, c in self.leaf:
            for k in range(d):
                internal.add((k, c >> (d - k)))
        self.internal = internal
        self.kind = {}
        for node in sorted(internal | set(self.leaf)):  # BFS: by depth, then prefix
            d, v = node
            if node in self.leaf:
                self.kind[node] = "leaf"
            if d and self.kind.get((d - 1, v >> 1)) in ("covered",) + tuple(range(2, HUF_MAXLEN + 1)):
                self.kind[node] = "covered"
            elif node in internal:
                u = self._uniform(node)
                self.kind[node] = u if u >= 2 else "bitmap"
        self.bfs = sorted(internal | set(self.leaf))

    def _uniform(self, node):
        d, v = node
        if node in self.leaf:
            return 0
        kids = [(d + 1, 2 * v), (d + 1, 2 * v + 1)]
        if any(k not in self.leaf and k not in self.internal for k in kids):
            return -1
        a, b = self._uniform(kids[0]), self._uniform(kids[1])
        return a + 1 if a == b and a >= 0 else -1

    def emitting(self):
        return [n for n in self.bfs if self.kind[n] not in ("leaf", "covered")]

    def flat_depths(self):
        return sorted({self.kind[n] for n in self.emitting() if self.kind[n] != "bitmap"})


def _group(keys, nodes):
    """for each node value in `nodes`: the positions of `keys` equal to it, in order"""
    order = np.argsort(keys, kind="stable")
    sk = keys[order]
    lo = np.searchsorted(sk, nodes, "left")
    hi = np.searchsorted(sk, nodes, "right")
    return [order[a:b] for a, b in zip(lo, hi)]


def pivco_runs(lens, syms, sizes=None):
    """the run area of `syms` under the code of `lens`, node by node in BFS order: a bitmap node writes one bit per
    symbol through it (1 = right), a flat root of depth D the symbol's D-bit path (first step in bit 0), both packed
    LSB-first; leaves and covered nodes write nothing.  `sizes`, a list, receives (node, kind, count, bytes) per run."""
    t = PivcoTree(lens)
    assert t.error is None, "the lengths do not make a code"
    syms = np.frombuffer(bytes(syms), np.uint8)
    assert all(t.lens[s] for s in set(syms.tolist())), "a symbol without a code"
    L = np.array(t.lens, np.int64)[syms]
    Cd = np.array(t.code, np.int64)[syms]
    out = bytearray()
    emit = t.emitting()
    for d in range(HUF_MAXLEN + 1):
        level = [n for n in emit if n[0] == d]
        if not level:
            continue
        act = np.nonzero(L > d)[0]
        groups = _group(Cd[act] >> (L[act] - d), np.array([v for _, v in level], np.int64))
        for (_, v), g in zip(level, groups):
            idx = act[g]
            kind = t.kind[(d, v)]
            if kind == "bitmap":
                bits = (Cd[idx] >> (L[idx] - d - 1)) & 1
            else:
                bits = np.stack([(Cd[idx] >> (L[idx] - d - 1 - j)) & 1 for j in range(kind)], 1).reshape(-1)
            run = np.packbits(bits.astype(np.uint8), bitorder="little").tobytes()
            if sizes is not None:
                sizes.append(((d, v), kind, idx.size, len(run)))
            out += run
    return bytes(out)


def pivco_section(lens, syms):
    """the whole section: the 128-byte table, then the runs"""
    return pack_lengths(lens) + pivco_runs(lens, syms)


def pivco_decode(table, runs, n):
    """(status, bytes) of n symbols read from `runs` under the 128-byte `table`: the explicit tree walked one branch at
    a time, every node's run consumed in order by the symbols that pass through it.  Verdicts are the reference's:
    CORRUPT for a bad table, an empty section, a run area too short, or a symbol routed to a missing child."""
    t = PivcoTree(unpack_lengths(table))
    if t.error is not None or n == 0:
        return CORRUPT, b""
    runs = np.frombuffer(bytes(runs), np.uint8)
    out = np.zeros(n, np.uint8)
    at = np.zeros(n, np.int64)  # prefix of the node each unresolved symbol sits at
    live = np.arange(n)
    pos = 0
    for d in range(HUF_MAXLEN + 1):
        level = [nd for nd in t.emitting() if nd[0] == d]
        if not level or not live.size:
            continue
        groups = _group(at[live], np.array([v for _, v in level], np.int64))
        nxt = []
        for (_, v), g in zip(level, groups):
            idx = live[g]
            c = idx.size
            kind = t.kind[(d, v)]
            nbytes = (c * (1 if kind == "bitmap" else kind) + 7) >> 3
            if runs.size - pos < nbytes:
                return CORRUPT, b""
            bits = np.unpackbits(runs[pos:pos + nbytes], bitorder="little").astype(np.int64)
            pos += nbytes
            if kind == "bitmap":
                b = bits[:c]
                for bit in (0, 1):
                    child = (d + 1, 2 * v + bit)
                    sel = idx[b == bit]
                    if child in t.leaf:
                        out[sel] = t.leaf[child]
                    elif child in t.internal:
                        at[sel] = child[1]
                        nxt.append(sel)
                    elif sel.size:
                        return CORRUPT, b""
            else:
                paths = bits[:c * kind].reshape(c, kind)
                leafv = v
                for j in range(kind):
                    leafv = (leafv << 1) | paths[:, j]
                lut = np.array([t.leaf.get((d + kind, x), 0) for x in range(v << kind, (v + 1) << kind)], np.uint8)
                out[idx] = lut[leafv - (v << kind)]
        live = np.sort(np.concatenate(nxt)) if nxt else np.zeros(0, np.int64)
    return n, out.tobytes()


class Huf:
    """How a GLO section is Huffman-coded.  `lens`: 256 code lengths (the writer builds the runs); `table`: 128 table
    bytes as they are (default: packed `lens`); `runs`: run bytes as they are (default: written from the symbols);
    `extra`: bytes after the runs inside the section; `comp`: the section size the header declares (default: its
    length)."""

    def __init__(self, lens=None, table=None, runs=None, extra=b"", comp=None):
        self.lens, self.table, self.runs, self.extra, self.comp = lens, table, runs, bytes(extra), comp

    def section(self, syms, with_table=True, written=None):
        """(section bytes, table, run area); `written` receives (lengths, symbols, table + runs) when the writer made
        the whole section from the lengths"""
        table = self.table if self.table is not None else pack_lengths(self.lens)
        runs = self.runs if self.runs is not None else pivco_runs(self.lens, syms)
        if written is not None and self.table is None and self.runs is None and not self.extra and self.comp is None:
            written.append((self.lens, bytes(syms), table + runs))
        sec = (table if with_table else b"") + runs + self.extra
        return sec, table, runs + self.extra


class Block:
    """A GLO or GHI block: `raw` is the on-disk block (8-byte header + payload [+ checksum]), `want` the status and
    bytes it decodes to with `dict_bytes` into `cap` bytes.

    GLO literals may be Huffman-coded (enc_lit = 2 with `lit_huf`, a Huf; enc_lit = 3 with the table `dict_huf` that
    comes with the dictionary, and `lit_huf` giving its lengths or runs) and so may the tokens (enc_tok = 2 with
    `tok_huf`).  `block_size` is the frame's block size: it bounds the Huffman-coded token count (block_size / 5 + 16,
    the reference's token buffer) and the decoded literal count."""

    def __init__(self, seqs, tail=b"", kind="glo", enc_off=0, enc_lit=0, rle_plan=None, dict_bytes=b"", cap=None,
                 extra_pad=0, checksum=False, n_lit=None, lit_huf=None, tok_huf=None, dict_huf=None, block_size=None,
                 n_seq=None):
        self.seqs, self.tail, self.kind = list(seqs), bytes(tail), kind
        self.dict_bytes = bytes(dict_bytes)
        self.dict_huf = dict_huf
        self.written_sections = []  # (lengths, symbols, table + runs) of the sections the writer made
        self.decoded = []  # (lengths, symbols) of the sections that decode
        self.pivco_verdict = False  # the verdict is the section decoder's
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
            lit_runs = tok_runs = None
            if enc_lit == 1:
                lsec, self.rle_plan = rle_encode(lits, rle_plan)
                desc = struct.pack("<I", len(lsec))
            elif enc_lit in (2, 3):
                lsec, _, lit_runs = lit_huf.section(lits, with_table=enc_lit == 2, written=self.written_sections)
                desc = struct.pack("<I", len(lsec) if lit_huf.comp is None else lit_huf.comp)
            else:
                lsec, desc = lits, b""
            enc_tok = 0
            if tok_huf is not None:
                enc_tok = 2
                tsec, tok_table, tok_runs = tok_huf.section(tok, written=self.written_sections)
                desc += struct.pack("<I", len(tsec) if tok_huf.comp is None else tok_huf.comp)
                tok = tsec
            body = tok + offs + ext
            hdr = struct.pack("<IIBBBB", len(self.seqs) if n_seq is None else n_seq, n_lit_decl, enc_lit, enc_tok, 0,
                              enc_off) + desc
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
        self.block_size = block_size or max(4096, 1 << (max(self.cap, 1) - 1).bit_length())
        self.status, self.want = None, b""
        if kind == "glo" and (enc_lit >= 2 or enc_tok == 2):
            self.status = self._huf_verdict(enc_lit, enc_tok, n_lit_decl, lits, lit_huf, tok_huf, lit_runs, tok_runs,
                                            len(hdr), len(lsec), tok_huf and len(tok), n_seq)
        if self.status is None:
            self.status, self.want = lz_decode(self.seqs, self.tail, self.cap, self.dict_bytes, n_lit_decl, lits)
        self.checksum = checksum
        self.raw = block_bytes(1 if kind == "glo" else 2, self.payload, checksum)


    def _huf_verdict(self, enc_lit, enc_tok, n_lit, lits, lit_huf, tok_huf, lit_runs, tok_runs, hdr_len, lsec_len,
                     tsec_len, n_seq):
        """the reference's section checks in its order (zxc_decompress.c:859-1023): a verdict, or None when the
        sections decode to the literals and tokens the sequences say"""
        avail = len(self.payload) - hdr_len
        n_seq = len(self.seqs) if n_seq is None else n_seq
        lit_comp = lsec_len if enc_lit < 2 or lit_huf.comp is None else lit_huf.comp
        if enc_lit >= 2:
            if lit_comp > avail:
                return CORRUPT
            if n_lit:
                if n_lit > self.cap:
                    return DST_TOO_SMALL
                if enc_lit == 3 and self.dict_huf is None:
                    return DICT_REQUIRED
                if n_lit > self.block_size:
                    return CORRUPT
                if enc_lit == 2 and lit_comp < 128:
                    return CORRUPT
                # a section declared shorter than written ends where the header says
                table = self.dict_huf if enc_lit == 3 else self.payload[hdr_len:hdr_len + 128]
                rlen = lit_comp - (128 if enc_lit == 2 else 0)
                st, got = pivco_decode(table, lit_runs[:rlen], n_lit)
                if st < 0:
                    self.pivco_verdict = True
                    return st
                self.decoded.append((unpack_lengths(table), got))
                assert got == lits, "a malformed literal run that still decodes: give the case its own expectation"
        tok_comp = n_seq if enc_tok != 2 else (tsec_len if tok_huf.comp is None else tok_huf.comp)
        if lit_comp + tok_comp + n_seq * (1 if self.payload[11] else 2) > avail or avail - lit_comp < SLACK:
            return CORRUPT
        if enc_tok == 2:
            if n_seq == 0 or n_seq > self.block_size // MIN_MATCH + 16 or tok_comp < 128:
                return CORRUPT
            table = self.payload[hdr_len + lit_comp:hdr_len + lit_comp + 128]
            st, got = pivco_decode(table, tok_runs[:tok_comp - 128], n_seq)
            if st < 0:
                self.pivco_verdict = True
                return st
            self.decoded.append((unpack_lengths(table), got))
            assert got[:len(self.seqs)] == bytes((min(len(s.lit), 15) << 4) | min(s.ml - MIN_MATCH, 15) for s in self.seqs)
        return None


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
