"""Shared ctypes driver for the push-streaming tests (tests/test_pstream_host.py, tests/test_pstream_gpu.py).

drive(lib, make, schedule) runs one stream through a schedule of (in_chunk, out_capacity) steps and the end / drain
loop, and returns the transcript of every call: (return value, in.pos, out.pos, produced bytes, finished, in_size
hint, out_size hint).  The tests drive the product and the reference with the same schedule and compare transcripts,
which pins consumption and error timing as well as the bytes.
"""
import ctypes as C


class InBuf(C.Structure):
    _fields_ = [("src", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


class OutBuf(C.Structure):
    _fields_ = [("dst", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


def bind(L):
    """Sets the pstream prototypes on a CDLL exporting the reference C ABI; returns it."""
    if getattr(L, "_pstream_bound", False):
        return L
    vp = C.c_void_p
    for k in ("c", "d"):
        getattr(L, f"zxc_{k}stream_create").restype = vp
        getattr(L, f"zxc_{k}stream_create").argtypes = [vp]
        getattr(L, f"zxc_{k}stream_free").restype = None
        getattr(L, f"zxc_{k}stream_free").argtypes = [vp]
        for h in ("in_size", "out_size"):
            getattr(L, f"zxc_{k}stream_{h}").restype = C.c_size_t
            getattr(L, f"zxc_{k}stream_{h}").argtypes = [vp]
    L.zxc_cstream_compress.restype = C.c_int64
    L.zxc_cstream_compress.argtypes = [vp, C.POINTER(OutBuf), C.POINTER(InBuf)]
    L.zxc_cstream_end.restype = C.c_int64
    L.zxc_cstream_end.argtypes = [vp, C.POINTER(OutBuf)]
    L.zxc_dstream_decompress.restype = C.c_int64
    L.zxc_dstream_decompress.argtypes = [vp, C.POINTER(OutBuf), C.POINTER(InBuf)]
    L.zxc_dstream_finished.restype = C.c_int
    L.zxc_dstream_finished.argtypes = [vp]
    L._pstream_bound = True
    return L


UNLIMITED = 1 << 62  # an out capacity meaning "as much as the stream can produce"


class Stream:
    """One cstream ("c") or dstream ("d") of a library, with the call helpers the driver uses."""

    def __init__(self, L, kind, opts):
        self.L, self.kind = bind(L), kind
        self.h = getattr(L, f"zxc_{kind}stream_create")(C.byref(opts) if opts is not None else None)
        self.bufs = {}

    def close(self):
        if self.h:
            getattr(self.L, f"zxc_{self.kind}stream_free")(self.h)
            self.h = None

    def hints(self):
        return (getattr(self.L, f"zxc_{self.kind}stream_in_size")(self.h),
                getattr(self.L, f"zxc_{self.kind}stream_out_size")(self.h))

    def finished(self):
        return self.L.zxc_dstream_finished(self.h) if self.kind == "d" else 0

    def call(self, inbuf, cap, fin=False):
        """One call with a fresh out buffer of `cap` bytes; returns (ret, out_pos, produced bytes)."""
        out = self.bufs.get(cap)
        if out is None:
            out = self.bufs[cap] = (C.c_uint8 * max(cap, 1))()
        ob = OutBuf(C.cast(out, C.c_void_p), cap, 0)
        if self.kind == "c":
            r = self.L.zxc_cstream_end(self.h, C.byref(ob)) if fin else \
                self.L.zxc_cstream_compress(self.h, C.byref(ob), C.byref(inbuf))
        else:
            r = self.L.zxc_dstream_decompress(self.h, C.byref(ob), C.byref(inbuf))
        return r, ob.pos, C.string_at(C.addressof(out), ob.pos)


def _cap(stream, cap, remaining_hint):
    if cap == "out_size":
        return stream.hints()[1]
    if cap == UNLIMITED:
        return remaining_hint
    return cap


def drive(L, make, schedule, end_cap=None, max_calls=1 << 20):
    """make = ("c", CompressOpts) or ("d", DecompressOpts); schedule = [(bytes, out_capacity), ...], where an out
    capacity is an int, "out_size" (the stream's hint at the time of the call) or UNLIMITED.  Each step is one call,
    repeated on the rest of its chunk (fresh out buffer each time) while the call makes progress and leaves input or
    output pending; then the stream is finished: cstream_end calls, or empty-input dstream calls, with end_cap
    (default: the last step's capacity) until nothing is pending.  Returns the transcript."""
    kind, opts = make
    s = Stream(L, kind, opts)
    if not s.h:
        return None
    t = []
    big = sum(len(c) for c, _ in schedule) * 8 + (1 << 20)
    try:
        def record(r, inb, pos, data):
            t.append((r, inb.pos if inb is not None else None, pos, data, s.finished()) + tuple(s.hints()))

        for chunk, cap in schedule:
            buf = C.create_string_buffer(bytes(chunk), max(len(chunk), 1))
            inb = InBuf(C.cast(buf, C.c_void_p), len(chunk), 0)
            while len(t) < max_calls:
                before = inb.pos
                r, pos, data = s.call(inb, _cap(s, cap, big))
                record(r, inb, pos, data)
                if r < 0:
                    return t
                if kind == "c":
                    if r == 0 and inb.pos == inb.size:
                        break
                else:
                    if s.finished() or (inb.pos == before and pos == 0):
                        break
                    if inb.pos == inb.size and pos < _cap(s, cap, big):
                        break
        ec = end_cap if end_cap is not None else (schedule[-1][1] if schedule else UNLIMITED)
        empty = InBuf(None, 0, 0)
        while len(t) < max_calls:
            r, pos, data = s.call(empty, _cap(s, ec, big), fin=(kind == "c"))
            record(r, empty if kind == "d" else None, pos, data)
            if r <= 0:
                break
        return t
    finally:
        s.close()


def joined(transcript):
    """All bytes a transcript produced, in order."""
    return b"".join(x[3] for x in transcript)


def chunks(data, sizes):
    """Cuts data into consecutive pieces of the given sizes (cycled); the last piece takes the rest."""
    out, i, k = [], 0, 0
    while i < len(data):
        n = sizes[k % len(sizes)]
        out.append(data[i:i + n])
        i += n
        k += 1
    return out
