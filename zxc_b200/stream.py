"""zlib-shaped push streaming over the library's zxc_cstream_* / zxc_dstream_* C ABI.

    c = compressobj(level=3, block_size=65536, checksum=True)
    frame = c.compress(part1) + c.compress(part2) + c.flush()

    d = decompressobj(checksum=True)
    data = d.decompress(frame[:1000]) + d.decompress(frame[1000:])
    d.eof, d.unused_data

The compressed stream is the frame zxc_compress writes for the same options (not seekable).  Blocks are encoded and
decoded on the GPU; a call hands every whole block it has to one kernel launch.  Errors raise ZxcError, whose `code`
is the library's negative zxc_error_t.  This module does not import torch.
"""
import ctypes as C

from . import lib as _lib


class ZxcError(RuntimeError):
    def __init__(self, code):
        self.code = int(code)
        name = _lib.zxc_error_name(self.code).decode()
        super().__init__(f"{name} ({self.code})")


class _In(C.Structure):
    _fields_ = [("src", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


class _Out(C.Structure):
    _fields_ = [("dst", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


class _CompressOpts(C.Structure):
    _fields_ = [("n_threads", C.c_int), ("level", C.c_int), ("block_size", C.c_size_t),
                ("checksum_enabled", C.c_int), ("seekable", C.c_int), ("dict", C.c_void_p),
                ("dict_size", C.c_size_t), ("dict_huf", C.c_void_p), ("progress_cb", C.c_void_p),
                ("user_data", C.c_void_p)]


class _DecompressOpts(C.Structure):
    _fields_ = [("n_threads", C.c_int), ("checksum_enabled", C.c_int), ("dict", C.c_void_p),
                ("dict_size", C.c_size_t), ("dict_huf", C.c_void_p), ("progress_cb", C.c_void_p),
                ("user_data", C.c_void_p)]


_vp = C.c_void_p
_lib.zxc_error_name.restype = C.c_char_p
_lib.zxc_error_name.argtypes = [C.c_int]
for _k in ("c", "d"):
    getattr(_lib, f"zxc_{_k}stream_create").restype = _vp
    getattr(_lib, f"zxc_{_k}stream_create").argtypes = [_vp]
    getattr(_lib, f"zxc_{_k}stream_free").restype = None
    getattr(_lib, f"zxc_{_k}stream_free").argtypes = [_vp]
    getattr(_lib, f"zxc_{_k}stream_out_size").restype = C.c_size_t
    getattr(_lib, f"zxc_{_k}stream_out_size").argtypes = [_vp]
_lib.zxc_cstream_compress.restype = C.c_int64
_lib.zxc_cstream_compress.argtypes = [_vp, C.POINTER(_Out), C.POINTER(_In)]
_lib.zxc_cstream_end.restype = C.c_int64
_lib.zxc_cstream_end.argtypes = [_vp, C.POINTER(_Out)]
_lib.zxc_dstream_decompress.restype = C.c_int64
_lib.zxc_dstream_decompress.argtypes = [_vp, C.POINTER(_Out), C.POINTER(_In)]
_lib.zxc_dstream_finished.restype = C.c_int
_lib.zxc_dstream_finished.argtypes = [_vp]

# output is collected in pieces of at least this size, so a large input is one call that batches all its blocks
_CHUNK = 64 << 20


class _Handle:
    def __init__(self, kind, opts):
        self._kind = kind
        self._h = getattr(_lib, f"zxc_{kind}stream_create")(C.byref(opts))
        if not self._h:
            raise ValueError(f"zxc_{kind}stream_create rejected the options")
        self._out = None

    def _buffer(self, hint):
        n = max(_CHUNK, hint)
        if self._out is None or len(self._out) < n:
            self._out = (C.c_uint8 * n)()
        return self._out

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            getattr(_lib, f"zxc_{self._kind}stream_free")(h)


class Compress(_Handle):
    def __init__(self, level=0, block_size=0, checksum=False):
        super().__init__("c", _CompressOpts(level=level, block_size=block_size, checksum_enabled=int(bool(checksum))))

    def _run(self, step):
        parts = []
        out = self._buffer(_lib.zxc_cstream_out_size(self._h))
        while True:
            ob = _Out(C.cast(out, C.c_void_p), len(out), 0)
            r = step(ob)
            if r < 0:
                raise ZxcError(r)
            parts.append(C.string_at(C.addressof(out), ob.pos))
            if r == 0:
                return b"".join(parts)

    def compress(self, data):
        """Feeds data; returns the compressed bytes this made available (whole blocks, and the header first)."""
        data = bytes(data)
        src = C.create_string_buffer(data, max(len(data), 1))
        ib = _In(C.cast(src, C.c_void_p), len(data), 0)
        return self._run(lambda ob: _lib.zxc_cstream_compress(self._h, C.byref(ob), C.byref(ib)))

    def flush(self):
        """Ends the stream: the last block, the EOF block and the footer.  The object is finished afterwards."""
        return self._run(lambda ob: _lib.zxc_cstream_end(self._h, C.byref(ob)))


class Decompress(_Handle):
    def __init__(self, checksum=False):
        super().__init__("d", _DecompressOpts(checksum_enabled=int(bool(checksum))))
        self.eof = False
        self.unused_data = b""

    def decompress(self, data):
        """Feeds compressed bytes; returns what they decode to.  Bytes after the stream's footer go to unused_data."""
        data = bytes(data)
        if self.eof:
            self.unused_data += data
            return b""
        src = C.create_string_buffer(data, max(len(data), 1))
        ib = _In(C.cast(src, C.c_void_p), len(data), 0)
        parts = []
        out = self._buffer(_lib.zxc_dstream_out_size(self._h))
        while True:
            ob = _Out(C.cast(out, C.c_void_p), len(out), 0)
            r = _lib.zxc_dstream_decompress(self._h, C.byref(ob), C.byref(ib))
            if r < 0:
                raise ZxcError(r)
            parts.append(C.string_at(C.addressof(out), ob.pos))
            if _lib.zxc_dstream_finished(self._h):
                self.eof = True
                self.unused_data = data[ib.pos:]
                break
            if ob.pos < ob.size:  # out not full: every byte of `data` has been taken
                break
        return b"".join(parts)


def compressobj(level=0, block_size=0, checksum=False):
    return Compress(level, block_size, checksum)


def decompressobj(checksum=False):
    return Decompress(checksum)
