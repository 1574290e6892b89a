"""ctypes bindings used by the tests and bench: the product library (libzxc.so.4),
the test-only oracle (oracle/libzxc_oracle.so) and, when present, the unmodified
reference compiled into oracle/_ref/libzxc_ref.so.

Product and reference share the reference's C ABI (include/zxc_buffer.h,
zxc_seekable.h, zxc_dict.h), so one binder serves both.
"""
import ctypes as C
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRODUCT_SO = os.environ.get("ZXC_B200_LIB") or os.path.join(ROOT, "zxc_b200", "lib", "libzxc.so.4")  # env: A/B builds
ORACLE_SO = os.path.join(ROOT, "oracle", "libzxc_oracle.so")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libzxc_ref.so")

ERR = {
    0: "OK", -1: "MEMORY", -2: "DST_TOO_SMALL", -3: "SRC_TOO_SMALL", -4: "BAD_MAGIC",
    -5: "BAD_VERSION", -6: "BAD_HEADER", -7: "BAD_CHECKSUM", -8: "CORRUPT_DATA", -9: "BAD_OFFSET",
    -10: "OVERFLOW", -11: "IO", -12: "NULL_INPUT", -13: "BAD_BLOCK_TYPE", -14: "BAD_BLOCK_SIZE",
    -15: "DICT_REQUIRED", -16: "DICT_MISMATCH", -17: "DICT_TOO_LARGE", -18: "BAD_LEVEL",
    -100: "B200_NO_DEVICE", -101: "B200_CUDA", -102: "B200_UNSUPPORTED",
}


class CompressOpts(C.Structure):
    _fields_ = [("n_threads", C.c_int), ("level", C.c_int), ("block_size", C.c_size_t),
                ("checksum_enabled", C.c_int), ("seekable", C.c_int), ("dict", C.c_void_p),
                ("dict_size", C.c_size_t), ("dict_huf", C.c_void_p), ("progress_cb", C.c_void_p),
                ("user_data", C.c_void_p)]


class DecompressOpts(C.Structure):
    _fields_ = [("n_threads", C.c_int), ("checksum_enabled", C.c_int), ("dict", C.c_void_p),
                ("dict_size", C.c_size_t), ("dict_huf", C.c_void_p), ("progress_cb", C.c_void_p),
                ("user_data", C.c_void_p)]


def _buf(b):
    """bytes/bytearray/numpy -> (ctypes pointer-ish, length, keepalive)"""
    import numpy as np
    if isinstance(b, np.ndarray):
        a = np.ascontiguousarray(b).view(np.uint8).reshape(-1)
        return a.ctypes.data_as(C.c_void_p), a.size, a
    if isinstance(b, (bytes, bytearray, memoryview)):
        b = bytes(b)
        return C.cast(C.c_char_p(b), C.c_void_p), len(b), b
    raise TypeError(type(b))


class ZxcLib:
    """Binder for a library exporting the reference C ABI."""

    def __init__(self, path):
        self.path = path
        self.lib = L = C.CDLL(path)
        L.zxc_compress_bound.restype = C.c_uint64
        L.zxc_compress_bound.argtypes = [C.c_size_t]
        L.zxc_compress.restype = C.c_int64
        L.zxc_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
        L.zxc_decompress.restype = C.c_int64
        L.zxc_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
        L.zxc_get_decompressed_size.restype = C.c_uint64
        L.zxc_get_decompressed_size.argtypes = [C.c_void_p, C.c_size_t]
        L.zxc_get_dict_id.restype = C.c_uint32
        L.zxc_get_dict_id.argtypes = [C.c_void_p, C.c_size_t]
        L.zxc_dict_id.restype = C.c_uint32
        L.zxc_dict_id.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
        L.zxc_seekable_open.restype = C.c_void_p
        L.zxc_seekable_open.argtypes = [C.c_void_p, C.c_size_t]
        L.zxc_seekable_free.restype = None
        L.zxc_seekable_free.argtypes = [C.c_void_p]
        L.zxc_seekable_get_num_blocks.restype = C.c_uint32
        L.zxc_seekable_get_num_blocks.argtypes = [C.c_void_p]
        L.zxc_seekable_get_decompressed_size.restype = C.c_uint64
        L.zxc_seekable_get_decompressed_size.argtypes = [C.c_void_p]
        L.zxc_seekable_get_block_comp_size.restype = C.c_uint32
        L.zxc_seekable_get_block_comp_size.argtypes = [C.c_void_p, C.c_uint32]
        L.zxc_seekable_get_block_decomp_size.restype = C.c_uint32
        L.zxc_seekable_get_block_decomp_size.argtypes = [C.c_void_p, C.c_uint32]
        L.zxc_seekable_decompress_range.restype = C.c_int64
        L.zxc_seekable_decompress_range.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_size_t]
        L.zxc_seekable_decompress_range_mt.restype = C.c_int64
        L.zxc_seekable_decompress_range_mt.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_size_t, C.c_int]
        L.zxc_seekable_set_dict.restype = C.c_int
        L.zxc_seekable_set_dict.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        L.zxc_dict_load.restype = C.c_int
        L.zxc_dict_load.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t),
                                    C.POINTER(C.c_void_p), C.POINTER(C.c_uint32)]
        L.zxc_error_name.restype = C.c_char_p
        L.zxc_error_name.argtypes = [C.c_int]
        L.zxc_version_string.restype = C.c_char_p
        L.zxc_compress_block_bound.restype = C.c_uint64
        L.zxc_compress_block_bound.argtypes = [C.c_size_t]
        L.zxc_decompress_block_bound.restype = C.c_uint64
        L.zxc_decompress_block_bound.argtypes = [C.c_size_t]
        L.zxc_create_dctx.restype = C.c_void_p
        L.zxc_free_dctx.argtypes = [C.c_void_p]
        L.zxc_free_dctx.restype = None
        L.zxc_create_cctx.restype = C.c_void_p
        L.zxc_create_cctx.argtypes = [C.c_void_p]
        L.zxc_free_cctx.argtypes = [C.c_void_p]
        L.zxc_free_cctx.restype = None
        for name in ("zxc_compress_block", "zxc_decompress_block", "zxc_decompress_block_safe",
                     "zxc_compress_cctx", "zxc_decompress_dctx"):
            f = getattr(L, name)
            f.restype = C.c_int64
            f.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]

    # ---- convenience wrappers -------------------------------------------------
    def compress(self, data, level=3, block_size=0, checksum=0, seekable=0, dict=None, dict_huf=None):
        import numpy as np
        p, n, keep = _buf(data)
        cap = int(self.lib.zxc_compress_bound(n))
        out = np.empty(cap, dtype=np.uint8)
        o = CompressOpts(level=level, block_size=block_size, checksum_enabled=checksum, seekable=seekable)
        keep2 = None
        if dict is not None:
            dp, dn, keep2 = _buf(dict)
            o.dict, o.dict_size = dp, dn
            if dict_huf is not None:
                hp, _, keep3 = _buf(dict_huf)
                o.dict_huf = hp
                keep2 = (keep2, keep3)
        r = self.lib.zxc_compress(p, n, out.ctypes.data_as(C.c_void_p), cap, C.byref(o))
        if r < 0:
            return r
        return out[:r].copy()

    def decompress(self, frame, cap=None, checksum=0, dict=None, dict_huf=None):
        """returns (code_or_size, ndarray)"""
        import numpy as np
        p, n, keep = _buf(frame)
        if cap is None:
            cap = int(self.lib.zxc_get_decompressed_size(p, n))
        out = np.empty(max(cap, 1), dtype=np.uint8)
        o = DecompressOpts(checksum_enabled=checksum)
        keep2 = None
        if dict is not None:
            dp, dn, keep2 = _buf(dict)
            o.dict, o.dict_size = dp, dn
            if dict_huf is not None:
                hp, _, keep3 = _buf(dict_huf)
                o.dict_huf = hp
                keep2 = (keep2, keep3)
        r = self.lib.zxc_decompress(p, n, out.ctypes.data_as(C.c_void_p) if cap > 0 else None, cap, C.byref(o))
        return r, (out[:r] if r > 0 else out[:0])

    def dict_load(self, zxd):
        p, n, keep = _buf(zxd)
        content, csz, huf, did = C.c_void_p(), C.c_size_t(), C.c_void_p(), C.c_uint32()
        rc = self.lib.zxc_dict_load(p, n, C.byref(content), C.byref(csz), C.byref(huf), C.byref(did))
        if rc != 0:
            return rc, None, None, 0
        base = p.value if isinstance(p, C.c_void_p) else C.cast(p, C.c_void_p).value
        raw = bytes(keep) if not isinstance(keep, bytes) else keep
        co = content.value - base
        ho = huf.value - base
        return 0, raw[co:co + csz.value], raw[ho:ho + 128], did.value


class Oracle:
    def __init__(self, path=ORACLE_SO):
        self.lib = L = C.CDLL(path)
        L.zxo_decompress.restype = C.c_int64
        L.zxo_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int,
                                     C.c_void_p, C.c_size_t, C.c_void_p]
        L.zxo_decode_block.restype = C.c_int
        L.zxo_decode_block.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                       C.c_size_t, C.c_void_p, C.c_int]
        L.zxo_decode_block_bs.restype = C.c_int
        L.zxo_decode_block_bs.argtypes = L.zxo_decode_block.argtypes + [C.c_size_t]
        L.zxo_hash8.restype = C.c_uint8
        L.zxo_hash8.argtypes = [C.c_void_p]
        L.zxo_hash16.restype = C.c_uint16
        L.zxo_hash16.argtypes = [C.c_void_p]
        L.zxo_rapidhash.restype = C.c_uint64
        L.zxo_rapidhash.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64]
        L.zxo_checksum.restype = C.c_uint32
        L.zxo_checksum.argtypes = [C.c_void_p, C.c_size_t]
        L.zxo_dict_id.restype = C.c_uint32
        L.zxo_dict_id.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
        L.zxo_seek_parse.restype = C.c_int64
        L.zxo_seek_parse.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64),
                                     C.c_void_p, C.c_size_t]
        L.zxo_frame_stats.restype = C.c_int
        L.zxo_frame_stats.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]

    def decompress(self, frame, cap, checksum=0, dict=None, dict_huf=None):
        import numpy as np
        p, n, keep = _buf(frame)
        out = np.empty(max(cap, 1), dtype=np.uint8)
        dp, dn, k2 = (None, 0, None)
        hp, k3 = None, None
        if dict is not None:
            dp, dn, k2 = _buf(dict)
            if dict_huf is not None:
                hp, _, k3 = _buf(dict_huf)
        r = self.lib.zxo_decompress(p, n, out.ctypes.data_as(C.c_void_p) if cap > 0 else None, cap, checksum,
                                    dp, dn, hp)
        return r, (out[:r] if r > 0 else out[:0])

    def dict_id(self, d, huf=None):
        dp, dn, k = _buf(d)
        hp = None
        if huf is not None:
            hp, _, k2 = _buf(huf)
        return self.lib.zxo_dict_id(dp, dn, hp)

    def stats(self, frame):
        class S(C.Structure):
            _fields_ = [(n, C.c_uint64) for n in (
                "blocks", "raw_blocks", "glo_blocks", "ghi_blocks", "sequences", "literals", "extras_bytes",
                "comp_bytes", "decoded_bytes", "ll_escapes", "ml_escapes", "off_lt32", "off_lt_ml",
                "rle_blocks", "huf_blocks", "off8_blocks", "ml_sum", "max_seq_per_block")]
        s = S()
        p, n, keep = _buf(frame)
        rc = self.lib.zxo_frame_stats(p, n, C.byref(s))
        return rc, {k: getattr(s, k) for k, _ in S._fields_}


def have_ref():
    return os.path.exists(REF_SO)


def have_product():
    return os.path.exists(PRODUCT_SO)
