"""Device-resident compress / decompress of torch CUDA tensors.

``compress`` runs zxc_b200_compress_device: the frame is encoded and assembled in HBM on a CUDA stream, with no copy
through the host.  ``decompress`` decodes such a frame with zxc_b200_decode_blocks from the decode plan the
compress call emitted.  ``decompress_frame`` decodes any frame held in a uint8 CUDA tensor with
zxc_b200_decompress_device, which plans, decodes and checks it on the device.  ``SeekableFrame`` decodes byte ranges of
a seekable frame in HBM with zxc_b200_seekable_device_decompress_ranges.  ``decompress_frames`` decodes many frames
in one zxc_b200_decompress_device_batch call, and ``compress_frames`` compresses many tensors into one frame each in
one zxc_b200_compress_device_batch call.  ``decompress_inplace`` decodes a frame that lies flush-right in a CUDA buffer
into the same buffer with zxc_b200_decompress_inplace_device, and ``load_frame`` uses it to bring a frame from the
host into HBM and expand it there with no second buffer.  ``compress_blocks`` and ``decompress_blocks`` are the block
API in HBM: many frameless blocks per zxc_b200_compress_blocks_device / zxc_b200_decompress_blocks_device call.
``DeviceDict`` prepares a dictionary in HBM once; passed as ``dict`` to those helpers it makes them call the _using_dict
entry points, which stage nothing per call.  Kept apart from ``zxc_b200`` so that importing the package does not
import torch.
"""
import ctypes as C
import warnings
from dataclasses import dataclass

import torch

from . import lib

BLOCK_SIZE_DEFAULT = 512 * 1024
JOB_BYTES = 24  # zxc_b200_job_t


class _Opts(C.Structure):  # zxc_compress_opts_t (include/zxc_opts.h)
    _fields_ = [("n_threads", C.c_int), ("level", C.c_int), ("block_size", C.c_size_t),
                ("checksum_enabled", C.c_int), ("seekable", C.c_int), ("dict", C.c_void_p),
                ("dict_size", C.c_size_t), ("dict_huf", C.c_void_p), ("progress_cb", C.c_void_p),
                ("user_data", C.c_void_p)]


lib.zxc_compress_bound.restype = C.c_uint64
lib.zxc_compress_bound.argtypes = [C.c_size_t]
lib.zxc_error_name.restype = C.c_char_p
lib.zxc_error_name.argtypes = [C.c_int]
lib.zxc_b200_encode_scratch_size.restype = C.c_size_t
lib.zxc_b200_encode_scratch_size.argtypes = [C.c_uint64, C.c_void_p]
lib.zxc_b200_compress_device.restype = C.c_int
lib.zxc_b200_compress_device.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                         C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
lib.zxc_b200_decode_scratch_size.restype = C.c_size_t
lib.zxc_b200_decode_scratch_size.argtypes = [C.c_uint32]
lib.zxc_b200_decode_blocks.restype = C.c_int
lib.zxc_b200_decode_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                       C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_int,
                                       C.c_void_p]
lib.zxc_b200_decompress_device_scratch_size.restype = C.c_size_t
lib.zxc_b200_decompress_device_scratch_size.argtypes = [C.c_uint64, C.c_uint32]
lib.zxc_b200_decompress_device.restype = C.c_int
lib.zxc_b200_decompress_device.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                           C.c_size_t, C.c_void_p, C.c_void_p]
lib.zxc_b200_reduce_status.restype = C.c_int64
lib.zxc_b200_reduce_status.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]


class _DOpts(C.Structure):  # zxc_decompress_opts_t (include/zxc_opts.h)
    _fields_ = [("n_threads", C.c_int), ("checksum_enabled", C.c_int), ("dict", C.c_void_p),
                ("dict_size", C.c_size_t), ("dict_huf", C.c_void_p), ("progress_cb", C.c_void_p),
                ("user_data", C.c_void_p)]


class ZxcError(RuntimeError):
    def __init__(self, code, what):
        super().__init__(f"{what}: {lib.zxc_error_name(int(code)).decode()} ({int(code)})")
        self.code = int(code)


lib.zxc_b200_dict_device_create.restype = C.c_void_p
lib.zxc_b200_dict_device_create.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int), C.c_void_p]
lib.zxc_b200_dict_device_id.restype = C.c_uint32
lib.zxc_b200_dict_device_id.argtypes = [C.c_void_p]
lib.zxc_b200_dict_device_size.restype = C.c_size_t
lib.zxc_b200_dict_device_size.argtypes = [C.c_void_p]
lib.zxc_b200_dict_device_free.restype = None
lib.zxc_b200_dict_device_free.argtypes = [C.c_void_p]


class DeviceDict:
    """A dictionary prepared once in HBM (zxc_b200_dict_device_create) on the current CUDA device, to which it is
    bound.  Pass it as `dict` to the helpers below: they then call the _using_dict entry points, which stage nothing
    per call.  The host bytes are kept (.dict, .dict_huf), so a DeviceFrame made with it can still be decoded by
    `decompress`.  Raises ZxcError with zxc_b200_dict_device_create's code when it returns NULL."""

    def __init__(self, dict, dict_huf=None, stream=None):
        self._h = None  # before any check: __del__ runs on a half-made object too
        self.dict = bytes(dict)
        self.dict_huf = bytes(dict_huf) if dict_huf is not None else None
        self.device = torch.device("cuda", torch.cuda.current_device())
        err = C.c_int(0)
        with torch.cuda.device(self.device):
            stream = stream or torch.cuda.current_stream(self.device)
            h = lib.zxc_b200_dict_device_create(self.dict, len(self.dict), self.dict_huf, C.byref(err),
                                                stream.cuda_stream)
        if not h:
            raise ZxcError(err.value, "zxc_b200_dict_device_create")
        self._h = h

    @property
    def id(self):
        return int(lib.zxc_b200_dict_device_id(self.handle))

    @property
    def size(self):
        return int(lib.zxc_b200_dict_device_size(self.handle))

    @property
    def handle(self):
        if self._h is None:
            raise ValueError("DeviceDict is closed")
        return self._h

    def close(self):
        """Frees the device copy (after the work in flight on its device); later use raises ValueError."""
        if self._h is not None:
            lib.zxc_b200_dict_device_free(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        self.close()


def _dict_opts(o, dict, dict_huf):
    """Puts host dictionary bytes into the options o; returns (the bytes to keep alive, None).  For a DeviceDict, leaves
    o without a dictionary and returns ([], the DeviceDict)."""
    if isinstance(dict, DeviceDict):
        if dict_huf is not None:
            raise ValueError("dict_huf goes into DeviceDict(dict, dict_huf), not beside it")
        return [], dict
    keep = []
    if dict is not None:
        d = bytes(dict)
        keep.append(d)
        o.dict, o.dict_size = C.cast(C.c_char_p(d), C.c_void_p), len(d)
        if dict_huf is not None:
            h = bytes(dict_huf)
            keep.append(h)
            o.dict_huf = C.cast(C.c_char_p(h), C.c_void_p)
    return keep, None


def _call(name, dd, head, tail):
    """lib.name(*head, *tail), or with a DeviceDict its _using_dict variant, which takes the handle between the two"""
    if dd is None:
        return getattr(lib, name)(*head, *tail)
    return getattr(lib, name + "_using_dict")(*head, dd.handle, *tail)


@dataclass
class DeviceFrame:
    frame: torch.Tensor  # uint8, the complete frame (a view of the compress buffer, trimmed to the frame size)
    jobs: torch.Tensor  # uint8, n_blocks zxc_b200_job_t: the frame's decode plan
    block_size: int
    decoded_size: int
    checksum: bool
    dict: bytes = None  # the dictionary the frame needs (host bytes), or None
    dict_huf: bytes = None

    @property
    def n_blocks(self):
        return self.jobs.numel() // JOB_BYTES


def _bytes_view(t):
    if not t.is_cuda:
        raise ValueError("src must be a CUDA tensor")
    if not t.is_contiguous():
        raise ValueError("src must be contiguous")
    return t.reshape(-1).view(torch.uint8)


def compress(src, *, level=0, block_size=0, checksum=False, seekable=False, dict=None, dict_huf=None, stream=None):
    """Compress a contiguous CUDA tensor (its bytes) into a ZXC frame on its device; returns a DeviceFrame.

    Runs on `stream` (default: torch's current stream of src's device) and synchronises it once to read the frame
    size.  The frame equals what zxc_compress returns for the same bytes and options.  dict / dict_huf are host bytes,
    or dict is a DeviceDict (zxc_b200_compress_device_using_dict: nothing is staged)."""
    b = _bytes_view(src)
    n = b.numel()
    bs = block_size or BLOCK_SIZE_DEFAULT
    o = _Opts(level=level, block_size=block_size, checksum_enabled=int(bool(checksum)), seekable=int(bool(seekable)))
    keep, dd = _dict_opts(o, dict, dict_huf)
    with torch.cuda.device(b.device):
        stream = stream or torch.cuda.current_stream(b.device)
        with torch.cuda.stream(stream):
            scratch_size = int(lib.zxc_b200_encode_scratch_size(n, C.byref(o)))
            if scratch_size == 0:
                raise ValueError("zxc_b200_encode_scratch_size: invalid options (level, block_size, dict) or no device")
            cap = int(lib.zxc_compress_bound(n))
            dst = torch.empty(cap, dtype=torch.uint8, device=b.device)
            scratch = torch.empty(scratch_size, dtype=torch.uint8, device=b.device)
            result = torch.empty(1, dtype=torch.int64, device=b.device)
            n_blocks = (n + bs - 1) // bs
            jobs = torch.empty(max(n_blocks, 1) * JOB_BYTES, dtype=torch.uint8, device=b.device)[: n_blocks * JOB_BYTES]
            rc = _call("zxc_b200_compress_device", dd, (b.data_ptr() if n else None, n, dst.data_ptr(), cap, C.byref(o)),
                       (scratch.data_ptr(), scratch_size, result.data_ptr(), jobs.data_ptr() if n_blocks else None,
                        stream.cuda_stream))
            if rc != 0:
                raise ZxcError(rc, "zxc_b200_compress_device")
            stream.synchronize()
            size = int(result.item())
    if size < 0:
        raise ZxcError(size, "zxc_b200_compress_device")
    if dd is not None:  # the handle keeps its host bytes, so decompress can stage them
        return DeviceFrame(dst[:size], jobs, bs, n, bool(checksum), dd.dict, dd.dict_huf)
    return DeviceFrame(dst[:size], jobs, bs, n, bool(checksum), keep[0] if dict is not None else None,
                       keep[1] if dict_huf is not None and dict is not None else None)


def decompress(f, *, verify=False, stream=None):
    """Decode a DeviceFrame on its device; returns a uint8 CUDA tensor of f.decoded_size bytes.

    Runs zxc_b200_decode_blocks on `stream` (default: torch's current stream) and zxc_b200_reduce_status, which
    synchronises it.  verify=True checks the block checksums (the frame must carry them)."""
    dev = f.frame.device
    with torch.cuda.device(dev):
        stream = stream or torch.cuda.current_stream(dev)
        with torch.cuda.stream(stream):
            out = torch.empty(f.decoded_size, dtype=torch.uint8, device=dev)
            n = f.n_blocks
            if n == 0:
                return out
            status = torch.empty(n, dtype=torch.int32, device=dev)
            scratch_size = int(lib.zxc_b200_decode_scratch_size(f.block_size))
            scratch = torch.empty(scratch_size, dtype=torch.uint8, device=dev)
            d_dict = d_huf = None
            dict_size = 0
            if f.dict is not None:
                host = f.dict + (f.dict_huf or b"")
                dd = torch.frombuffer(bytearray(host), dtype=torch.uint8).to(dev)
                d_dict, dict_size = dd.data_ptr(), len(f.dict)
                d_huf = d_dict + dict_size if f.dict_huf is not None else None
            rc = lib.zxc_b200_decode_blocks(f.frame.data_ptr(), out.data_ptr(), f.jobs.data_ptr(), n,
                                            status.data_ptr(), d_dict, dict_size, d_huf, scratch.data_ptr(),
                                            scratch_size, f.block_size, int(bool(verify and f.checksum)),
                                            stream.cuda_stream)
            if rc != 0:
                raise ZxcError(rc, "zxc_b200_decode_blocks")
            r = int(lib.zxc_b200_reduce_status(status.data_ptr(), f.jobs.data_ptr(), n, stream.cuda_stream))
    if r != f.decoded_size:
        raise ZxcError(r if r < 0 else -8, "zxc_b200_decode_blocks")
    return out


def decompress_frame(frame, *, capacity=None, dict=None, dict_huf=None, checksum=False, stream=None):
    """Decode the ZXC frame held in a contiguous uint8 CUDA tensor; returns a uint8 tensor of the decoded bytes.

    Runs zxc_b200_decompress_device on `stream` (default: torch's current stream of the frame's device): the frame is
    planned, decoded and checked on the device, and the stream is synchronised once to read the result.  The result
    and the bytes are what zxc_decompress returns for the same frame, capacity and options; an error raises ZxcError
    with its exact code.  capacity=None reads the decoded size from the frame's 8-byte footer with one small
    device-to-host copy (together with the header byte that sizes the scratch) and allocates that much output and the
    scratch for it.  The footer is trusted only as far as zxc_get_decompressed_size trusts it (at most one block of
    block_size per 8 bytes of frame); a footer past that raises ValueError, and a large plausible one can still ask
    for more device memory than there is (torch's OutOfMemoryError).  For frames from an untrusted source pass
    capacity: the output room to allow.  checksum=True verifies the block
    checksums and the global hash when the frame has them.  dict / dict_huf are host bytes, or dict is a DeviceDict."""
    if not frame.is_cuda or frame.dtype != torch.uint8 or not frame.is_contiguous():
        raise ValueError("frame must be a contiguous uint8 CUDA tensor")
    f = frame.reshape(-1)
    n = f.numel()
    o = _DOpts(checksum_enabled=int(bool(checksum)))
    keep, dd = _dict_opts(o, dict, dict_huf)
    dev = f.device
    with torch.cuda.device(dev):
        stream = stream or torch.cuda.current_stream(dev)
        with torch.cuda.stream(stream):
            # one small copy: the header's block-size code sizes the scratch, the footer gives the default capacity
            bs, footer = 4096, 0
            if n >= 28:
                h = torch.cat([f[5:6], f[n - 12:n - 4]]).cpu().numpy().tobytes()
                bs, footer = 1 << h[0] if 12 <= h[0] <= 21 else 4096, int.from_bytes(h[1:], "little")
            if capacity is None:
                if -(-footer // bs) > n // 8:  # zxf_dsize_plausible: more blocks than the frame has room for
                    raise ValueError(f"the frame's footer claims {footer} bytes, more than it can hold; pass capacity")
                capacity = footer
            capacity = int(capacity)
            scratch_size = int(lib.zxc_b200_decompress_device_scratch_size(capacity, bs))
            if scratch_size == 0:
                raise ValueError("zxc_b200_decompress_device_scratch_size: capacity too large, or no device")
            out = torch.empty(max(capacity, 1), dtype=torch.uint8, device=dev)
            scratch = torch.empty(scratch_size, dtype=torch.uint8, device=dev)
            result = torch.empty(1, dtype=torch.int64, device=dev)
            rc = _call("zxc_b200_decompress_device", dd,
                       (f.data_ptr(), n, out.data_ptr() if capacity else None, capacity, C.byref(o)),
                       (scratch.data_ptr(), scratch_size, result.data_ptr(), stream.cuda_stream))
            if rc != 0:
                raise ZxcError(rc, "zxc_b200_decompress_device")
            stream.synchronize()
            r = int(result.item())
    if r < 0:
        raise ZxcError(r, "zxc_b200_decompress_device")
    return out[:r]


lib.zxc_decompress_inplace_bound.restype = C.c_size_t
lib.zxc_decompress_inplace_bound.argtypes = [C.c_void_p, C.c_size_t]
lib.zxc_b200_decompress_inplace_device_bound.restype = C.c_size_t
lib.zxc_b200_decompress_inplace_device_bound.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
lib.zxc_b200_decompress_inplace_device_scratch_size.restype = C.c_size_t
lib.zxc_b200_decompress_inplace_device_scratch_size.argtypes = [C.c_uint64, C.c_uint32, C.c_uint64]
lib.zxc_b200_decompress_inplace_device.restype = C.c_int
lib.zxc_b200_decompress_inplace_device.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p,
                                                   C.c_size_t, C.c_void_p, C.c_void_p]

WINDOW_DEFAULT = 256 << 20


def _host_bytes(frame):
    """a host frame (bytes-like or array) as a contiguous uint8 numpy array"""
    import numpy as np
    return np.ascontiguousarray(np.frombuffer(frame, np.uint8) if isinstance(frame, (bytes, bytearray, memoryview))
                                else np.asarray(frame).reshape(-1).view(np.uint8))


def inplace_bound(frame, stream=None):
    """zxc_decompress_inplace_bound: the buffer size that decodes `frame` in place (0 for a frame it rejects).

    `frame` is a contiguous uint8 CUDA tensor (its header and footer are read with zxc_b200_decompress_inplace_device_bound,
    which synchronises `stream`, default the current stream) or host bytes / an array."""
    if isinstance(frame, torch.Tensor) and frame.is_cuda:
        if frame.dtype != torch.uint8 or not frame.is_contiguous():
            raise ValueError("frame must be a contiguous uint8 CUDA tensor")
        with torch.cuda.device(frame.device):
            stream = stream or torch.cuda.current_stream(frame.device)
            return int(lib.zxc_b200_decompress_inplace_device_bound(frame.data_ptr(), frame.numel(),
                                                                    stream.cuda_stream))
    h = _host_bytes(frame.numpy() if isinstance(frame, torch.Tensor) else frame)
    return int(lib.zxc_decompress_inplace_bound(h.ctypes.data, h.size))


def decompress_inplace(buf, comp_size, *, dict=None, dict_huf=None, checksum=False, window=None, stream=None):
    """Decode the frame of comp_size bytes that lies flush-right in `buf`, a contiguous uint8 CUDA tensor, into the
    same tensor; returns buf[:n], n the decoded size.

    Runs zxc_b200_decompress_inplace_device on `stream` (default: the current stream of buf's device) and synchronises
    it once to read the result, which is what zxc_decompress_inplace returns for the same buffer and options; an error
    raises ZxcError with its exact code (the buffer's contents are then unspecified, except for ZXC_ERROR_MEMORY from
    the round schedule, which leaves it as it was).  `window` is the compressed bytes staged per round, default
    min(comp_size, 256 MiB); a window of comp_size decodes in one round unless the scratch it takes reads as one for a
    larger block size (see zxc_b200_decompress_inplace_device in zxc_b200.h).  Reads the frame's header byte that
    sizes the scratch with one small copy.  dict / dict_huf are host bytes, or dict is a DeviceDict."""
    if not buf.is_cuda or buf.dtype != torch.uint8 or not buf.is_contiguous():
        raise ValueError("buf must be a contiguous uint8 CUDA tensor")
    b = buf.reshape(-1)
    cap, comp_size = b.numel(), int(comp_size)
    o = _DOpts(checksum_enabled=int(bool(checksum)))
    keep, dd = _dict_opts(o, dict, dict_huf)
    window = min(int(window) if window is not None else WINDOW_DEFAULT, comp_size)
    dev = b.device
    with torch.cuda.device(dev):
        stream = stream or torch.cuda.current_stream(dev)
        with torch.cuda.stream(stream):
            bs = 4096
            if 28 <= comp_size <= cap:
                code = int(b[cap - comp_size + 5].item())
                bs = 1 << code if 12 <= code <= 21 else 4096
            scratch_size = int(lib.zxc_b200_decompress_inplace_device_scratch_size(cap, bs, window))
            if scratch_size == 0:
                raise ValueError("zxc_b200_decompress_inplace_device_scratch_size: buffer too large, or no device")
            scratch = torch.empty(scratch_size, dtype=torch.uint8, device=dev)
            result = torch.empty(1, dtype=torch.int64, device=dev)
            rc = _call("zxc_b200_decompress_inplace_device", dd, (b.data_ptr(), cap, comp_size, C.byref(o)),
                       (scratch.data_ptr(), scratch_size, result.data_ptr(), stream.cuda_stream))
            if rc != 0:
                raise ZxcError(rc, "zxc_b200_decompress_inplace_device")
            stream.synchronize()
            r = int(result.item())
    if r < 0:
        raise ZxcError(r, "zxc_b200_decompress_inplace_device")
    return b[:r]


def load_frame(frame, *, device=None, dict=None, dict_huf=None, checksum=False, window=None, stream=None):
    """Bring a ZXC frame from host memory (bytes or an array) into HBM and decode it there in place; returns a uint8
    CUDA tensor of the decoded bytes.

    Allocates one buffer of zxc_decompress_inplace_bound bytes on `device` (default: the current CUDA device), copies
    the frame to its end and runs decompress_inplace on it: the device memory taken is that buffer and the decode's
    scratch, with no separate copy of the compressed frame.  The result is a view of the buffer.  A frame the bound
    rejects is decoded in a buffer of its own size, so it raises ZxcError with zxc_decompress_inplace's code for it."""
    h = _host_bytes(frame)
    bound = int(lib.zxc_decompress_inplace_bound(h.ctypes.data, h.size)) or max(h.size, 1)
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(dev):
        stream = stream or torch.cuda.current_stream(dev)
        with torch.cuda.stream(stream):
            buf = torch.empty(bound, dtype=torch.uint8, device=dev)
            with warnings.catch_warnings():  # a frame from bytes is read-only; it is only read
                warnings.simplefilter("ignore")
                buf[bound - h.size:].copy_(torch.from_numpy(h))
    return decompress_inplace(buf, h.size, dict=dict, dict_huf=dict_huf, checksum=checksum, window=window,
                              stream=stream)


lib.zxc_b200_decompress_device_batch_scratch_size.restype = C.c_size_t
lib.zxc_b200_decompress_device_batch_scratch_size.argtypes = [C.c_uint32, C.c_uint64, C.c_uint32]
lib.zxc_b200_decompress_device_batch.restype = C.c_int
lib.zxc_b200_decompress_device_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t,
                                                 C.c_void_p, C.c_void_p]


def decompress_frames(frames, capacities=None, *, out=None, dict=None, dict_huf=None, checksum=False, block_size=None,
                      stream=None):
    """Decode many ZXC frames, each a contiguous uint8 CUDA tensor on one device, in one batch call.

    Returns (outs, results): outs[i] is frame i's output tensor, results an int64 CUDA tensor where results[i] is
    exactly what decompress_frame's zxc_b200_decompress_device call gives frame i (its byte count or a negative
    zxc_error_t code; the bytes of a failed frame are unspecified).  capacities gives each frame's output room; with
    capacities=None every frame's footer and header byte are read with one gathered device-to-host copy, sized with
    decompress_frame's plausibility rule (ValueError for a footer past it, or a frame below 28 bytes).  `out`, a list
    of contiguous uint8 tensors on the frames' device, one per frame, takes the outputs instead (its sizes are the
    capacities).  block_size is the largest block size to accept (frames with larger blocks get ZXC_ERROR_MEMORY, as
    zxc_b200_decompress_device with a scratch sized for it gives): by default the largest any frame's header names
    when capacities are read from the footers, else 64 KiB.  The work runs on `stream` (default: the current stream), which first waits for the current stream; with `out` or
    capacities given nothing synchronises.  Argument errors raise ValueError before anything is enqueued; a rejected
    call raises ZxcError.  dict / dict_huf are host bytes, one dictionary for the batch, or dict is a DeviceDict."""
    frames = list(frames)
    if not frames:
        raise ValueError("frames is empty")
    dev = frames[0].device
    for f in frames:
        if not f.is_cuda or f.dtype != torch.uint8 or not f.is_contiguous():
            raise ValueError("every frame must be a contiguous uint8 CUDA tensor")
        if f.device != dev:
            raise ValueError(f"every frame must be on {dev}, not {f.device}")
    frames = [f.reshape(-1) for f in frames]
    n = len(frames)
    if out is not None:
        out = list(out)
        if len(out) != n:
            raise ValueError("out must hold one tensor per frame")
        for o in out:
            _check_out(o, dev)
        if capacities is not None and [int(c) for c in capacities] != [o.numel() for o in out]:
            raise ValueError("capacities differ from the sizes of out")
        capacities = [o.numel() for o in out]
    if block_size is not None and block_size not in [1 << k for k in range(12, 22)]:
        raise ValueError("block_size must be a power of two from 4 KiB to 2 MiB")
    if capacities is not None:
        block_size = block_size or 65536
        capacities = [int(c) for c in capacities]
        if len(capacities) != n:
            raise ValueError("capacities must hold one value per frame")
        if any(c < 0 for c in capacities):
            raise ValueError("capacities must not be negative")
    o = _DOpts(checksum_enabled=int(bool(checksum)))
    keep, dd = _dict_opts(o, dict, dict_huf)
    with torch.cuda.device(dev):
        current = torch.cuda.current_stream(dev)
        stream = stream or current
        if stream != current:
            # the inputs were made (or written) on the current stream; the caller may drop them on return
            stream.wait_stream(current)
            for t in frames + (out or []):
                t.record_stream(stream)
        with torch.cuda.stream(stream):
            if capacities is None:
                # one gathered copy: every frame's header block-size byte and 8-byte footer
                sizes = [f.numel() for f in frames]
                if min(sizes) < 28:
                    raise ValueError("a frame below 28 bytes has no footer; pass capacities")
                h = torch.cat([t for f in frames for t in (f[5:6], f[-12:-4])]).cpu().numpy().reshape(n, 9)
                capacities, bs = [], 4096
                for i, row in enumerate(h):
                    b = 1 << int(row[0]) if 12 <= row[0] <= 21 else 4096
                    footer = int.from_bytes(row[1:].tobytes(), "little")
                    if -(-footer // b) > sizes[i] // 8:  # zxf_dsize_plausible
                        raise ValueError(f"frame {i}'s footer claims {footer} bytes, more than it can hold; "
                                         "pass capacities")
                    capacities.append(footer)
                    bs = max(bs, b)
                block_size = block_size or bs
            if out is None:
                out = [torch.empty(max(c, 1), dtype=torch.uint8, device=dev)[:c] for c in capacities]
            # page-locked, so the upload does not wait for the stream (the host allocator keeps it until it ran)
            desc = torch.tensor([[f.data_ptr(), f.numel(), t.data_ptr() if c else 0, c]
                                 for f, t, c in zip(frames, out, capacities)], dtype=torch.int64)
            desc = desc.pin_memory().to(dev, non_blocking=True)
            scratch_size = int(lib.zxc_b200_decompress_device_batch_scratch_size(n, sum(capacities), block_size))
            if scratch_size == 0:
                raise ValueError("zxc_b200_decompress_device_batch_scratch_size: too many frames or bytes, or no device")
            scratch = torch.empty(scratch_size, dtype=torch.uint8, device=dev)
            results = torch.empty(n, dtype=torch.int64, device=dev)
            rc = _call("zxc_b200_decompress_device_batch", dd, (desc.data_ptr(), n, C.byref(o)),
                       (scratch.data_ptr(), scratch_size, results.data_ptr(), stream.cuda_stream))
            if rc != 0:
                raise ZxcError(rc, "zxc_b200_decompress_device_batch")
    return out, results


lib.zxc_b200_compress_device_batch_scratch_size.restype = C.c_size_t
lib.zxc_b200_compress_device_batch_scratch_size.argtypes = [C.c_uint32, C.c_uint64, C.c_void_p]
lib.zxc_b200_compress_device_batch.restype = C.c_int
lib.zxc_b200_compress_device_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                               C.c_void_p]


def compress_frames(srcs, *, level=0, block_size=0, checksum=False, seekable=False, dict=None, dict_huf=None, out=None,
                    stream=None):
    """Compress many contiguous CUDA tensors (their bytes), all on one device, into one ZXC frame each in one batch call.

    Returns (outs, results): outs[i] is the tensor frame i was written to (by default zxc_compress_bound(len) bytes),
    results an int64 CUDA tensor where results[i] is exactly what compress's zxc_b200_compress_device call gives
    input i alone: its frame size (the frame is outs[i][:results[i]]) or a negative zxc_error_t code.  `out`, a list of
    contiguous uint8 tensors on the inputs' device, one per input, takes the frames instead.  The work runs on `stream`
    (default: the current stream), which first waits for the current stream; nothing synchronises.  Argument errors
    raise ValueError before anything is enqueued; a rejected call raises ZxcError with its code.  dict / dict_huf are
    host bytes, one dictionary for the batch, or dict is a DeviceDict."""
    srcs = list(srcs)
    if not srcs:
        raise ValueError("srcs is empty")
    dev = srcs[0].device
    for t in srcs:
        if not t.is_cuda or not t.is_contiguous():
            raise ValueError("every input must be a contiguous CUDA tensor")
        if t.device != dev:
            raise ValueError(f"every input must be on {dev}, not {t.device}")
    srcs = [t.reshape(-1).view(torch.uint8) for t in srcs]
    n = len(srcs)
    if out is not None:
        out = list(out)
        if len(out) != n:
            raise ValueError("out must hold one tensor per input")
        for o in out:
            _check_out(o, dev)
    o = _Opts(level=level, block_size=block_size, checksum_enabled=int(bool(checksum)), seekable=int(bool(seekable)))
    keep, dd = _dict_opts(o, dict, dict_huf)
    # 0 for options the call rejects (it then gives their exact code below with a token scratch), or a batch too large
    scratch_size = int(lib.zxc_b200_compress_device_batch_scratch_size(n, sum(t.numel() for t in srcs), C.byref(o)))
    with torch.cuda.device(dev):
        current = torch.cuda.current_stream(dev)
        stream = stream or current
        if stream != current:
            # the inputs were made (or written) on the current stream; the caller may drop them on return
            stream.wait_stream(current)
            for t in srcs + (out or []):
                t.record_stream(stream)
        with torch.cuda.stream(stream):
            if out is None:
                out = [torch.empty(int(lib.zxc_compress_bound(t.numel())), dtype=torch.uint8, device=dev) for t in srcs]
            # page-locked, so the upload does not wait for the stream (the host allocator keeps it until it ran)
            desc = torch.tensor([[t.data_ptr() if t.numel() else 0, t.numel(), d.data_ptr() if d.numel() else 0,
                                  d.numel()] for t, d in zip(srcs, out)], dtype=torch.int64)
            desc = desc.pin_memory().to(dev, non_blocking=True)
            scratch = torch.empty(max(scratch_size, 1), dtype=torch.uint8, device=dev)
            results = torch.empty(n, dtype=torch.int64, device=dev)
            rc = _call("zxc_b200_compress_device_batch", dd, (desc.data_ptr(), n, C.byref(o)),
                       (scratch.data_ptr(), scratch_size, results.data_ptr(), stream.cuda_stream))
            if rc != 0:
                raise ZxcError(rc, "zxc_b200_compress_device_batch")
    return out, results


lib.zxc_compress_block_bound.restype = C.c_uint64
lib.zxc_compress_block_bound.argtypes = [C.c_size_t]
lib.zxc_b200_compress_blocks_device_scratch_size.restype = C.c_size_t
lib.zxc_b200_compress_blocks_device_scratch_size.argtypes = [C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p]
lib.zxc_b200_compress_blocks_device.restype = C.c_int
lib.zxc_b200_compress_blocks_device.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t,
                                                C.c_void_p, C.c_void_p]
lib.zxc_b200_decompress_blocks_device_scratch_size.restype = C.c_size_t
lib.zxc_b200_decompress_blocks_device_scratch_size.argtypes = [C.c_uint32, C.c_uint64]
lib.zxc_b200_decompress_blocks_device.restype = C.c_int
lib.zxc_b200_decompress_blocks_device.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t,
                                                  C.c_void_p, C.c_void_p]
# the _using_dict variants: the base call's arguments with the DeviceDict handle right after opts
for _name, _opts_at in (("compress_device", 4), ("compress_device_batch", 2), ("compress_blocks_device", 2),
                        ("decompress_device", 4), ("decompress_inplace_device", 3), ("decompress_device_batch", 2),
                        ("decompress_blocks_device", 2)):
    _base = getattr(lib, f"zxc_b200_{_name}")
    _var = getattr(lib, f"zxc_b200_{_name}_using_dict")
    _var.restype = C.c_int
    _var.argtypes = _base.argtypes[: _opts_at + 1] + [C.c_void_p] + _base.argtypes[_opts_at + 1:]


def _same_device(tensors, what):
    tensors = list(tensors)
    if not tensors:
        raise ValueError(f"{what} is empty")
    dev = tensors[0].device
    for t in tensors:
        if not t.is_cuda or not t.is_contiguous():
            raise ValueError(f"every {what[:-1]} must be a contiguous CUDA tensor")
        if t.device != dev:
            raise ValueError(f"every {what[:-1]} must be on {dev}, not {t.device}")
    return [t.reshape(-1).view(torch.uint8) for t in tensors], dev


def _run_items(dev, ins, out, stream, call):
    """Uploads the item descriptors (in, out) and runs call(desc, results, stream) on `stream` after the current
    stream; returns the results tensor."""
    with torch.cuda.device(dev):
        current = torch.cuda.current_stream(dev)
        stream = stream or current
        if stream != current:
            # the inputs were made (or written) on the current stream; the caller may drop them on return
            stream.wait_stream(current)
            for t in ins + out:
                t.record_stream(stream)
        with torch.cuda.stream(stream):
            # page-locked, so the upload does not wait for the stream (the host allocator keeps it until it ran)
            desc = torch.tensor([[s.data_ptr() if s.numel() else 0, s.numel(), d.data_ptr() if d.numel() else 0,
                                  d.numel()] for s, d in zip(ins, out)], dtype=torch.int64)
            desc = desc.pin_memory().to(dev, non_blocking=True)
            results = torch.empty(len(ins), dtype=torch.int64, device=dev)
            call(desc, results, stream)
    return results


def compress_blocks(srcs, *, level=0, checksum=False, dict=None, out=None, stream=None):
    """Compress many contiguous CUDA tensors (their bytes), all on one device, into one frameless block each, in one
    zxc_b200_compress_blocks_device call.

    Returns (outs, results): results[i] (an int64 CUDA tensor) is exactly what zxc_compress_block gives input i on a
    fresh context: its block size (the block is outs[i][:results[i]]) or a negative zxc_error_t code.  outs[i] holds
    zxc_compress_block_bound(len) bytes by default; `out`, a list of contiguous uint8 tensors on the inputs' device,
    one per input, takes the blocks instead.  The work runs on `stream` (default: the current stream), which first
    waits for the current stream; nothing synchronises.  Argument errors raise ValueError before anything is enqueued;
    a rejected call raises ZxcError.  dict is host bytes, one dictionary for the batch, or a DeviceDict."""
    srcs, dev = _same_device(srcs, "srcs")
    if out is not None:
        out = list(out)
        if len(out) != len(srcs):
            raise ValueError("out must hold one tensor per input")
        for o in out:
            _check_out(o, dev)
    o = _Opts(level=level, checksum_enabled=int(bool(checksum)))
    keep, dd = _dict_opts(o, dict, None)
    sizes = [t.numel() for t in srcs]
    # 0 for a batch the call cannot plan (it then gives its exact code with a token scratch)
    scratch_size = int(lib.zxc_b200_compress_blocks_device_scratch_size(len(srcs), sum(sizes),
                                                                        min(max(sizes), 1 << 21), C.byref(o)))
    if out is None:
        out = [torch.empty(max(int(lib.zxc_compress_block_bound(n)), 1), dtype=torch.uint8, device=dev)
               for n in sizes]

    def call(desc, results, stream):
        scratch = torch.empty(max(scratch_size, 1), dtype=torch.uint8, device=dev)
        rc = _call("zxc_b200_compress_blocks_device", dd, (desc.data_ptr(), len(srcs), C.byref(o)),
                   (scratch.data_ptr(), scratch_size, results.data_ptr(), stream.cuda_stream))
        if rc != 0:
            raise ZxcError(rc, "zxc_b200_compress_blocks_device")

    return out, _run_items(dev, srcs, out, stream, call)


def decompress_blocks(blocks, sizes, *, safe=False, checksum=False, dict=None, out=None, stream=None):
    """Decode many frameless blocks, each a contiguous uint8 CUDA tensor on one device, in one
    zxc_b200_decompress_blocks_device call.

    sizes[i] is block i's output room (its dst_capacity).  Returns (outs, results): results[i] (an int64 CUDA tensor)
    is exactly what zxc_decompress_block (zxc_decompress_block_safe with safe=True) gives block i: its decoded size
    (the bytes are outs[i][:results[i]]) or a negative zxc_error_t code.  `out`, a list of contiguous uint8 tensors on
    the blocks' device, one per block, takes the outputs instead (its sizes must equal sizes).  The work runs on
    `stream` (default: the current stream), which first waits for the current stream; nothing synchronises.  Argument
    errors raise ValueError before anything is enqueued; a rejected call raises ZxcError.  dict is host bytes or a
    DeviceDict."""
    blocks, dev = _same_device(blocks, "blocks")
    sizes = [int(c) for c in sizes]
    if len(sizes) != len(blocks):
        raise ValueError("sizes must hold one value per block")
    if any(c < 0 for c in sizes):
        raise ValueError("sizes must not be negative")
    if out is not None:
        out = list(out)
        if len(out) != len(blocks):
            raise ValueError("out must hold one tensor per block")
        for o in out:
            _check_out(o, dev)
        if [o.numel() for o in out] != sizes:
            raise ValueError("sizes differ from the sizes of out")
    o = _DOpts(checksum_enabled=int(bool(checksum)))
    keep, dd = _dict_opts(o, dict, None)
    scratch_size = int(lib.zxc_b200_decompress_blocks_device_scratch_size(len(blocks), max(sizes)))
    if scratch_size == 0:
        raise ValueError("zxc_b200_decompress_blocks_device_scratch_size: too many blocks, or no device")
    if out is None:
        out = [torch.empty(max(c, 1), dtype=torch.uint8, device=dev)[:c] for c in sizes]

    def call(desc, results, stream):
        scratch = torch.empty(scratch_size, dtype=torch.uint8, device=dev)
        rc = _call("zxc_b200_decompress_blocks_device", dd, (desc.data_ptr(), len(blocks), C.byref(o)),
                   (int(bool(safe)), scratch.data_ptr(), scratch_size, results.data_ptr(), stream.cuda_stream))
        if rc != 0:
            raise ZxcError(rc, "zxc_b200_decompress_blocks_device")

    return out, _run_items(dev, blocks, out, stream, call)


lib.zxc_b200_seekable_device_open.restype = C.c_void_p
lib.zxc_b200_seekable_device_open.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
lib.zxc_b200_seekable_device_set_dict.restype = C.c_int
lib.zxc_b200_seekable_device_set_dict.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
lib.zxc_b200_seekable_device_num_blocks.restype = C.c_uint32
lib.zxc_b200_seekable_device_num_blocks.argtypes = [C.c_void_p]
lib.zxc_b200_seekable_device_decompressed_size.restype = C.c_uint64
lib.zxc_b200_seekable_device_decompressed_size.argtypes = [C.c_void_p]
lib.zxc_b200_seekable_device_block_size.restype = C.c_uint32
lib.zxc_b200_seekable_device_block_size.argtypes = [C.c_void_p]
lib.zxc_b200_seekable_device_scratch_size.restype = C.c_size_t
lib.zxc_b200_seekable_device_scratch_size.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64]
lib.zxc_b200_seekable_device_decompress_ranges.restype = C.c_int
lib.zxc_b200_seekable_device_decompress_ranges.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64,
                                                           C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
lib.zxc_b200_seekable_device_free.restype = None
lib.zxc_b200_seekable_device_free.argtypes = [C.c_void_p]


def _check_out(out, device):
    """An output the range call may write out.numel() bytes into from out.data_ptr(): a contiguous uint8 tensor on
    the frame's CUDA device.  ValueError otherwise, before anything is enqueued."""
    if out.dtype != torch.uint8:
        raise ValueError(f"out must be a uint8 tensor, not {out.dtype}")
    if not out.is_contiguous():
        raise ValueError("out must be contiguous")
    if out.device != device:
        raise ValueError(f"out must be on the frame's device {device}, not {out.device}")


class SeekableFrame:
    """Random access into a seekable ZXC frame held in a contiguous uint8 CUDA tensor.

    Opens the frame with zxc_b200_seekable_device_open (the SEK table is parsed once; its block offsets stay on the
    device) and decodes byte ranges of the decompressed content with zxc_b200_seekable_device_decompress_ranges.  The
    frame tensor is kept alive and must not change while the object is open.  dict / dict_huf are host bytes, set
    with zxc_b200_seekable_device_set_dict.  Raises ValueError when the frame is not seekable (where
    zxc_seekable_open returns NULL) and ZxcError for a rejected dictionary."""

    def __init__(self, frame, dict=None, dict_huf=None):
        self._h = None  # before any check: __del__ runs on a half-made object too
        if not frame.is_cuda or frame.dtype != torch.uint8 or not frame.is_contiguous():
            raise ValueError("frame must be a contiguous uint8 CUDA tensor")
        self.frame = frame.reshape(-1)
        with torch.cuda.device(self.frame.device):
            h = lib.zxc_b200_seekable_device_open(self.frame.data_ptr(), self.frame.numel(),
                                                  torch.cuda.current_stream().cuda_stream)
        if not h:
            raise ValueError("not a seekable ZXC frame (or no device)")
        self._h = h
        if dict is not None:
            d = bytes(dict)
            hf = bytes(dict_huf) if dict_huf is not None else None
            rc = lib.zxc_b200_seekable_device_set_dict(self._h, d, len(d), hf)
            if rc != 0:
                self.close()
                raise ZxcError(rc, "zxc_b200_seekable_device_set_dict")

    @property
    def decompressed_size(self):
        return int(lib.zxc_b200_seekable_device_decompressed_size(self._handle()))

    @property
    def block_size(self):
        return int(lib.zxc_b200_seekable_device_block_size(self._handle()))

    @property
    def n_blocks(self):
        return int(lib.zxc_b200_seekable_device_num_blocks(self._handle()))

    def _handle(self):
        if self._h is None:
            raise ValueError("SeekableFrame is closed")
        return self._h

    def close(self):
        if self._h is not None:
            lib.zxc_b200_seekable_device_free(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        self.close()

    def gather(self, offsets, lengths, out=None, stream=None):
        """Decode the ranges [offsets[i], offsets[i] + lengths[i]) back to back into one uint8 tensor.

        offsets and lengths are int64 CUDA tensors of one length; range i lands at the sum of the lengths before it
        (an exclusive cumsum computed on the device).  Returns (out, results) with no synchronisation when `out` is
        given (its size bounds the scratch); without it, the total length is read back once to allocate out.  `out`
        must be a contiguous uint8 tensor on the frame's device (ValueError otherwise).  The work runs on `stream`
        (default: the current stream), which first waits for the current stream; the returned tensors are written on
        `stream`, so a caller reading them on another stream orders it after `stream` first.
        results[i] (int64, on the device) is the range's byte count or a negative zxc_error_t code, exactly what
        zxc_seekable_decompress_range returns for it; the bytes of a failed range are unspecified."""
        h = self._handle()
        dev = self.frame.device
        if out is not None:
            _check_out(out, dev)
        offsets = offsets.reshape(-1).to(dev, torch.int64)
        lengths = lengths.reshape(-1).to(dev, torch.int64)
        if offsets.numel() != lengths.numel():
            raise ValueError("offsets and lengths differ in length")
        n = offsets.numel()
        with torch.cuda.device(dev):
            current = torch.cuda.current_stream(dev)
            stream = stream or current
            if stream != current:
                # the inputs were made (or written) on the current stream; the caller may drop them on return
                stream.wait_stream(current)
                for t in (offsets, lengths) + ((out,) if out is not None else ()):
                    t.record_stream(stream)
            with torch.cuda.stream(stream):
                dst_off = torch.cumsum(lengths, 0) - lengths
                if out is None:
                    out = torch.empty(int(lengths.sum().item()) if n else 0, dtype=torch.uint8, device=dev)
                results = torch.empty(n, dtype=torch.int64, device=dev)
                if n == 0:
                    return out, results
                ranges = torch.stack([offsets, lengths, dst_off], 1).contiguous()
                scratch_size = int(lib.zxc_b200_seekable_device_scratch_size(h, n, out.numel()))
                if scratch_size == 0:
                    raise ValueError("zxc_b200_seekable_device_scratch_size: too many ranges or bytes")
                scratch = torch.empty(scratch_size, dtype=torch.uint8, device=dev)
                rc = lib.zxc_b200_seekable_device_decompress_ranges(
                    h, ranges.data_ptr(), n, out.data_ptr() if out.numel() else None, out.numel(), scratch.data_ptr(),
                    scratch_size, results.data_ptr(), stream.cuda_stream)
                if rc != 0:
                    raise ZxcError(rc, "zxc_b200_seekable_device_decompress_ranges")
        return out, results

    def read(self, offset, length, stream=None):
        """Decode bytes [offset, offset + length) into a new uint8 tensor; synchronises and raises ZxcError with the
        exact code of zxc_seekable_decompress_range on failure."""
        dev = self.frame.device
        o = torch.tensor([int(offset)], dtype=torch.int64, device=dev)
        n = torch.tensor([int(length)], dtype=torch.int64, device=dev)
        out = torch.empty(int(length), dtype=torch.uint8, device=dev)
        stream = stream or torch.cuda.current_stream(dev)
        out, res = self.gather(o, n, out=out, stream=stream)
        stream.synchronize()
        r = int(res.item())
        if r < 0:
            raise ZxcError(r, "zxc_b200_seekable_device_decompress_ranges")
        return out


# ---------------------------------------------------------------------------------------------------------------------
# push streaming in HBM: zxc_b200_cstream_device / zxc_b200_dstream_device with zlib's compressobj / decompressobj shape
# ---------------------------------------------------------------------------------------------------------------------
class _InBuf(C.Structure):  # zxc_inbuf_t (include/zxc_pstream.h)
    _fields_ = [("src", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


class _OutBuf(C.Structure):  # zxc_outbuf_t
    _fields_ = [("dst", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


for _k in ("c", "d"):
    getattr(lib, f"zxc_b200_{_k}stream_device_create").restype = C.c_void_p
    getattr(lib, f"zxc_b200_{_k}stream_device_create").argtypes = [C.c_void_p]
    getattr(lib, f"zxc_b200_{_k}stream_device_free").restype = None
    getattr(lib, f"zxc_b200_{_k}stream_device_free").argtypes = [C.c_void_p]
    getattr(lib, f"zxc_b200_{_k}stream_device_out_size").restype = C.c_size_t
    getattr(lib, f"zxc_b200_{_k}stream_device_out_size").argtypes = [C.c_void_p]
lib.zxc_b200_cstream_device_compress.restype = C.c_int64
lib.zxc_b200_cstream_device_compress.argtypes = [C.c_void_p, C.POINTER(_OutBuf), C.POINTER(_InBuf), C.c_void_p]
lib.zxc_b200_cstream_device_end.restype = C.c_int64
lib.zxc_b200_cstream_device_end.argtypes = [C.c_void_p, C.POINTER(_OutBuf), C.c_void_p]
lib.zxc_b200_dstream_device_decompress.restype = C.c_int64
lib.zxc_b200_dstream_device_decompress.argtypes = [C.c_void_p, C.POINTER(_OutBuf), C.POINTER(_InBuf), C.c_void_p]
lib.zxc_b200_dstream_device_finished.restype = C.c_int
lib.zxc_b200_dstream_device_finished.argtypes = [C.c_void_p]

# out is collected in pieces of at least this size, so a large input is one call that batches all its blocks
_STREAM_CHUNK = 64 << 20


class _DeviceStream:
    def __init__(self, kind, opts):
        self._kind = kind
        self._device = torch.device("cuda", torch.cuda.current_device())
        with torch.cuda.device(self._device):
            self._h = getattr(lib, f"zxc_b200_{kind}stream_device_create")(C.byref(opts))
        if not self._h:
            raise ValueError(f"zxc_b200_{kind}stream_device_create rejected the options (or there is no device)")

    def _src(self, t):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise ValueError("data must be a CUDA tensor")
        if not t.is_contiguous():
            raise ValueError("data must be contiguous")
        if t.device != self._device:
            raise ValueError(f"data is on {t.device}, the stream on {self._device}")
        return t.reshape(-1).view(torch.uint8)

    def _run(self, step, stream):
        """Calls step(out, stream) with fresh out buffers until it has nothing more to give; the bytes, one tensor.
        The result owns storage of its own size: a view of a partly filled out buffer would keep all of it alive."""
        hint = int(getattr(lib, f"zxc_b200_{self._kind}stream_device_out_size")(self._h))
        parts = []
        with torch.cuda.device(self._device):
            stream = stream or torch.cuda.current_stream(self._device)
            while True:
                out = torch.empty(max(_STREAM_CHUNK, hint), dtype=torch.uint8, device=self._device)
                ob = _OutBuf(out.data_ptr(), out.numel(), 0)
                more = step(ob, stream.cuda_stream)
                parts.append(out if ob.pos == out.numel() else out[: ob.pos].clone())
                if not more:
                    break
            return parts[0] if len(parts) == 1 else torch.cat(parts)

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            getattr(lib, f"zxc_b200_{self._kind}stream_device_free")(h)


class DeviceCompress(_DeviceStream):
    """zxc_b200_cstream_device: CUDA tensors in, the compressed stream out as uint8 CUDA tensors.  Every call runs on
    `stream` (default: torch's current stream of the stream's device) and returns once its work is complete."""

    def __init__(self, level=0, block_size=0, checksum=False):
        super().__init__("c", _Opts(level=level, block_size=block_size, checksum_enabled=int(bool(checksum))))

    def _call(self, fn, what, *args):
        r = fn(self._h, *args)
        if r < 0:
            raise ZxcError(r, what)
        return r != 0

    def compress(self, data, stream=None):
        """Feeds data; returns the compressed bytes this made available (whole blocks, and the header first)."""
        b = self._src(data)
        ib = _InBuf(b.data_ptr() if b.numel() else None, b.numel(), 0)
        return self._run(lambda ob, st: self._call(lib.zxc_b200_cstream_device_compress, "zxc_b200_cstream_device_compress",
                                                   C.byref(ob), C.byref(ib), st), stream)

    def flush(self, stream=None):
        """Ends the stream: the last block, the EOF block and the footer.  The object is finished afterwards."""
        return self._run(lambda ob, st: self._call(lib.zxc_b200_cstream_device_end, "zxc_b200_cstream_device_end",
                                                   C.byref(ob), st), stream)


class DeviceDecompress(_DeviceStream):
    """zxc_b200_dstream_device: compressed CUDA tensors in, decoded bytes out as uint8 CUDA tensors; `eof` and
    `unused_data` (a view of the last input, then of the inputs after the end) as for zlib's decompressobj."""

    def __init__(self, checksum=False):
        super().__init__("d", _DOpts(checksum_enabled=int(bool(checksum))))
        self.eof = False
        self.unused_data = torch.empty(0, dtype=torch.uint8, device=self._device)

    def decompress(self, data, stream=None):
        """Feeds compressed bytes; returns what they decode to.  Bytes after the stream's footer go to unused_data."""
        b = self._src(data)
        if self.eof:
            self.unused_data = torch.cat([self.unused_data, b]) if self.unused_data.numel() else b
            return torch.empty(0, dtype=torch.uint8, device=self._device)
        ib = _InBuf(b.data_ptr() if b.numel() else None, b.numel(), 0)

        def step(ob, st):
            r = lib.zxc_b200_dstream_device_decompress(self._h, C.byref(ob), C.byref(ib), st)
            if r < 0:
                raise ZxcError(r, "zxc_b200_dstream_device_decompress")
            if lib.zxc_b200_dstream_device_finished(self._h):
                self.eof = True
                self.unused_data = b[ib.pos:]
                return False
            return ob.pos == ob.size  # out full: more may be waiting
        return self._run(step, stream)


def compressobj(level=0, block_size=0, checksum=False):
    """A push-streaming compressor for CUDA tensors on the current device (zxc_b200.stream.compressobj's shape)."""
    return DeviceCompress(level, block_size, checksum)


def decompressobj(checksum=False):
    """A push-streaming decompressor for CUDA tensors on the current device (zxc_b200.stream.decompressobj's shape)."""
    return DeviceDecompress(checksum)
