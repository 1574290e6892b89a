"""compute-sanitizer driver for the prepared device dictionaries (zxc_b200_dict_device_* and the _using_dict calls):
handles of 1, 4, 5, 16 Ki and 65 535 bytes, with and without a literal table, used by all seven variants at levels 1,
3 and 6 on inputs in exactly sized allocations -- memcheck must stay silent and every result must equal the base call
with the dictionary as host bytes.  Usage on a GPU machine:
    compute-sanitizer --tool memcheck python tests/sanitize_dict_device.py"""
import os
import sys

os.environ.setdefault("PYTORCH_NO_CUDA_MEMORY_CACHING", "1")  # every tensor its own cudaMalloc: exact bounds

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import zxc_corpus as zc  # noqa: E402
import zxc_b200.device as D  # noqa: E402
from test_oracle import golden_dicts  # noqa: E402

n = bad = 0


def same(what, a, b):
    global n, bad
    n += 1
    if not torch.equal(a, b):
        bad += 1
        print("MISMATCH", what)


text = zc.silesia_shaped(1 << 17, seed=3).tobytes()
c16, h16 = sorted(golden_dicts().values())[0]
dicts = [(text[:1], None), (text[:4], None), (text[:5], None), (c16, None), (c16, h16), (text[:65535], None)]
src = np.ascontiguousarray(zc.records(24, 4096, seed=9))
s = torch.from_numpy(src).cuda()
srcs = [torch.from_numpy(src[i * 5000:i * 5000 + k].copy()).cuda() for i, k in enumerate((1, 4096, 9000, 30000))]
for c, h in dicts:
    with D.DeviceDict(c, h) as dd:
        for level in (1, 3, 6):
            kw = dict(level=level, block_size=4096, checksum=True, seekable=True)
            fb, fd = D.compress(s, dict=c, dict_huf=h, **kw), D.compress(s, dict=dd, **kw)
            same(("compress", len(c), level), fb.frame, fd.frame)
            same(("decompress_frame", len(c), level), D.decompress_frame(fd.frame, dict=dd, checksum=True), s)
            same(("load_frame", len(c), level), D.load_frame(fd.frame.cpu().numpy(), dict=dd, checksum=True), s)
            ob, rb = D.compress_frames(srcs, dict=c, dict_huf=h, **kw)
            od, rd = D.compress_frames(srcs, dict=dd, **kw)
            same(("compress_frames", len(c), level), rb, rd)
            frames = [o[:r] for o, r in zip(od, rd.tolist())]
            xd, yd = D.decompress_frames(frames, [t.numel() for t in srcs], dict=dd, checksum=True)
            for a, b in zip(xd, srcs):
                same(("decompress_frames", len(c), level), a, b)
            bb, rbb = D.compress_blocks(srcs, level=level, checksum=True, dict=c)
            bd, rbd = D.compress_blocks(srcs, level=level, checksum=True, dict=dd)
            same(("compress_blocks", len(c), level), rbb, rbd)
            blocks = [torch.cat([b[:r], torch.zeros(8, dtype=torch.uint8, device="cuda")]) for b, r in
                      zip(bd, rbd.tolist())]
            views = [b[:r] for b, r in zip(blocks, rbd.tolist())]
            pd_, qd = D.decompress_blocks(views, [t.numel() for t in srcs], checksum=True, dict=dd)
            for a, b in zip(pd_, srcs):
                same(("decompress_blocks", len(c), level), a, b)
torch.cuda.synchronize()
print("sanitize_dict_device: ran", n, "checks, mismatches:", bad)
sys.exit(1 if bad else 0)
