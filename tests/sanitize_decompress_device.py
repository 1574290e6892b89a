"""compute-sanitizer driver for zxc_b200_decompress_device: valid frames (seekable or not, checksums, a dictionary,
short non-final blocks) from unaligned sources that end at the end of their allocation, exact and short capacities,
and hostile frames (single-byte mutations, forged SEK tables, the invalid conformance vectors) -- memcheck must stay
silent and every result must equal zxc_decompress's.  Usage on the GPU machine:
    compute-sanitizer --tool memcheck python tests/sanitize_decompress_device.py"""
import glob
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import zxc_corpus as zc  # noqa: E402
import zxc_ctypes as z  # noqa: E402
from test_decompress_device import Dev, _mutants, _stitched  # noqa: E402
from test_oracle import G, golden_dicts, make_case  # noqa: E402

prod = z.ZxcLib(z.PRODUCT_SO)
dev = Dev(prod)
n = bad = 0


def check(frame, cap, cks=0, d=None, h=None, src_off=0):
    global n, bad
    r1, o1 = dev.run(frame, cap, cks, d, h, src_off=src_off)
    r0, o0 = prod.decompress(frame, cap, checksum=cks, dict=d, dict_huf=h)
    n += 1
    if r1 != r0 or (r0 > 0 and not np.array_equal(o0, o1)):
        bad += 1
        print("MISMATCH", frame.size, cap, cks, src_off, r0, r1)


d, h = next(iter(golden_dicts().values()))
data = zc.silesia_shaped(1 << 20, seed=5)[:140001]
for level, bs, cks, seek, dd, hh in ((1, 4096, 1, 1, None, None), (3, 65536, 0, 0, None, None),
                                     (6, 4096, 1, 0, None, None), (6, 4096, 1, 1, d, h)):
    frame = prod.compress(data, level=level, block_size=bs, checksum=cks, seekable=seek, dict=dd, dict_huf=hh)
    if isinstance(frame, int):
        sys.exit("zxc_compress failed: %s" % z.ERR.get(frame, frame))
    for src_off in (0, 1, 15):
        for cap in (data.size, data.size - 1, 5000, 0):
            check(frame, cap, cks, dd, hh, src_off)
    for _, m in _mutants(frame, 40, seed=level):
        check(m, data.size, 1, dd, hh)
frame, _ = _stitched(prod, data, 65536, 3, 4)
check(frame, data.size)
check(frame, data.size - 1)
for p in sorted(glob.glob(os.path.join(G, "invalid", "*.zxc"))):
    check(np.fromfile(p, np.uint8), 1 << 20, 1)
text = make_case("text", 60000)
seekf = prod.compress(text, level=2, block_size=4096, checksum=1, seekable=1)
for _, m in _mutants(seekf, 60, seed=99):
    check(m, text.size, 1)
print("sanitize_decompress_device: ran", n, "calls, mismatches:", bad)
sys.exit(1 if bad else 0)
