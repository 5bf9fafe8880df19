"""Regenerate tests/golden/yuv_golden.npz: libyuv's own RGBA8 output (the reference's nv12ToRgba8 / nv21ToRgba8 / i420ToRgba8, through
oracle/_ref/libyuv_ref.so, built by oracle/yuv.mk from the reference checkout) for BT.601 and BT.709 and all three 4:2:0 formats.

- "pairs": one 1 x 131072 frame (width 1, so that each chroma sample covers two luma rows) whose chroma samples take every (U, V) pair
  and whose luma rows take every Y value. NV12, NV21 and I420 of the same samples give the same image (checked here), stored once per
  matrix as pairs_rgba_<matrix>.
- "odd": random frames of 1 x 1, 3 x 5 and 33 x 17 (H x W), whose last chroma column and row cover one luma column / row, per format
  and matrix: odd_<h>x<w>_y / _u / _v and odd_<h>x<w>_<format>_<matrix>.

    python tests/golden/make_yuv_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import yuv  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "yuv_golden.npz")
ODD = [(1, 1), (3, 5), (33, 17)]


def pairs_planes():
    i = np.arange(65536)
    u, v = (i & 255).astype(np.uint8)[:, None], (i >> 8).astype(np.uint8)[:, None]
    y = ((np.arange(2 * 65536) * 37) & 255).astype(np.uint8)[:, None]  # 37 is odd: every Y value, 512 times
    return y, u, v


def main():
    if yuv.libyuv() is None:
        sys.exit("oracle/_ref/libyuv_ref.so is missing: run `make -C oracle -f yuv.mk yuv` with the reference checkout present")
    data = {}
    y, u, v = pairs_planes()
    for m in yuv.MATRICES:
        outs = [yuv.libyuv_to_rgba(fmt, *yuv.planes_from_yuv(fmt, y, u, v), matrix=m) for fmt in yuv.FORMATS]
        assert all(np.array_equal(outs[0], o) for o in outs[1:]), m
        data["pairs_rgba_" + m] = outs[0][:, 0]
    rng = np.random.default_rng(1744)
    for h, w in ODD:
        ch, cw = yuv.chroma_shape(h, w)
        k = "odd_%dx%d" % (h, w)
        data[k + "_y"] = rng.integers(0, 256, (h, w), dtype=np.uint8)
        data[k + "_u"] = rng.integers(0, 256, (ch, cw), dtype=np.uint8)
        data[k + "_v"] = rng.integers(0, 256, (ch, cw), dtype=np.uint8)
        for fmt in yuv.FORMATS:
            for m in yuv.MATRICES:
                data["%s_%s_%s" % (k, fmt, m)] = yuv.libyuv_to_rgba(fmt, *yuv.planes_from_yuv(fmt, data[k + "_y"], data[k + "_u"], data[k + "_v"]), matrix=m)
    np.savez_compressed(OUT, **data)
    print("wrote %s (%d bytes, %d arrays)" % (OUT, os.path.getsize(OUT), len(data)))


if __name__ == "__main__":
    main()
