"""Regenerate tests/golden/yuv_out_golden.npz: libyuv's own planes (the reference's rgba8ToNv12 / rgba8ToNv21 / rgba8ToI420 = ABGRToNV12 /
ABGRToNV21 / ABGRToI420, through oracle/_ref/libyuv_out_ref.so, built by oracle/yuv_out.mk from the reference checkout).

- "dense": one 2 x (2 * K) RGBA8 frame of uniform 2 x 2 blocks, block k taking the k-th triple of {0, 5, ..., 255}^3 (K = 52^3). The Y,
  U and V of each triple are stored once (dense_y / dense_u / dense_v, [K]); NV12, NV21 and I420 give the same samples (checked here).
- "random": one 2 x 16384 random RGBA8 frame (random_rgba), i.e. 8192 non-uniform blocks, and its planes per format.
- "odd": random RGBA8 frames of 1 x 1, 1 x 2, 2 x 1, 3 x 5 and 33 x 17 (H x W), whose last chroma column / row covers one pixel column /
  row, and their planes per format: odd_<h>x<w>_rgba and odd_<h>x<w>_<format>_y / _c1 / _c2 (I420 only).

    python tests/golden/make_yuv_out_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import yuv, yuv_out  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "yuv_out_golden.npz")
ODD = [(1, 1), (1, 2), (2, 1), (3, 5), (33, 17)]
LEVELS = np.arange(0, 256, 5)


def dense_frame():
    """The 2 x (2 * K) frame of uniform blocks, block k = (R, G, B) of triple k (R slowest), alpha 255."""
    r, g, b = (a.ravel() for a in np.meshgrid(LEVELS, LEVELS, LEVELS, indexing="ij"))
    px = np.stack([r, g, b, np.full_like(r, 255)], axis=-1).astype(np.uint8)
    return np.ascontiguousarray(np.broadcast_to(np.repeat(px, 2, axis=0)[None], (2, 2 * len(px), 4)))


def planes(prefix, fmt, data, rgba):
    y, c1, c2 = yuv_out.libyuv_from_rgba(fmt, rgba)
    data[prefix + "_y"], data[prefix + "_c1"] = y, c1
    if c2 is not None:
        data[prefix + "_c2"] = c2


def main():
    if yuv_out.libyuv() is None:
        sys.exit("oracle/_ref/libyuv_out_ref.so is missing: run `make -C oracle -f yuv_out.mk yuv_out` with the reference checkout present")
    data = {}
    frame = dense_frame()
    ys, us, vs = [], [], []
    for fmt in yuv.FORMATS:
        y, c1, c2 = yuv_out.libyuv_from_rgba(fmt, frame)
        u, v = (c1, c2) if fmt == "i420" else ((c1[:, 0::2], c1[:, 1::2]) if fmt == "nv12" else (c1[:, 1::2], c1[:, 0::2]))
        assert (y[:, 0::2] == y[:, 1::2]).all() and (y[0] == y[1]).all()
        ys.append(y[0, 0::2]), us.append(u[0]), vs.append(v[0])
    assert all(np.array_equal(ys[0], a) for a in ys) and all(np.array_equal(us[0], a) for a in us) and all(np.array_equal(vs[0], a) for a in vs)
    data["dense_y"], data["dense_u"], data["dense_v"] = ys[0], us[0], vs[0]
    rng = np.random.default_rng(1744)
    data["random_rgba"] = rng.integers(0, 256, (2, 16384, 4), dtype=np.uint8)
    for fmt in yuv.FORMATS:
        planes("random_" + fmt, fmt, data, data["random_rgba"])
    for h, w in ODD:
        k = "odd_%dx%d" % (h, w)
        data[k + "_rgba"] = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        for fmt in yuv.FORMATS:
            planes("%s_%s" % (k, fmt), fmt, data, data[k + "_rgba"])
    np.savez_compressed(OUT, **data)
    print("wrote %s (%d bytes, %d arrays)" % (OUT, os.path.getsize(OUT), len(data)))


if __name__ == "__main__":
    main()
