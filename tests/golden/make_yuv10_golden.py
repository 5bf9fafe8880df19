"""Writes tests/golden/yuv10_golden.npz from libyuv's own rows (oracle/_ref/libyuv10_ref.so, built by oracle/yuv10.mk from the reference's
vendored libyuv 1744): seeded samples of I210ToAR30Row_C with each of the four tables, and of the 8-bit I422ToARGBRow_C with the
BT.2020 and JPEG tables. tests/test_p010_cpu.py compares oracle/yuv10.py with it where the library is absent.

    python tests/golden/make_yuv10_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import yuv10  # noqa: E402

PAIRS = 10000  # chroma samples per table; two luma samples each


def samples(seed, bits):
    rng = np.random.default_rng(seed)
    top = 1 << bits
    return (rng.integers(0, top, 2 * PAIRS), rng.integers(0, top, PAIRS), rng.integers(0, top, PAIRS))


def main():
    assert yuv10.libyuv() is not None, "oracle/_ref/libyuv10_ref.so is missing: run oracle/yuv10.mk first"
    out = {}
    for k, matrix in enumerate(yuv10.MATRICES):
        y, u, v = (a.astype(np.uint16) for a in samples(100 + k, 10))
        out["y10_" + matrix], out["u10_" + matrix], out["v10_" + matrix] = y, u, v
        out["ar30_" + matrix] = yuv10.libyuv_i210_ar30(y, u, v, matrix)
    for k, matrix in enumerate(("bt2020", "jpeg")):
        y, u, v = (a.astype(np.uint8) for a in samples(200 + k, 8))
        out["y8_" + matrix], out["u8_" + matrix], out["v8_" + matrix] = y, u, v
        out["rgba_" + matrix] = yuv10.libyuv_i422_argb(y, u, v, matrix)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "yuv10_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main()
