"""TEST INFRASTRUCTURE - numpy restatement of the output side of the reference's frame pipeline (snnb_model_transform_frames): the
model-size RGBA8 image resized as ImageTexture::resize (resize_rgba8), then rgba8ToNv12 / rgba8ToNv21 / rgba8ToI420 (core/src/image.cpp:
1051-1100), i.e. libyuv 1744's ABGRToNV12 / ABGRToNV21 / ABGRToI420 with its portable C rows (row_common.cc:423-473: RGBToY, RGBToU,
RGBToV and MAKEROWY's 2 x 2 average). tests/test_frames_out_cpu.py holds it to libyuv itself (tests/golden/yuv_out_golden.npz, and
oracle/_ref/libyuv_out_ref.so where it is built); the GPU tests then use it to make the frames the device must write."""
import ctypes as C
import os

import numpy as np

from oracle import oracle, yuv


def rgba_to_frames(fmt, rgba):
    """The planes (y, c1, c2) of `fmt` (as yuv.planes_from_yuv lays them out) of RGBA8 frames [..., H, W, 4], any H, W >= 1.
    Y = (66 R + 129 G + 25 B + 0x1080) >> 8; each chroma sample averages its 2 x 2 block per component as (a + b + c + d) >> 2, an odd
    last column as (a + b) >> 1 over its two rows, and an odd last row is paired with itself (libyuv passes stride 0);
    U = (112 B - 74 G - 38 R + 0x8080) >> 8, V = (112 R - 94 G - 18 B + 0x8080) >> 8."""
    p = np.asarray(rgba).astype(np.int64)
    h, w = p.shape[-3:-1]
    y = ((66 * p[..., 0] + 129 * p[..., 1] + 25 * p[..., 2] + 0x1080) >> 8).astype(np.uint8)
    if h % 2:
        p = np.concatenate([p, p[..., -1:, :, :]], axis=-3)
    rows = p[..., 0::2, :, :3] + p[..., 1::2, :, :3]  # [..., ceil(H/2), W, 3]: the two rows of each chroma sample
    ch, cw = yuv.chroma_shape(h, w)
    avg = np.empty(rows.shape[:-2] + (cw, 3), np.int64)
    even = w // 2 * 2
    avg[..., :w // 2, :] = (rows[..., 0:even:2, :] + rows[..., 1:even:2, :]) >> 2
    if w % 2:
        avg[..., -1, :] = rows[..., -1, :] >> 1
    r, g, b = avg[..., 0], avg[..., 1], avg[..., 2]
    u = ((112 * b - 74 * g - 38 * r + 0x8080) >> 8).astype(np.uint8)
    v = ((112 * r - 94 * g - 18 * b + 0x8080) >> 8).astype(np.uint8)
    return yuv.planes_from_yuv(fmt, y, u, v)


def resize_rgba8(m, out_hw, linear=True):
    """ImageTexture::resize of RGBA8 images [N, h, w, 4] to out_hw: the identity at equal size; otherwise the taps and float32 blend of
    oracle.resize_normalize (two lerps along x, then one along y, every step rounded to float32), then rint."""
    m = np.asarray(m, np.uint8)
    if tuple(m.shape[1:3]) == tuple(out_hw):
        return m.copy()
    v = oracle.resize_normalize(m, out_hw, [0.0] * 4, [1.0] * 4, linear=linear)
    return np.rint(v).astype(np.uint8)


LIBYUV_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libyuv_out_ref.so")
_libyuv = None


def libyuv():
    """oracle/_ref/libyuv_out_ref.so (oracle/yuv_out.mk), or None where it was not built."""
    global _libyuv
    if _libyuv is None and os.path.exists(LIBYUV_PATH):
        _libyuv = C.CDLL(LIBYUV_PATH)
    return _libyuv


def libyuv_from_rgba(fmt, rgba):
    """libyuv's own planes (y, c1, c2) of one RGBA8 frame [H, W, 4], through yuv_out_shim.cpp."""
    lib = libyuv()
    src = np.ascontiguousarray(rgba, np.uint8)
    h, w = src.shape[:2]
    ch, cw = yuv.chroma_shape(h, w)
    y = np.zeros((h, w), np.uint8)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    if fmt == "i420":
        c1, c2 = np.zeros((ch, cw), np.uint8), np.zeros((ch, cw), np.uint8)
        rc = lib.yuv_rgba_to_i420(ptr(src), 4 * w, ptr(y), w, ptr(c1), cw, ptr(c2), cw, w, h)
    else:
        c1, c2 = np.zeros((ch, 2 * cw), np.uint8), None
        fn = lib.yuv_rgba_to_nv12 if fmt == "nv12" else lib.yuv_rgba_to_nv21
        rc = fn(ptr(src), 4 * w, ptr(y), w, ptr(c1), 2 * cw, w, h)
    assert rc == 0, "libyuv returned %d" % rc
    return y, c1, c2
