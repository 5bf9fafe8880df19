"""TEST INFRASTRUCTURE - numpy restatement of the reference's 8-bit frame conversion: nv12ToRgba8 / nv21ToRgba8 / i420ToRgba8
(core/src/image.cpp:1076-1136), i.e. libyuv's integer YuvPixel (row_common.cc:1444-1484, the portable C rows of libyuv 1744) with
its chroma siting (pixel (x, y) takes chroma sample (x // 2, y // 2)). tests/test_frames_cpu.py holds it to libyuv itself
(tests/golden/yuv_golden.npz, and oracle/_ref/libyuv_ref.so where it is built); the GPU tests then use it to make the RGBA8 image that
snnb_model_submit_image is fed."""
import ctypes as C
import os

import numpy as np

# libyuv row_common.cc:1115-1358: YG, YGB, UB, UG, VG, VR of kYuvI601Constants and kYuvH709Constants
MATRICES = {"bt601": (18997, -1160, -128, 25, 52, -102), "bt709": (18997, -1160, -128, 14, 34, -115)}
FORMATS = ("nv12", "nv21", "i420")


def yuv_pixel(y, u, v, matrix="bt601"):
    """RGBA8 of (Y, U, V) samples of any (equal) shape: [..., 4] uint8, alpha 255."""
    yg, ygb, ub, ug, vg, vr = MATRICES[matrix]
    bb, bg, br = ub * 128 + ygb, ug * 128 + vg * 128 + ygb, vr * 128 + ygb
    y, u, v = (np.asarray(a).astype(np.int64) for a in (y, u, v))
    y1 = ((y * 0x0101 * yg) & 0xFFFFFFFF) >> 16
    out = np.empty(y.shape + (4,), np.uint8)
    out[..., 0] = np.clip((-(v * vr) + y1 + br) >> 6, 0, 255)
    out[..., 1] = np.clip((-(u * ug + v * vg) + y1 + bg) >> 6, 0, 255)
    out[..., 2] = np.clip((-(u * ub) + y1 + bb) >> 6, 0, 255)
    out[..., 3] = 255
    return out


def chroma_shape(height, width):
    """Rows and columns of a 4:2:0 chroma plane (odd sizes round up, as libyuv)."""
    return (height + 1) // 2, (width + 1) // 2


def frames_to_rgba(fmt, y, c1, c2=None, matrix="bt601"):
    """RGBA8 frames [..., H, W, 4] from the planes of `fmt`: y [..., H, W]; NV12 / NV21: c1 the interleaved UV / VU plane
    [..., ceil(H/2), >= 2 * ceil(W/2)]; I420: c1 = U, c2 = V, [..., ceil(H/2), >= ceil(W/2)]. Planes may be wider than their rows."""
    y = np.asarray(y)
    h, w = y.shape[-2:]
    ch, cw = chroma_shape(h, w)
    if fmt in ("nv12", "nv21"):
        c = np.asarray(c1)[..., :ch, :2 * cw]
        first, second = c[..., 0::2], c[..., 1::2]
        u, v = (first, second) if fmt == "nv12" else (second, first)
    elif fmt == "i420":
        u, v = np.asarray(c1)[..., :ch, :cw], np.asarray(c2)[..., :ch, :cw]
    else:
        raise ValueError("unknown frame format %r" % (fmt,))
    up = np.repeat(np.repeat(u, 2, axis=-2), 2, axis=-1)[..., :h, :w]
    vp = np.repeat(np.repeat(v, 2, axis=-2), 2, axis=-1)[..., :h, :w]
    return yuv_pixel(y, up, vp, matrix)


def planes_from_yuv(fmt, y, u, v):
    """The planes of `fmt` for full-size Y and chroma-size U, V arrays (the inverse of what frames_to_rgba reads): (y, c1, c2)."""
    if fmt == "i420":
        return y, u, v
    c = np.empty(u.shape[:-1] + (2 * u.shape[-1],), np.uint8)
    c[..., 0::2], c[..., 1::2] = (u, v) if fmt == "nv12" else (v, u)
    return y, c, None


LIBYUV_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libyuv_ref.so")
_libyuv = None


def libyuv():
    """oracle/_ref/libyuv_ref.so (oracle/yuv.mk), or None where it was not built."""
    global _libyuv
    if _libyuv is None and os.path.exists(LIBYUV_PATH):
        _libyuv = C.CDLL(LIBYUV_PATH)
    return _libyuv


def libyuv_to_rgba(fmt, y, c1, c2=None, matrix="bt601", bt601_rows=False):
    """libyuv's own RGBA8 of one frame (2-D planes), through yuv_shim.cpp. bt601_rows: BT.601 through the shim's row loop for NV12 / NV21
    instead of the public entry point."""
    lib = libyuv()
    y = np.ascontiguousarray(y, np.uint8)
    h, w = y.shape
    dst = np.zeros((h, w, 4), np.uint8)
    sel = 2 if bt601_rows else (1 if matrix == "bt709" else 0)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    c1 = np.ascontiguousarray(c1, np.uint8)
    if fmt == "i420":
        c2 = np.ascontiguousarray(c2, np.uint8)
        rc = lib.yuv_i420_to_rgba(ptr(y), w, ptr(c1), c1.shape[1], ptr(c2), c2.shape[1], ptr(dst), 4 * w, w, h, sel)
    else:
        fn = lib.yuv_nv12_to_rgba if fmt == "nv12" else lib.yuv_nv21_to_rgba
        rc = fn(ptr(y), w, ptr(c1), c1.shape[1], ptr(dst), 4 * w, w, h, sel)
    assert rc == 0, "libyuv returned %d" % rc
    return dst
