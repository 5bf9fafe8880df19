"""TEST INFRASTRUCTURE - numpy restatement of the 10-bit frame path (SNNB_FRAME_P010) and of the BT.2020 and full-range BT.601 (JPEG)
matrices, as include/snnb.h defines them.

Input: libyuv 1744's YuvPixel16 (row_common.cc:1531-1573: Y with 10 bits, U and V truncated to 8) and StoreAR30's Clamp10(c >> 4)
(row_common.cc:1713-1750), the texel R10 * 0.25, then ImageTexture::resize's taps with every + - * of the blend rounded to float32 on
its own, and (x - mean) * norm. Output: M10 = clamp(rint(4 * (v * scale + offset)), 0, 1023), the same resize and rint, then the 8-bit
BT.601 coefficients with the 10-bit offsets. The 8-bit rows with the new matrices are libyuv's YuvPixel (oracle/yuv.py) with their
constants. tests/test_p010_cpu.py holds this to libyuv's rows (tests/golden/yuv10_golden.npz, and oracle/_ref/libyuv10_ref.so where it
is built); the GPU tests then use it to make the model inputs and the words the device must write."""
import ctypes as C
import os

import numpy as np

from oracle import yuv

# libyuv row_common.cc:1115-1420: YG, YGB, UB, UG, VG, VR of kYuvI601Constants, kYuvH709Constants, kYuv2020Constants, kYuvJPEGConstants
MATRICES = {"bt601": (18997, -1160, -128, 25, 52, -102), "bt709": (18997, -1160, -128, 14, 34, -115),
            "bt2020": (19003, -1160, -128, 12, 42, -107), "jpeg": (16320, 32, -113, 22, 46, -90)}
# the shim's table index of each matrix
TABLE = {"bt601": 0, "bt709": 1, "bt2020": 2, "jpeg": 3}
f32 = np.float32


def _biases(matrix):
    yg, ygb, ub, ug, vg, vr = MATRICES[matrix]
    return yg, ub, ug, vg, vr, ub * 128 + ygb, ug * 128 + vg * 128 + ygb, vr * 128 + ygb


def yuv_pixel(y, u, v, matrix):
    """libyuv's 8-bit YuvPixel with any of the four matrices: RGBA8 [..., 4] uint8, alpha 255 (oracle/yuv.py's, for every table)."""
    yg, ub, ug, vg, vr, bb, bg, br = _biases(matrix)
    y, u, v = (np.asarray(a).astype(np.int64) for a in (y, u, v))
    y1 = ((y * 0x0101 * yg) & 0xFFFFFFFF) >> 16
    out = np.empty(y.shape + (4,), np.uint8)
    out[..., 0] = np.clip((-(v * vr) + y1 + br) >> 6, 0, 255)
    out[..., 1] = np.clip((-(u * ug + v * vg) + y1 + bg) >> 6, 0, 255)
    out[..., 2] = np.clip((-(u * ub) + y1 + bb) >> 6, 0, 255)
    out[..., 3] = 255
    return out


def yuv_pixel16(y10, u10, v10, matrix):
    """YuvPixel16 + StoreAR30 of 10-bit samples: (R10, G10, B10) int64 arrays. U and V are truncated to 8 bits (u10 >> 2)."""
    yg, ub, ug, vg, vr, bb, bg, br = _biases(matrix)
    y, u, v = (np.asarray(a).astype(np.int64) for a in (y10, u10, v10))
    u, v = np.minimum(u >> 2, 255), np.minimum(v >> 2, 255)
    y1 = (((y << 6) * yg) & 0xFFFFFFFF) >> 16
    r = np.clip((-(v * vr) + y1 + br) >> 4, 0, 1023)
    g = np.clip((-(u * ug + v * vg) + y1 + bg) >> 4, 0, 1023)
    b = np.clip((-(u * ub) + y1 + bb) >> 4, 0, 1023)
    return r, g, b


def ar30(r, g, b):
    """StoreAR30's word: B | G << 10 | R << 20 | 0xC0000000."""
    return (np.asarray(b, np.uint32) | (np.asarray(g, np.uint32) << 10) | (np.asarray(r, np.uint32) << 20) | np.uint32(0xC0000000)).astype(np.uint32)


def p010_pack(y10, u10, v10, low=0):
    """P010 frames [N, H * 3 // 2, W] uint16 (H, W even) of 10-bit Y [N, H, W] and U, V [N, H/2, W/2]: word = value << 6 | low, `low`
    (an int or an array of the frame's shape) filling the 6 ignored bits."""
    y10, u10, v10 = (np.asarray(a).astype(np.uint16) for a in (y10, u10, v10))
    n, h, w = y10.shape
    c = np.empty((n, h // 2, w), np.uint16)
    c[..., 0::2], c[..., 1::2] = u10, v10
    return ((np.concatenate([y10, c], axis=1) << 6) | (np.asarray(low, np.uint16) & 0x3F)).astype(np.uint16)


def p010_split(words):
    """The 10-bit Y [N, H, W] and U, V [N, H/2, W/2] of P010 frames [N, H * 3 // 2, W] (the words' top 10 bits)."""
    s = np.asarray(words).astype(np.uint16) >> 6
    h = s.shape[1] // 3 * 2
    return s[:, :h].astype(np.int64), s[:, h:, 0::2].astype(np.int64), s[:, h:, 1::2].astype(np.int64)


def texels(y10, u10, v10, matrix):
    """The float32 RGBA texels [N, H, W, 4] of 10-bit frames: pixel (x, y) takes chroma (x // 2, y // 2); R10 * 0.25 ..., alpha 255."""
    h, w = y10.shape[-2:]
    up = np.repeat(np.repeat(u10, 2, axis=-2), 2, axis=-1)[..., :h, :w]
    vp = np.repeat(np.repeat(v10, 2, axis=-2), 2, axis=-1)[..., :h, :w]
    r, g, b = yuv_pixel16(y10, up, vp, matrix)
    out = np.empty(np.shape(y10) + (4,), f32)
    out[..., 0], out[..., 1], out[..., 2] = (a.astype(f32) * f32(0.25) for a in (r, g, b))
    out[..., 3] = 255.0
    return out


def luma_texels(y10):
    """The float32 texels [N, H, W, 4] of the Y plane of P010 frames: every component Y10 * 0.25."""
    t = np.asarray(y10).astype(f32) * f32(0.25)
    return np.repeat(t[..., None], 4, axis=-1)


def resize(img, out_hw, linear=True):
    """ImageTexture::resize of float32 images [N, h, w, C] to out_hw: the identity at equal size; else the taps of
    oracle.resize_normalize with every + - * of the blend rounded to float32 on its own (blend_rn)."""
    img = np.asarray(img, f32)
    n, sh, sw, c = img.shape
    oh, ow = out_hw
    if (sh, sw) == (oh, ow):
        return img.copy()
    fx = (np.arange(ow, dtype=f32) + f32(0.5)) / f32(ow) * f32(sw)
    fy = (np.arange(oh, dtype=f32) + f32(0.5)) / f32(oh) * f32(sh)
    if not linear:
        return img[:, np.minimum(fy.astype(int), sh - 1)][:, :, np.minimum(fx.astype(int), sw - 1)]
    sx, sy = fx - f32(0.5), fy - f32(0.5)
    x0f, y0f = np.floor(sx), np.floor(sy)
    ax, ay = (sx - x0f).astype(f32)[None, None, :, None], (sy - y0f).astype(f32)[None, :, None, None]
    x0, x1 = np.clip(x0f.astype(int), 0, sw - 1), np.clip(x0f.astype(int) + 1, 0, sw - 1)
    y0, y1 = np.clip(y0f.astype(int), 0, sh - 1), np.clip(y0f.astype(int) + 1, 0, sh - 1)
    p00, p01 = img[:, y0][:, :, x0], img[:, y0][:, :, x1]
    p10, p11 = img[:, y1][:, :, x0], img[:, y1][:, :, x1]
    top = p00 + ax * (p01 - p00)
    bot = p10 + ax * (p11 - p10)
    return (top + ay * (bot - top)).astype(f32)


def normalize(v, c, mean4, norm4):
    """(v - mean4[k]) * norm4[k] of the first c components, in float32: the model input [N, H, W, c]."""
    mean = np.array([mean4[k & 3] for k in range(c)], f32)
    norm = np.array([norm4[k & 3] for k in range(c)], f32)
    return ((np.asarray(v, f32)[..., :c] - mean) * norm).astype(f32)


def model_input(tex, out_hw, c, linear=True, mean4=(0.0,) * 4, norm4=(1.0,) * 4):
    """The model input [N, H, W, c] of P010 texels (texels() or luma_texels())."""
    return normalize(resize(tex, out_hw, linear), c, mean4, norm4)


def quant10(v, scale, offset):
    """M10 of model output values: clamp(rint(4 * (v * scale + offset)), 0, 1023), every step in float32."""
    v = np.asarray(v, f32)
    return np.clip(np.rint(f32(4.0) * ((v * f32(scale)).astype(f32) + f32(offset)).astype(f32)), 0, 1023).astype(f32)


def m10(out, scale, offset):
    """The model-size 10-bit RGBA image [N, h, w, 4] (float32 of integers) of output 0 [N, h, w, C]: C = 4 RGBA, 3 RGB + alpha 255, 1
    grey + alpha 255."""
    out = np.asarray(out, f32)
    q = quant10(out, scale, offset)
    m = np.full(out.shape[:3] + (4,), 255.0, f32)
    if out.shape[3] == 1:
        m[..., 0] = m[..., 1] = m[..., 2] = q[..., 0]
    else:
        m[..., :3] = q[..., :3]
        if out.shape[3] == 4:
            m[..., 3] = q[..., 3]
    return m


def rgb10_to_yuv10(p):
    """Y10 [..., H, W] and U10, V10 [..., ceil(H/2), ceil(W/2)] of 10-bit RGB[A] [..., H, W, >= 3] with yuv_out.rgba_to_frames' 2 x 2 rules
    (odd last column averaged over its two rows, odd last row paired with itself) and the 10-bit offsets."""
    p = np.asarray(p).astype(np.int64)
    h, w = p.shape[-3:-1]
    y = (66 * p[..., 0] + 129 * p[..., 1] + 25 * p[..., 2] + 0x4080) >> 8
    if h % 2:
        p = np.concatenate([p, p[..., -1:, :, :]], axis=-3)
    rows = p[..., 0::2, :, :3] + p[..., 1::2, :, :3]
    cw = (w + 1) // 2
    avg = np.empty(rows.shape[:-2] + (cw, 3), np.int64)
    even = w // 2 * 2
    avg[..., :w // 2, :] = (rows[..., 0:even:2, :] + rows[..., 1:even:2, :]) >> 2
    if w % 2:
        avg[..., -1, :] = rows[..., -1, :] >> 1
    r, g, b = avg[..., 0], avg[..., 1], avg[..., 2]
    u = (112 * b - 74 * g - 38 * r + 0x20080) >> 8
    v = (112 * r - 94 * g - 18 * b + 0x20080) >> 8
    return y, u, v


def frames_out(out, out_hw, linear, scale, offset):
    """transform_frames' P010 output of model output 0 [N, h, w, C] float32: (Y10, U10, V10) at out_hw."""
    return rgb10_to_yuv10(np.rint(resize(m10(out, scale, offset), out_hw, linear)))


def resize_plane(p, out_hw, linear=True):
    """ImageTexture::resize of planes of integers [N, h, w] to out_hw (blend_rn, then rint): int64."""
    return np.rint(resize(np.asarray(p, f32)[..., None], out_hw, linear))[..., 0].astype(np.int64)


def luma_out(out, u10, v10, out_hw, linear, scale, offset):
    """transform_luma's P010 output: Y10 from M10 of the 1-channel output [N, h, w, 1], and the source U10, V10 resized plane to plane."""
    y = resize_plane(quant10(np.asarray(out, f32)[..., 0], scale, offset), out_hw, linear)
    ch, cw = yuv.chroma_shape(*out_hw)
    return y, resize_plane(u10, (ch, cw), linear), resize_plane(v10, (ch, cw), linear)


LIBYUV_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libyuv10_ref.so")
_libyuv = None


def libyuv():
    """oracle/_ref/libyuv10_ref.so (oracle/yuv10.mk), or None where it was not built."""
    global _libyuv
    if _libyuv is None and os.path.exists(LIBYUV_PATH):
        _libyuv = C.CDLL(LIBYUV_PATH)
    return _libyuv


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def libyuv_i210_ar30(y10, u10, v10, matrix):
    """libyuv's I210ToAR30Row_C over one row: y10 [W] (W even), u10, v10 [W / 2] (uint16) -> AR30 words [W] uint32."""
    y, u, v = (np.ascontiguousarray(a, np.uint16) for a in (y10, u10, v10))
    dst = np.zeros(y.shape[0], np.uint32)
    assert libyuv().yuv10_i210_ar30_row(_ptr(y), _ptr(u), _ptr(v), _ptr(dst), y.shape[0], TABLE[matrix]) == 0
    return dst


def libyuv_i422_argb(y, u, v, matrix):
    """libyuv's 8-bit I422ToARGBRow_C over one row: y [W] (W even), u, v [W / 2] (uint8) -> RGBA8 [W, 4] (reordered from libyuv's B, G,
    R, A bytes)."""
    y, u, v = (np.ascontiguousarray(a, np.uint8) for a in (y, u, v))
    dst = np.zeros((y.shape[0], 4), np.uint8)
    assert libyuv().yuv10_i422_argb_row(_ptr(y), _ptr(u), _ptr(v), _ptr(dst), y.shape[0], TABLE[matrix]) == 0
    return dst[:, [2, 1, 0, 3]]
