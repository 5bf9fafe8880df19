"""The 10-bit frame path (P010) and the BT.2020 / full-range BT.601 matrices without a GPU: oracle/yuv10.py held to libyuv's own rows
(exhaustively where oracle/_ref/libyuv10_ref.so is built, else on tests/golden/yuv10_golden.npz), the P010 output restatement's
invariants, and the header's new values against the ctypes mirror."""
import os
import re

import numpy as np
import pytest

from oracle import yuv, yuv10
from shadernn_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "yuv10_golden.npz")
need_libyuv = pytest.mark.skipif(yuv10.libyuv() is None, reason="oracle/_ref/libyuv10_ref.so not built (no reference checkout)")


@pytest.mark.parametrize("matrix", list(yuv10.MATRICES))
def test_golden_10bit_rows(matrix):
    g = np.load(GOLDEN)
    y, u, v = g["y10_" + matrix], g["u10_" + matrix], g["v10_" + matrix]
    got = yuv10.ar30(*yuv10.yuv_pixel16(y, np.repeat(u, 2), np.repeat(v, 2), matrix))
    assert np.array_equal(got, g["ar30_" + matrix])


@pytest.mark.parametrize("matrix", ["bt2020", "jpeg"])
def test_golden_8bit_rows_new_matrices(matrix):
    g = np.load(GOLDEN)
    y, u, v = g["y8_" + matrix], g["u8_" + matrix], g["v8_" + matrix]
    assert np.array_equal(yuv10.yuv_pixel(y, np.repeat(u, 2), np.repeat(v, 2), matrix), g["rgba_" + matrix])


@need_libyuv
@pytest.mark.parametrize("matrix", list(yuv10.MATRICES))
def test_10bit_restatement_equals_libyuv_for_every_input(matrix):
    # every (Y10, U, V) the row can see: U and V reach it as U10 >> 2, so each 8-bit pair is fed with low bits that vary with V and U
    y = np.repeat(np.arange(1024, dtype=np.uint16)[None], 256, axis=0).reshape(-1)  # 1024 Y per V, in pairs sharing one chroma sample
    vv = np.repeat(np.arange(256, dtype=np.int64), 512)
    for u8 in range(256):
        u10 = ((u8 << 2) | (vv & 3)).astype(np.uint16)
        v10 = ((vv << 2) | (u8 & 3)).astype(np.uint16)
        want = yuv10.libyuv_i210_ar30(y, u10, v10, matrix)
        got = yuv10.ar30(*yuv10.yuv_pixel16(y, np.repeat(u10, 2), np.repeat(v10, 2), matrix))
        assert np.array_equal(got, want), "U %d" % u8


@need_libyuv
@pytest.mark.parametrize("matrix", list(yuv10.MATRICES))
def test_10bit_chroma_truncates_to_8_bits(matrix):
    rng = np.random.default_rng(7)
    y = rng.integers(0, 1024, 4096).astype(np.uint16)
    u, v = rng.integers(0, 1024, 2048).astype(np.uint16), rng.integers(0, 1024, 2048).astype(np.uint16)
    assert np.array_equal(yuv10.libyuv_i210_ar30(y, u, v, matrix), yuv10.libyuv_i210_ar30(y, u & 0x3FC, v & 0x3FC, matrix))


@need_libyuv
@pytest.mark.parametrize("matrix", list(yuv10.MATRICES))
def test_8bit_restatement_equals_libyuv_over_all_triples(matrix):
    y = np.tile(np.arange(256, dtype=np.uint8), 256)  # 256 Y per V, in pairs
    v = np.repeat(np.arange(256, dtype=np.uint8), 128)
    for u8 in range(256):
        u = np.full(v.shape, u8, np.uint8)
        want = yuv10.libyuv_i422_argb(y, u, v, matrix)
        assert np.array_equal(yuv10.yuv_pixel(y, np.repeat(u, 2), np.repeat(v, 2), matrix), want), "U %d" % u8
    if matrix in yuv.MATRICES:  # the existing tables agree with oracle/yuv.py
        rng = np.random.default_rng(3)
        t = [rng.integers(0, 256, 5000) for _ in range(3)]
        assert np.array_equal(yuv10.yuv_pixel(*t, matrix), yuv.yuv_pixel(*t, matrix))


def test_p010_words_and_chroma_siting_at_odd_sizes():
    rng = np.random.default_rng(11)
    for h, w in [(1, 1), (3, 5), (7, 2), (2, 9)]:
        ch, cw = yuv.chroma_shape(h, w)
        y, u, v = rng.integers(0, 1024, (1, h, w)), rng.integers(0, 1024, (1, ch, cw)), rng.integers(0, 1024, (1, ch, cw))
        t = yuv10.texels(y, u, v, "bt2020")
        for yy in range(h):
            for xx in range(w):
                r, g, b = yuv10.yuv_pixel16(y[0, yy, xx], u[0, yy // 2, xx // 2], v[0, yy // 2, xx // 2], "bt2020")
                assert tuple(t[0, yy, xx]) == (r * 0.25, g * 0.25, b * 0.25, 255.0)
    y, u, v = rng.integers(0, 1024, (2, 4, 6)), rng.integers(0, 1024, (2, 2, 3)), rng.integers(0, 1024, (2, 2, 3))
    low = rng.integers(0, 64, (2, 6, 6))
    words = yuv10.p010_pack(y, u, v, low)
    assert words.dtype == np.uint16 and words.shape == (2, 6, 6)
    for a, b in zip(yuv10.p010_split(words), (y, u, v)):
        assert np.array_equal(a, b)
    assert np.array_equal(words[:, 4:, 0::2] >> 6, u) and np.array_equal(words[:, 4:, 1::2] >> 6, v)  # U first


def test_texels_are_exact_quarters_and_extremes_clamp():
    r, g, b = yuv10.yuv_pixel16(np.array([0, 1023, 64, 940]), np.array([0, 1023, 512, 512]), np.array([1023, 0, 512, 512]), "bt601")
    for c in (r, g, b):
        assert c.min() >= 0 and c.max() <= 1023
    assert max(r[2], g[2], b[2]) <= 1 and min(r[3], g[3], b[3]) >= 1016  # limited-range black (Y10 64) and white (940)
    t = yuv10.texels(np.arange(1024).reshape(1, 32, 32), np.full((1, 16, 16), 512), np.full((1, 16, 16), 512), "jpeg")
    assert np.array_equal(t * 4, np.rint(t * 4))


def test_p010_output_restatement_invariants():
    rng = np.random.default_rng(5)
    for c in (1, 3, 4):
        out = rng.uniform(-40, 300, (2, 9, 7, c)).astype(np.float32)
        for hw, linear in [((9, 7), True), ((13, 11), True), ((5, 3), False), ((1, 1), True), ((6, 10), False)]:
            y, u, v = yuv10.frames_out(out, hw, linear, 1.0, 0.0)
            assert y.shape == (2,) + hw and u.shape == v.shape == (2,) + yuv.chroma_shape(*hw)
            assert y.min() >= 64 and y.max() <= 943
            assert u.min() >= 64 and u.max() <= 960 and v.min() >= 64 and v.max() <= 960
    # M10 at equal size is the identity resize; 4x the 8-bit scale, clamped
    q = yuv10.quant10(np.array([-1.0, 0.0, 0.125, 100.0, 255.75, 400.0], np.float32), 1.0, 0.0)
    assert list(q) == [0.0, 0.0, 0.0, 400.0, 1023.0, 1023.0]
    # odd edges: a last odd column averages its two rows; a last odd row pairs with itself
    m = np.zeros((1, 3, 3, 3), np.int64)
    m[0, :, :, 0] = [[100, 200, 300], [400, 500, 600], [700, 800, 900]]
    y, u, v = yuv10.rgb10_to_yuv10(m)
    rr = np.array([[(100 + 200 + 400 + 500) >> 2, (300 + 600) >> 1], [(700 + 800 + 700 + 800) >> 2, (900 + 900) >> 1]])
    assert np.array_equal(v[0], (112 * rr + 0x20080) >> 8) and np.array_equal(u[0], (-38 * rr + 0x20080) >> 8)
    # the words: value << 6 with the low 6 bits zero
    words = yuv10.p010_pack(y[:, :2, :2], u[:, :1, :1], v[:, :1, :1])
    assert not (words & 0x3F).any()


def test_luma_out_resizes_chroma_plane_to_plane():
    rng = np.random.default_rng(8)
    out = rng.uniform(0, 255, (1, 6, 8, 1)).astype(np.float32)
    u, v = rng.integers(0, 1024, (1, 3, 4)), rng.integers(0, 1024, (1, 3, 4))
    y, uo, vo = yuv10.luma_out(out, u, v, (6, 8), True, 1.0, 0.0)
    assert np.array_equal(uo, u) and np.array_equal(vo, v)  # equal chroma size: a copy
    assert np.array_equal(y, yuv10.quant10(out[..., 0], 1.0, 0.0))
    y, uo, vo = yuv10.luma_out(out, u, v, (11, 15), True, 1.0, 0.0)
    assert uo.shape == (1, 6, 8) and uo.min() >= u.min() and uo.max() <= u.max()


def test_header_values_match_the_ctypes_mirror():
    h = open(os.path.join(ROOT, "include", "snnb.h")).read()

    def value(name):
        return int(re.search(r"\b%s\s*=\s*(0x[0-9a-fA-F]+|\d+)" % name, h).group(1), 0)
    assert value("SNNB_FRAME_P010") == _lib.FRAME_P010 == 16
    assert value("SNNB_YUV_BT2020") == _lib.YUV_BT2020 == 9
    assert value("SNNB_YUV_FULL_RANGE") == _lib.YUV_FULL_RANGE == 0x100
    assert value("SNNB_FRAME_RGBA8") == _lib.FRAME_RGBA8 and value("SNNB_YUV_BT709") == _lib.YUV_BT709
    from shadernn_b200 import core
    assert core.MixedInferenceCore._FRAME_FORMATS["p010"] == 16
    assert core.MixedInferenceCore._YUV_MATRICES["jpeg"] == 0x100 and core.MixedInferenceCore._YUV_MATRICES["bt2020"] == 9
