"""snnb_model_transform_frames without a GPU: the numpy restatement of the reference's RGBA8 -> YUV conversion (oracle/yuv_out.py) equals
libyuv, the C struct and its ctypes mirror agree, and the entry point refuses a null model."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import yuv, yuv_out
from shadernn_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "yuv_out_golden.npz")
ODD = [(1, 1), (1, 2), (2, 1), (3, 5), (33, 17)]
FORMATS = ["nv12", "nv21", "i420"]
no_libyuv = pytest.mark.skipif(yuv_out.libyuv() is None, reason="oracle/_ref/libyuv_out_ref.so was not built (the reference checkout is absent)")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def assert_planes_equal(got, want, what):
    for i, (g, w) in enumerate(zip(got, want)):
        assert (g is None) == (w is None), (what, i)
        if g is not None:
            assert g.shape == w.shape and np.array_equal(g, w), (what, i)


def uv_of(fmt, c1, c2):
    if fmt == "i420":
        return c1, c2
    first, second = c1[..., 0::2], c1[..., 1::2]
    return (first, second) if fmt == "nv12" else (second, first)


def uniform_blocks(rgb):
    """A 2 x (2 * K) RGBA8 frame whose 2 x 2 block k is the triple rgb[k], alpha 255."""
    px = np.concatenate([rgb, np.full((len(rgb), 1), 255)], axis=1).astype(np.uint8)
    return np.ascontiguousarray(np.broadcast_to(np.repeat(px, 2, axis=0)[None], (2, 2 * len(px), 4)))


@pytest.mark.parametrize("fmt", FORMATS)
def test_restatement_equals_libyuv_golden_on_uniform_blocks(golden, fmt):
    levels = np.arange(0, 256, 5)
    rgb = np.stack([a.ravel() for a in np.meshgrid(levels, levels, levels, indexing="ij")], axis=1)
    y, c1, c2 = yuv_out.rgba_to_frames(fmt, uniform_blocks(rgb))
    u, v = uv_of(fmt, c1, c2)
    assert np.array_equal(y[0, 0::2], golden["dense_y"]) and np.array_equal(y[1, 1::2], golden["dense_y"])
    assert np.array_equal(u[0], golden["dense_u"]) and np.array_equal(v[0], golden["dense_v"])


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("key", ["random"] + ["odd_%dx%d" % hw for hw in ODD])
def test_restatement_equals_libyuv_golden(golden, fmt, key):
    want = tuple(golden.get("%s_%s_%s" % (key, fmt, p)) for p in ("y", "c1", "c2"))
    assert_planes_equal(yuv_out.rgba_to_frames(fmt, golden[key + "_rgba"]), want, key)


def test_golden_reaches_the_limits_of_limited_range(golden):
    assert golden["dense_y"].min() == 16 and golden["dense_y"].max() == 235
    assert golden["dense_u"].min() == 16 and golden["dense_u"].max() == 240
    assert golden["dense_v"].min() == 16 and golden["dense_v"].max() == 240


@no_libyuv
def test_restatement_equals_libyuv_on_every_rgb_triple():
    # all 2^24 (R, G, B) triples as uniform 2 x 2 blocks, 2^20 at a time
    k = np.arange(1 << 20)
    for chunk in range(16):
        t = (chunk << 20) | k
        rgb = np.stack([t >> 16, (t >> 8) & 255, t & 255], axis=1)
        frame = uniform_blocks(rgb)
        for fmt in FORMATS:
            assert_planes_equal(yuv_out.rgba_to_frames(fmt, frame), yuv_out.libyuv_from_rgba(fmt, frame), (fmt, chunk))


@no_libyuv
@pytest.mark.parametrize("fmt", FORMATS)
def test_restatement_equals_libyuv_on_random_blocks_and_odd_sizes(fmt):
    rng = np.random.default_rng(11)
    frame = rng.integers(0, 256, (2, 1 << 21, 4), dtype=np.uint8)  # 2^20 non-uniform blocks
    assert_planes_equal(yuv_out.rgba_to_frames(fmt, frame), yuv_out.libyuv_from_rgba(fmt, frame), "random")
    for h, w in ODD + [(7, 1), (1, 9), (45, 63)]:
        rgba = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        assert_planes_equal(yuv_out.rgba_to_frames(fmt, rgba), yuv_out.libyuv_from_rgba(fmt, rgba), (h, w))


def test_rgba_to_frames_takes_a_batch():
    rgba = np.random.default_rng(2).integers(0, 256, (3, 5, 7, 4), dtype=np.uint8)
    for fmt in FORMATS:
        batch = yuv_out.rgba_to_frames(fmt, rgba)
        for n in range(3):
            assert_planes_equal([None if p is None else p[n] for p in batch], yuv_out.rgba_to_frames(fmt, rgba[n]), (fmt, n))


def test_resize_rgba8_is_the_identity_at_equal_size():
    m = np.random.default_rng(3).integers(0, 256, (2, 9, 13, 4), dtype=np.uint8)
    for linear in (True, False):
        assert np.array_equal(yuv_out.resize_rgba8(m, (9, 13), linear), m)
    up = yuv_out.resize_rgba8(m, (18, 26), True)
    assert up.shape == (2, 18, 26, 4) and up.dtype == np.uint8
    assert np.array_equal(yuv_out.resize_rgba8(m, (18, 26), False), np.repeat(np.repeat(m, 2, axis=1), 2, axis=2))


PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "snnb.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(snnb_frames_out), offsetof(snnb_frames_out, format), offsetof(snnb_frames_out, width),
           offsetof(snnb_frames_out, height), offsetof(snnb_frames_out, plane), offsetof(snnb_frames_out, pitch), offsetof(snnb_frames_out, image_stride),
           offsetof(snnb_frames_out, linear_filter), offsetof(snnb_frames_out, scale), offsetof(snnb_frames_out, offset));
    return 0;
}
"""


def test_frames_out_layout_matches_the_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(PROBE)
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    sizes = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    F = _lib.FramesOut
    fields = ("format", "width", "height", "plane", "pitch", "image_stride", "linear_filter", "scale", "offset")
    assert [int(v) for v in sizes] == [C.sizeof(F)] + [getattr(F, f).offset for f in fields]


def test_transform_frames_refuses_a_null_model(built):
    lib = _lib.lib()
    f, o = _lib.Frames(), _lib.FramesOut()
    assert lib.snnb_model_transform_frames(None, C.byref(f), C.byref(o), None) != 0
    assert b"snnb_model_transform_frames: null model" in lib.snnb_last_error()
