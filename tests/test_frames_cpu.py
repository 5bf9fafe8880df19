"""snnb_model_run_frames / snnb_model_detect_frames without a GPU: the numpy restatement of the reference's frame conversion
(oracle/yuv.py) equals libyuv, the C struct and its ctypes mirror agree, and the entry points refuse cleanly."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import yuv
from shadernn_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "yuv_golden.npz")
ODD = [(1, 1), (3, 5), (33, 17)]


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("matrix", ["bt601", "bt709"])
@pytest.mark.parametrize("fmt", ["nv12", "nv21", "i420"])
def test_restatement_equals_libyuv_golden_on_every_uv_pair(golden, fmt, matrix):
    i = np.arange(65536)
    u, v = (i & 255).astype(np.uint8)[:, None], (i >> 8).astype(np.uint8)[:, None]
    y = ((np.arange(2 * 65536) * 37) & 255).astype(np.uint8)[:, None]
    assert len(np.unique(y)) == 256
    got = yuv.frames_to_rgba(fmt, *yuv.planes_from_yuv(fmt, y, u, v), matrix=matrix)[:, 0]
    assert np.array_equal(got, golden["pairs_rgba_" + matrix])


@pytest.mark.parametrize("matrix", ["bt601", "bt709"])
@pytest.mark.parametrize("fmt", ["nv12", "nv21", "i420"])
@pytest.mark.parametrize("hw", ODD)
def test_restatement_equals_libyuv_golden_on_odd_sizes(golden, fmt, matrix, hw):
    k = "odd_%dx%d" % hw
    planes = yuv.planes_from_yuv(fmt, golden[k + "_y"], golden[k + "_u"], golden[k + "_v"])
    assert np.array_equal(yuv.frames_to_rgba(fmt, *planes, matrix=matrix), golden["%s_%s_%s" % (k, fmt, matrix)])


def test_golden_reaches_black_white_and_saturation(golden):
    for m in ("bt601", "bt709"):
        assert np.array_equal(yuv.yuv_pixel([16, 235], [128, 128], [128, 128], m)[:, :3], [[0, 0, 0], [255, 255, 255]])
        rgba = golden["pairs_rgba_" + m]
        assert (rgba[:, :3] == 0).any() and (rgba[:, :3] == 255).any() and (rgba[:, 3] == 255).all()


@pytest.mark.skipif(yuv.libyuv() is None, reason="oracle/_ref/libyuv_ref.so was not built (the reference checkout is absent)")
@pytest.mark.parametrize("matrix", ["bt601", "bt709"])
def test_restatement_equals_libyuv_on_all_yuv_triples(matrix):
    # 2048 x 2048 chroma samples = every (U, V) pair 64 times; the 4 x 64 luma pixels under the samples of one pair take every Y
    cu, cv = np.meshgrid(np.arange(2048), np.arange(2048))
    pair = (cv * 2048 + cu) % 65536
    rep = (cv * 2048 + cu) // 65536  # 0..63
    u, v = (pair & 255).astype(np.uint8), (pair >> 8).astype(np.uint8)
    y = np.empty((4096, 4096), np.uint8)
    for dy in (0, 1):
        for dx in (0, 1):
            y[dy::2, dx::2] = (rep * 4 + dy * 2 + dx).astype(np.uint8)
    seen = np.zeros(1 << 24, bool)
    ys, us, vs = y.astype(np.int64), np.repeat(np.repeat(u, 2, 0), 2, 1).astype(np.int64), np.repeat(np.repeat(v, 2, 0), 2, 1).astype(np.int64)
    seen[(ys << 16) | (us << 8) | vs] = True
    assert seen.all()  # every (Y, U, V) triple occurs
    want = None
    for fmt in ("nv12", "nv21", "i420"):
        planes = yuv.planes_from_yuv(fmt, y, u, v)
        lib = yuv.libyuv_to_rgba(fmt, *planes, matrix=matrix)
        if want is None:
            want = yuv.frames_to_rgba(fmt, *planes, matrix=matrix)
        assert np.array_equal(lib, want), fmt


@pytest.mark.skipif(yuv.libyuv() is None, reason="oracle/_ref/libyuv_ref.so was not built (the reference checkout is absent)")
@pytest.mark.parametrize("fmt", ["nv12", "nv21"])
def test_shim_row_loop_equals_the_public_bt601_entry_points(fmt):
    # BT.709 NV12 / NV21 go through the shim's own loop over libyuv's rows: with BT.601 constants it must equal NV12ToABGR / NV21ToABGR
    rng = np.random.default_rng(5)
    for h, w in ODD + [(64, 48)]:
        ch, cw = yuv.chroma_shape(h, w)
        planes = yuv.planes_from_yuv(fmt, rng.integers(0, 256, (h, w), dtype=np.uint8), rng.integers(0, 256, (ch, cw), dtype=np.uint8),
                                     rng.integers(0, 256, (ch, cw), dtype=np.uint8))
        assert np.array_equal(yuv.libyuv_to_rgba(fmt, *planes, bt601_rows=True), yuv.libyuv_to_rgba(fmt, *planes, matrix="bt601"))


PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "snnb.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(snnb_frames), offsetof(snnb_frames, format), offsetof(snnb_frames, matrix),
           offsetof(snnb_frames, width), offsetof(snnb_frames, height), offsetof(snnb_frames, plane), offsetof(snnb_frames, pitch),
           offsetof(snnb_frames, image_stride), offsetof(snnb_frames, linear_filter), offsetof(snnb_frames, mean4), offsetof(snnb_frames, norm4));
    printf("%d %d %d %d %d %d\n", SNNB_FRAME_NV12, SNNB_FRAME_NV21, SNNB_FRAME_I420, SNNB_FRAME_RGBA8, SNNB_YUV_BT601, SNNB_YUV_BT709);
    return 0;
}
"""


def test_frames_layout_matches_the_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(PROBE)
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    sizes, enums = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")[:2]
    F = _lib.Frames
    fields = ("format", "matrix", "width", "height", "plane", "pitch", "image_stride", "linear_filter", "mean4", "norm4")
    assert [int(v) for v in sizes.split()] == [C.sizeof(F)] + [getattr(F, f).offset for f in fields]
    assert [int(v) for v in enums.split()] == [_lib.FRAME_NV12, _lib.FRAME_NV21, _lib.FRAME_I420, _lib.FRAME_RGBA8, _lib.YUV_BT601, _lib.YUV_BT709]


def test_frame_entry_points_refuse_null_arguments(built):
    lib = _lib.lib()
    f = _lib.Frames()
    assert lib.snnb_model_run_frames(None, C.byref(f), None, 0, None, None) != 0
    assert b"snnb_model_run_frames: null model" in lib.snnb_last_error()
    assert lib.snnb_model_detect_frames(None, C.byref(f), None, 1, None, None) != 0
    assert b"snnb_model_detect_frames: null model" in lib.snnb_last_error()
