"""Frame lists without a GPU (snnb_model_run_frame_list, snnb_model_detect_frame_list, snnb_model_run_rois_list,
snnb_rois_from_detections_list): the C structs and their ctypes mirrors agree, every entry point refuses null arguments with its own
message, and rois_from_detections_list below, the float32 restatement of snnb_rois_from_detections_list that the GPU tests hold the
kernel to, gives hand-worked regions for frames of different sizes (dyadic coordinates, so every product is exact) and, with every size
equal, exactly oracle/rois.py's single-size regions."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import rois
from shadernn_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "snnb.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu %zu\n", sizeof(snnb_frame_image), offsetof(snnb_frame_image, plane), offsetof(snnb_frame_image, pitch),
           offsetof(snnb_frame_image, width), offsetof(snnb_frame_image, height), offsetof(snnb_frame_image, matrix));
    printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(snnb_frame_list), offsetof(snnb_frame_list, format), offsetof(snnb_frame_list, count),
           offsetof(snnb_frame_list, images), offsetof(snnb_frame_list, linear_filter), offsetof(snnb_frame_list, mean4),
           offsetof(snnb_frame_list, norm4));
    printf("%d %d\n", (int) SNNB_FRAME_LIST_MAX, SNNB_VERSION);
    return 0;
}
"""


def test_frame_list_layouts_match_the_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(PROBE)
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    image, lst, consts = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")[:3]
    I, L = _lib.FrameImage, _lib.FrameList
    assert [int(v) for v in image.split()] == [C.sizeof(I)] + [getattr(I, f).offset for f in ("plane", "pitch", "width", "height", "matrix")]
    assert [int(v) for v in lst.split()] == [C.sizeof(L)] + [getattr(L, f).offset for f in ("format", "count", "images", "linear_filter", "mean4", "norm4")]
    assert [int(v) for v in consts.split()] == [_lib.FRAME_LIST_MAX, 100]


def test_frame_list_entry_points_refuse_null_arguments(built):
    lib = _lib.lib()
    fl = _lib.FrameList()
    assert lib.snnb_model_run_frame_list(None, C.byref(fl), None, 0, None, None) != 0
    assert b"snnb_model_run_frame_list: null model" in lib.snnb_last_error()
    assert lib.snnb_model_detect_frame_list(None, C.byref(fl), None, 1, None, None) != 0
    assert b"snnb_model_detect_frame_list: null model" in lib.snnb_last_error()
    assert lib.snnb_model_run_rois_list(None, C.byref(fl), None, None, None, 0, None, None) != 0
    assert b"snnb_model_run_rois_list: null model" in lib.snnb_last_error()
    sel = _lib.RoiSelect(0.0, -1, 0.0)
    wh = (C.c_int * 2)(16, 16)
    assert lib.snnb_rois_from_detections_list(None, None, None, 1, 1, wh, C.byref(sel), None, 1, None, None) != 0
    assert b"snnb_rois_from_detections_list: null context" in lib.snnb_last_error()


ROW = [0, 0.5, 0.25, 0.25, 0.5, 0.5]


def rois_from_detections_list(rows, counts, frame_hw, capacity, min_score=0.0, class_id=-1, expand=0.0):
    """snnb_rois_from_detections_list restated: oracle/rois.py's rois_from_detections, with frame n's rows mapped by roi_of_row with
    frame n's own size. frame_hw is a list of one (H, W) per frame."""
    rows = np.asarray(rows, np.float32)
    n_frames, max_rows = rows.shape[:2]
    out = np.zeros((capacity, 6), np.int32)
    kept = 0
    for n in range(n_frames):
        for r in range(min(int(counts[n]), max_rows)):
            roi = rois.roi_of_row(rows[n, r], frame_hw[n][1], frame_hw[n][0], min_score, class_id, expand)
            if roi is None:
                continue
            if kept < capacity:
                out[kept] = (n, r) + roi
            kept += 1
    return out, min(kept, capacity)


def test_regions_of_frames_of_different_sizes():
    rows = np.zeros((3, 2, 6), np.float32)
    rows[:, 0] = ROW
    rows[:, 1] = [1, 0.25, 0.875, 0.125, 0.25, 0.25]
    sizes = [(50, 100), (64, 32), (1, 1)]  # (H, W) per frame
    out, count = rois_from_detections_list(rows, np.array([2, 2, 2], np.int32), sizes, 8)
    want = [(0, 0, 25, 12, 50, 26),  # y 12.5 .. 37.5 -> 12 .. 38
            (0, 1, 87, 6, 13, 13),  # x 87.5 .. 112.5 clipped to 100; y 6.25 .. 18.75
            (1, 0, 8, 16, 16, 32),  # x 8 .. 24 of 32, y 16 .. 48 of 64
            (1, 1, 28, 8, 4, 16),  # x 28 .. 36 clipped to 32; y 8 .. 24
            (2, 0, 0, 0, 1, 1),  # 0.25 .. 0.75 of one pixel
            (2, 1, 0, 0, 1, 1)]  # 0.875 .. 1.125 clipped to 1
    assert count == 6 and [tuple(int(v) for v in o) for o in out[:count]] == want and not out[count:].any()
    # the same rows with every frame 50 x 100: a list of equal sizes is the single size
    same, c = rois_from_detections_list(rows, np.array([2, 2, 2], np.int32), [(50, 100)] * 3, 8)
    one, c1 = rois.rois_from_detections(rows, np.array([2, 2, 2], np.int32), (50, 100), 8)
    assert c == c1 == 6 and np.array_equal(same, one)
    assert tuple(one[2]) == (1, 0, 25, 12, 50, 26)


def test_each_frame_scales_by_its_own_size():
    rows = np.array([[ROW], [ROW]], np.float32)
    out, count = rois_from_detections_list(rows, [1, 1], [(1080, 1920), (720, 1280)], 2)
    assert count == 2 and tuple(out[0]) == (0, 0, 480, 270, 960, 540) and tuple(out[1]) == (1, 0, 320, 180, 640, 360)
    # the 1080p region lies outside the 720p frame (x + width = 1440 > 1280): run_rois_list clears a slot that names frame 1 with it
