"""snnb_model_run_rois / snnb_rois_from_detections without a GPU: the C structs and their ctypes mirrors agree, the entry points refuse
null arguments, and the float32 restatement of rois_from_detections (oracle/rois.py), which the GPU tests hold the kernel to, gives the
regions worked out by hand below (dyadic coordinates, so every product is exact)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import rois
from shadernn_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HW = (50, 100)  # frame height, width

PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "snnb.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(snnb_roi), offsetof(snnb_roi, frame), offsetof(snnb_roi, row), offsetof(snnb_roi, x),
           offsetof(snnb_roi, y), offsetof(snnb_roi, width), offsetof(snnb_roi, height));
    printf("%zu %zu %zu %zu\n", sizeof(snnb_roi_select), offsetof(snnb_roi_select, min_score), offsetof(snnb_roi_select, class_id),
           offsetof(snnb_roi_select, expand));
    return 0;
}
"""


def test_roi_layouts_match_the_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(PROBE)
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    roi, sel = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")[:2]
    R, S = _lib.Roi, _lib.RoiSelect
    assert [int(v) for v in roi.split()] == [24] + [getattr(R, f).offset for f in ("frame", "row", "x", "y", "width", "height")]
    assert C.sizeof(R) == 24
    assert [int(v) for v in sel.split()] == [C.sizeof(S)] + [getattr(S, f).offset for f in ("min_score", "class_id", "expand")]


def test_roi_entry_points_refuse_null_arguments(built):
    lib = _lib.lib()
    f = _lib.Frames()
    assert lib.snnb_model_run_rois(None, C.byref(f), 1, None, None, None, 0, None, None) != 0
    assert b"snnb_model_run_rois: null model" in lib.snnb_last_error()
    sel = _lib.RoiSelect(0.0, -1, 0.0)
    assert lib.snnb_rois_from_detections(None, None, None, 1, 1, 16, 16, C.byref(sel), None, 1, None, None) != 0
    assert b"snnb_rois_from_detections: null context" in lib.snnb_last_error()


def one(row, **kw):
    """The region of one row of frame 0 (or None)."""
    out, count = rois.rois_from_detections(np.asarray(row, np.float32).reshape(1, 1, 6), [1], HW, 4, **kw)
    assert not out[count:].any()
    return None if count == 0 else tuple(int(v) for v in out[0])


def test_boxes_inside_partly_outside_and_wholly_outside_the_frame():
    assert one([0, 0.5, 0.25, 0.25, 0.5, 0.5]) == (0, 0, 25, 12, 50, 26)  # y: 12.5 -> 12, 37.5 -> 38
    assert one([0, 0.5, 0.875, 0.125, 0.25, 0.25]) == (0, 0, 87, 6, 13, 13)  # right edge 112.5 clipped to 100; y 6.25 .. 18.75
    assert one([0, 0.5, 0.75, 0.75, 0.5, 0.5]) == (0, 0, 75, 37, 25, 13)  # clipped right and bottom
    assert one([0, 0.5, 1.25, 0.25, 0.25, 0.25]) is None  # wholly right of the frame: empty after clipping
    assert one([0, 0.5, 0.25, -0.75, 0.25, 0.5]) is None  # wholly above
    assert one([0, 0.5, 0.0, 0.0, 1.0, 1.0]) == (0, 0, 0, 0, 100, 50)  # the whole frame


def test_negative_x_and_huge_w():
    assert one([0, 0.5, -0.25, 0.5, 0.5, 0.25]) == (0, 0, 0, 25, 25, 13)  # x -25 clipped to 0; y 25 .. 37.5
    assert one([0, 0.5, 0.5, 0.0, 1e30, 0.5]) == (0, 0, 50, 0, 50, 25)  # (x + w) * W = 1e32
    assert one([0, 0.5, 0.5, 0.0, 3e38, 0.5]) == (0, 0, 50, 0, 50, 25)  # overflows to +inf, clipped to W
    assert one([0, 0.5, -3e38, 0.0, 3e38, 0.5]) is None  # x + w = 0 exactly: an empty box
    assert one([0, 0.5, 0.5, 0.0, np.inf, 0.5]) is None  # ex = expand * w = 0 * inf is NaN: dropped
    assert one([0, 0.5, 0.5, 0.0, np.inf, 0.5], expand=0.25) == (0, 0, 0, 0, 100, 32)  # ex = inf: x - ex = -inf, clipped to 0
    assert one([0, 0.5, -np.inf, 0.0, np.inf, 0.5], expand=0.25) is None  # x + w = -inf + inf is NaN: dropped


def test_expand():
    # ex = 0.125, ey = 0.125: x 12.5 .. 87.5, y 6.25 .. 43.75
    assert one([0, 0.5, 0.25, 0.25, 0.5, 0.5], expand=0.25) == (0, 0, 12, 6, 76, 38)
    assert one([0, 0.5, 0.0, 0.0, 0.5, 0.5], expand=0.5) == (0, 0, 0, 0, 75, 38)  # grown past the top-left corner, clipped
    assert one([0, 0.5, 0.25, 0.25, 0.0, 0.0], expand=1.0) is None  # a point grows by nothing


def test_class_and_score_filters():
    row = [3, 0.5, 0.25, 0.25, 0.5, 0.5]
    assert one(row, class_id=3) is not None and one(row, class_id=2) is None and one(row, class_id=-1) is not None
    assert one(row, min_score=0.5) is not None  # score >= min_score
    assert one(row, min_score=np.nextafter(np.float32(0.5), np.float32(1))) is None
    assert one([3, -1.0, 0.25, 0.25, 0.5, 0.5]) is None  # the default min_score 0 drops negative scores


def test_nan_drops_the_row():
    for i in range(1, 6):
        row = [0, 0.5, 0.25, 0.25, 0.5, 0.5]
        row[i] = np.nan
        assert one(row) is None, i
    assert one([np.nan, 0.5, 0.25, 0.25, 0.5, 0.5]) is not None  # a NaN class passes "any class"
    assert one([np.nan, 0.5, 0.25, 0.25, 0.5, 0.5], class_id=0) is None


def test_visit_order_capacity_truncation_and_counts():
    rows = np.zeros((3, 4, 6), np.float32)
    for n in range(3):
        for r in range(4):
            rows[n, r] = [r, 0.9 - 0.1 * r, 0.125 * r, 0.125 * n, 0.25, 0.25]
    rows[1, 1, 1] = 0.0  # kept: score >= 0
    rows[1, 2, 4] = 0.0  # empty: dropped
    counts = np.array([2, 4, 9], np.int32)  # frame 2 claims 9 rows: capped at max_rows 4
    out, count = rois.rois_from_detections(rows, counts, HW, 16)
    want = [(0, 0), (0, 1), (1, 0), (1, 1), (1, 3), (2, 0), (2, 1), (2, 2), (2, 3)]
    assert count == len(want) and [tuple(int(v) for v in o[:2]) for o in out[:count]] == want
    assert tuple(out[4]) == (1, 3, 37, 6, 26, 13) and not out[count:].any()
    short, c2 = rois.rois_from_detections(rows, counts, HW, 4)
    assert c2 == 4 and np.array_equal(short, out[:4])  # the first `capacity` kept rows, in visit order
    none, c0 = rois.rois_from_detections(rows, np.array([0, -5, 0], np.int32), HW, 3)
    assert c0 == 0 and not none.any()  # zero (and negative) counts: no regions, every entry zero


def test_crop_rgba():
    F = np.arange(2 * 5 * 7 * 4, dtype=np.uint8).reshape(2, 5, 7, 4)
    s = rois.crop_rgba(F, (1, 9, 2, 1, 3, 4))
    assert s.shape == (4, 3, 4) and np.array_equal(s, F[1, 1:5, 2:5]) and s.flags.c_contiguous
    assert np.array_equal(rois.crop_rgba(F[0], (0, 0, 6, 4, 1, 1)), F[0, 4:5, 6:7])
