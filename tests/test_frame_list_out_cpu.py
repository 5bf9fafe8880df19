"""Output lists without a GPU (snnb_model_transform_frame_list, snnb_model_transform_luma_list, snnb_model_segment_frame_list): the C
structs and their ctypes mirrors agree, and every entry point refuses a null model with its own message instead of crashing."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

from shadernn_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "snnb.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu\n", sizeof(snnb_frame_out_image), offsetof(snnb_frame_out_image, plane), offsetof(snnb_frame_out_image, pitch),
           offsetof(snnb_frame_out_image, width), offsetof(snnb_frame_out_image, height));
    printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(snnb_frame_out_list), offsetof(snnb_frame_out_list, format), offsetof(snnb_frame_out_list, count),
           offsetof(snnb_frame_out_list, images), offsetof(snnb_frame_out_list, linear_filter), offsetof(snnb_frame_out_list, scale),
           offsetof(snnb_frame_out_list, offset));
    printf("%zu %zu %zu %zu %zu\n", sizeof(snnb_labels_image), offsetof(snnb_labels_image, plane), offsetof(snnb_labels_image, pitch),
           offsetof(snnb_labels_image, width), offsetof(snnb_labels_image, height));
    printf("%zu %zu %zu %zu %zu\n", sizeof(snnb_labels_list), offsetof(snnb_labels_list, count), offsetof(snnb_labels_list, images),
           offsetof(snnb_labels_list, linear_filter), offsetof(snnb_labels_list, threshold));
    return 0;
}
"""


def test_output_list_layouts_match_the_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(PROBE)
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")[:4]
    for line, (cls, fields) in zip(lines, [(_lib.FrameOutImage, ("plane", "pitch", "width", "height")),
                                           (_lib.FrameOutList, ("format", "count", "images", "linear_filter", "scale", "offset")),
                                           (_lib.LabelsImage, ("plane", "pitch", "width", "height")),
                                           (_lib.LabelsList, ("count", "images", "linear_filter", "threshold"))]):
        assert [int(v) for v in line.split()] == [C.sizeof(cls)] + [getattr(cls, f).offset for f in fields], cls.__name__


def test_output_list_entry_points_refuse_null_arguments(built):
    lib = _lib.lib()
    fl, ol, ll = _lib.FrameList(), _lib.FrameOutList(), _lib.LabelsList()
    assert lib.snnb_model_transform_frame_list(None, C.byref(fl), C.byref(ol), None) != 0
    assert b"snnb_model_transform_frame_list: null model" in lib.snnb_last_error()
    assert lib.snnb_model_transform_luma_list(None, C.byref(fl), C.byref(ol), None) != 0
    assert b"snnb_model_transform_luma_list: null model" in lib.snnb_last_error()
    assert lib.snnb_model_segment_frame_list(None, C.byref(fl), 1, C.byref(ll), None) != 0
    assert b"snnb_model_segment_frame_list: null model" in lib.snnb_last_error()
