"""snnb_model_run_device without a GPU: the C struct and its ctypes mirror agree, and bad arguments are errors, not crashes."""
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
    printf("%zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(snnb_device_buffer), offsetof(snnb_device_buffer, data), offsetof(snnb_device_buffer, dtype),
           offsetof(snnb_device_buffer, layout), offsetof(snnb_device_buffer, mean4), offsetof(snnb_device_buffer, norm4), offsetof(snnb_device_buffer, scale),
           offsetof(snnb_device_buffer, offset));
    printf("%d %d %d %d %d\n", SNNB_DTYPE_F32, SNNB_DTYPE_F16, SNNB_DTYPE_U8, SNNB_LAYOUT_NHWC, SNNB_LAYOUT_NCHW);
    return 0;
}
"""


def test_device_buffer_layout_matches_the_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(PROBE)
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    sizes, enums = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")[:2]
    B = _lib.DeviceBuffer
    want = [C.sizeof(B)] + [getattr(B, f).offset for f in ("data", "dtype", "layout", "mean4", "norm4", "scale", "offset")]
    assert [int(v) for v in sizes.split()] == want
    assert [int(v) for v in enums.split()] == [_lib.DTYPE_F32, _lib.DTYPE_F16, _lib.DTYPE_U8, _lib.LAYOUT_NHWC, _lib.LAYOUT_NCHW]


def test_run_device_null_arguments_are_errors(built):
    lib = _lib.lib()
    buf = _lib.DeviceBuffer()
    assert lib.snnb_model_run_device(None, None, 0, None, 0, None, None) != 0
    assert b"null model" in lib.snnb_last_error()
    assert lib.snnb_model_run_device(None, C.byref(buf), 1, C.byref(buf), 1, None, None) != 0
    assert b"snnb_model_run_device" in lib.snnb_last_error()
