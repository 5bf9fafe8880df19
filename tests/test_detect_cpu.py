"""snnb_model_detect_device without a GPU: the header's prototype is the one the ctypes binding calls, and null arguments are errors."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

from shadernn_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROBE = r"""
#include "snnb.h"
/* compiles only if the header declares exactly this signature */
int (*probe)(snnb_model*, const snnb_device_buffer*, int, float*, int, int*, void*) = snnb_model_detect_device;
"""


def test_detect_device_prototype_matches_the_binding(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    src = tmp_path / "probe.c"
    src.write_text(PROBE)
    subprocess.run([cc, "-std=c99", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o", str(tmp_path / "probe.o")], check=True)
    restype, argtypes = _lib.SIGNATURES["snnb_model_detect_device"]
    assert restype is C.c_int
    assert len(argtypes) == 7 and argtypes[1] is C.POINTER(_lib.DeviceBuffer) and argtypes[2] is C.c_int and argtypes[4] is C.c_int


def test_detect_device_resolves_and_refuses_null_arguments(built):
    lib = _lib.lib()
    assert lib.snnb_model_detect_device.argtypes is not None
    buf = _lib.DeviceBuffer()
    assert lib.snnb_model_detect_device(None, None, 0, None, 0, None, None) != 0
    assert b"snnb_model_detect_device: null model" in lib.snnb_last_error()
    assert lib.snnb_model_detect_device(None, C.byref(buf), 1, None, 100, None, None) != 0
    assert b"snnb_model_detect_device" in lib.snnb_last_error()
