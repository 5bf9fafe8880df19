"""CPU test of the device-frame kernels' machine code.

The input-side kernels (frame_input_kernel, frame_roi_input_kernel, roi_clear_kernel) are templates over where batch slot n's image comes
from: FrameBatchV (an snnb_frames batch) or FrameListV (a frame list, 26 KB of descriptors), passed as a __grid_constant__ parameter
(csrc/kernels_simt.cu). A reference to a kernel parameter that is not __grid_constant__ makes the compiler copy the parameter to local
memory, which would give every thread a stack frame and local loads. So every frame-path kernel must report STACK:0 and LOCAL:0, and each
input family must be instantiated for both source types and for every format it serves."""
import os
import re
import shutil
import subprocess

import pytest

from shadernn_b200 import _lib

FRAME_KERNELS = ("frame_input_kernel", "frame_roi_input_kernel", "roi_clear_kernel", "rois_from_detections_kernel", "frame_output_kernel",
                 "luma_output_kernel", "segment_output_kernel", "frame_list_output_kernel", "luma_list_output_kernel", "segment_list_output_kernel")
SOURCES = ("FrameBatchV", "FrameListV")
FORMATS = {_lib.FRAME_NV12, _lib.FRAME_NV21, _lib.FRAME_I420, _lib.FRAME_RGBA8, _lib.FRAME_P010}
LUMA = {-1, -2}  # FRAME_LUMA and FRAME_LUMA10: the Y plane of 8-bit YUV and of P010 frames
INPUT_FAMILIES = {"frame_input_kernel": FORMATS | LUMA, "frame_roi_input_kernel": FORMATS}


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and os.path.exists(cand):
            return cand
    return None


def _frame_functions():
    """[(kernel name, template arguments (the rest of the mangled name), {resource: value})] of the library's frame-path kernels."""
    tool = _cuobjdump()
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libsnn_b200.so has not been built")
    if tool is None:
        pytest.skip("cuobjdump not found")
    r = subprocess.run([tool, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    out, cur = [], None
    for line in r.stdout.splitlines():
        m = re.match(r"\s*Function (_ZN4snnb(\d+)(\S+)):", line)
        if m:
            n = int(m.group(2))
            name, rest = m.group(3)[:n], m.group(3)[n:]
            cur = (name, rest) if name in FRAME_KERNELS else None
        elif cur is not None and "REG:" in line:
            out.append(cur + ({k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)},))
            cur = None
    return out


def test_frame_kernels_use_no_local_memory():
    funcs = _frame_functions()
    for name in FRAME_KERNELS:
        assert any(f[0] == name for f in funcs), "no %s in the library" % name
    spilled = ["%s%s: STACK %d, LOCAL %d" % (name, rest, res["STACK"], res["LOCAL"]) for name, rest, res in funcs if res["STACK"] or res["LOCAL"]]
    assert not spilled, "frame kernels with a stack frame or local memory: %s" % spilled


def test_input_families_cover_both_sources_and_every_format():
    have = set()
    for name, rest, _ in _frame_functions():
        m = re.match(r"ILi(n?)(\d+)ENS_\d+(\w+?)EE", rest)
        if name in INPUT_FAMILIES and m:
            have.add((name, -int(m.group(2)) if m.group(1) else int(m.group(2)), m.group(3)))
    missing = [(name, fmt, src) for name, fmts in INPUT_FAMILIES.items() for fmt in sorted(fmts) for src in SOURCES if (name, fmt, src) not in have]
    assert not missing, "input kernel instantiations missing (family, format, source): %s" % missing
    clear = {rest for name, rest, _ in _frame_functions() if name == "roi_clear_kernel"}
    for src in ("FrameSizeV", "FrameListV"):  # the batch's clear needs the frame size alone
        assert any(src + "E" in rest for rest in clear), "roi_clear_kernel has no %s instantiation" % src
