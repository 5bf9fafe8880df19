"""Count-sized region batches on the host: the size count_select_kernel picks for a device-side count (snnb_debug_count_body runs the
kernel's own count_body), the Python-side argument checks of set_count_batches, and the selector's machine code."""
import ctypes as C
import os
import re
import subprocess

import pytest

from shadernn_b200 import _lib, core
from test_frame_kernels_sass_cpu import _cuobjdump


def restated(sizes, batch, count):
    """snnb_model_set_count_batches' rule: the smallest declared size >= clamp(count, 0, batch), else batch; 0 runs nothing."""
    c = min(max(count, 0), batch)
    if c == 0:
        return 0
    return min([s for s in sizes if c <= s < batch] + [batch])


@pytest.mark.parametrize("sizes,batch", [([1, 4, 8, 16, 32], 64), ([8, 16, 32], 64), ([4, 8, 16], 12), ([64], 64), ([], 64), ([1], 1),
                                         ([3, 5, 7, 9, 11], 10), ([2, 100, 200], 150)])
def test_count_body_matches_the_restatement(sizes, batch):
    arr = (C.c_int * max(1, len(sizes)))(*sizes)
    for count in range(-5, batch + 6):
        assert _lib.lib().snnb_debug_count_body(arr, len(sizes), batch, count) == restated(sizes, batch, count), (sizes, batch, count)
    for count in (-2 ** 31, 2 ** 31 - 1):
        assert _lib.lib().snnb_debug_count_body(arr, len(sizes), batch, count) == restated(sizes, batch, count)


def test_count_body_refuses_bad_arguments():
    lib = _lib.lib()
    assert lib.snnb_debug_count_body(None, 2, 8, 3) == -1
    assert lib.snnb_debug_count_body((C.c_int * 1)(4), -1, 8, 3) == -1
    assert lib.snnb_debug_count_body((C.c_int * 1)(4), 1, 0, 3) == -1
    assert lib.snnb_debug_count_body(None, 0, 8, 3) == 8


def test_exports_and_python_argument_checks():
    lib = _lib.lib()
    assert hasattr(lib, "snnb_model_set_count_batches") and hasattr(lib, "snnb_debug_count_body")
    m = core.MixedInferenceCore.__new__(core.MixedInferenceCore)  # the checks run before the handle is used
    for bad in ((1, 2.0), [True], "1,2", 4, [None], [1, "2"]):
        with pytest.raises(ValueError, match="sizes must be a list of ints"):
            m.set_count_batches(bad)


def test_selector_kernel_has_no_stack_or_local_memory():
    tool = _cuobjdump()
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libsnn_b200.so has not been built")
    if tool is None:
        pytest.skip("cuobjdump not found")
    r = subprocess.run([tool, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    res, cur = None, False
    for line in r.stdout.splitlines():
        if re.match(r"\s*Function \S*count_select_kernel\S*:", line):
            cur = True
        elif cur and "REG:" in line:
            res = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
            break
    assert res is not None, "no count_select_kernel in the library"
    assert res["STACK"] == 0 and res["LOCAL"] == 0, res
