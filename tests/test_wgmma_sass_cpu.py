"""CPU test of the tensor-core convolution kernels' machine code: their wgmmas must stay asynchronous.

ptxas serializes every wgmma of a kernel that contains a function call (a printf, an out-of-line helper): each HGMMA is then followed by its
own WARPGROUP.DEPBAR, so the tensor cores are fed one instruction deep. In conv_umma_kernel and conv_rowwin_kernel a K block's HGMMAs issue
back to back with one wait per K block (csrc/kernels_umma.cu), so every such function must have at most half as many WARPGROUP.DEPBAR as
HGMMA."""
import os
import re
import shutil
import subprocess

import pytest

from shadernn_b200 import _lib

FAMILIES = ("conv_umma_kernel", "conv_rowwin_kernel")


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and os.path.exists(cand):
            return cand
    return None


def _counts():
    """{mangled function name: (HGMMA count, WARPGROUP.DEPBAR count)} of the library's tensor-core convolution kernels."""
    tool = _cuobjdump()
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libsnn_b200.so has not been built")
    if tool is None:
        pytest.skip("cuobjdump not found")
    r = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    counts, cur = {}, None
    for line in r.stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1) if any(f in m.group(1) for f in FAMILIES) else None
            if cur is not None:
                counts[cur] = [0, 0]
        elif cur is not None:
            if "HGMMA" in line:
                counts[cur][0] += 1
            elif "WARPGROUP.DEPBAR" in line:
                counts[cur][1] += 1
    return counts


def test_conv_kernels_keep_wgmmas_in_flight():
    counts = _counts()
    for fam in FAMILIES:
        assert any(fam in name for name in counts), "no %s in the library" % fam
    serialized = {name: c for name, c in counts.items() if c[0] == 0 or 2 * c[1] > c[0]}
    assert not serialized, "HGMMA / WARPGROUP.DEPBAR counts of kernels whose wgmmas are serialized: %s" % serialized
