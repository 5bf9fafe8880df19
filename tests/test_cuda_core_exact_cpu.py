"""The CUDA-core layer table without a GPU: its coverage list against the library's kernels, the snnb_debug_launches binding, the
bilinear upsampling restatement, and bounds that a wrong kernel would leave (numpy simulations of the kernels' fp32 arithmetic,
each mutated as a plausible bug, must fall outside oracle/exact.py's bound somewhere in the data)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import exact, oracle
from shadernn_b200 import _lib

import test_cuda_core_exact_gpu as table
import test_io_exact_gpu as io_table

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
# kernel families held elsewhere: convolutions, device frame / region / luma / segmentation paths, YOLO, count select; the model
# input / output transfers have their own table (test_io_exact_gpu.py)
OUTSIDE = ("conv", "frame_", "roi_", "rois_", "luma_", "segment_", "yolo_", "count_select")


def _library_kernels():
    tool = next((c for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump") if c and os.path.exists(c)), None)
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libsnn_b200.so has not been built")
    if tool is None:
        pytest.skip("cuobjdump not found")
    r = subprocess.run([tool, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    names = set()
    for m in re.finditer(r"Function _ZN4snnb(\d+)(\S+):", r.stdout):
        n = int(m.group(1))
        name, rest = m.group(2)[:n], m.group(2)[n:]
        args = re.match(r"I((?:Li-?\d+E)+)E", rest)
        names.add(name + ("<%s>" % ", ".join(re.findall(r"Li(-?\d+)E", args.group(1))) if args else ""))
    return names


def test_every_layer_kernel_has_a_case():
    have = _library_kernels()
    layer = sorted(k for k in have if not k.startswith(OUTSIDE))
    assert "pool_kernel<3>" in layer and "depthwise_tma_kernel<2>" in layer, layer  # the demangling works
    io = {k.split("<")[0] for k in io_table.COVERED}
    missing = [k for k in layer if k not in table.COVERED and k not in io]
    assert not missing, "layer kernels without a case in test_cuda_core_exact_gpu.py: %s" % missing
    assert not [k for k in table.COVERED if k not in have], "COVERED names kernels the library does not have"


PROBE = r"""
#include "snnb.h"
int (*probe)(snnb_context*, char*, int, int) = snnb_debug_launches;
"""


def test_debug_launches_prototype_matches_the_binding(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    src = tmp_path / "probe.c"
    src.write_text(PROBE)
    subprocess.run([cc, "-std=c99", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o", str(tmp_path / "probe.o")], check=True)
    assert _lib.SIGNATURES["snnb_debug_launches"] == (C.c_int, [C.c_void_p, C.c_char_p, C.c_int, C.c_int])


def test_debug_launches_refuses_null_arguments(built):
    lib = _lib.lib()
    buf = C.create_string_buffer(16)
    assert lib.snnb_debug_launches(None, buf, 16, 0) == -1
    assert b"snnb_debug_launches" in lib.snnb_last_error()
    assert lib.snnb_debug_launches(None, None, 0, 1) == -1


# ---- the bilinear restatement --------------------------------------------------------------------------------------------------
def upsample_sim(x, scale, out_hw, contract, swap=False):
    """upsample_kernel's bilinear branch in float32 (contract: the compiler fused ox * inv - offs and each tap's multiply-add)."""
    n, h, w, c = x.shape
    inv = f32(1) / f32(scale)
    offs = f32(f32(0.5) - f32(f32(0.5) * inv))

    def coord(o, size):
        o = np.arange(o, dtype=f32)
        s = f32(np.float64(o) * np.float64(inv) - np.float64(offs)) if contract else f32(o * inv) - offs
        return np.minimum(np.maximum(s, f32(0)), f32(size - 1)).astype(f32)

    sx, sy = coord(out_hw[1], w), coord(out_hw[0], h)
    x11, y11 = np.floor(sx).astype(int), np.floor(sy).astype(int)
    fx1, fy1 = (x11 + 1).astype(f32), (y11 + 1).astype(f32)
    ax, bx = (fx1 - sx)[None, :, None], (sx - x11.astype(f32))[None, :, None]
    ay, by = (fy1 - sy)[:, None, None], (sy - y11.astype(f32))[:, None, None]
    w1, w2, w3, w4 = ax * ay, bx * ay, bx * by, ax * by
    if swap:
        w1, w2 = w2, w1
    xp = np.zeros((n, h + 1, w + 1, c), f32)
    xp[:, :h, :w] = x
    v = np.zeros((n, out_hw[0], out_hw[1], c), f32)
    for (yy, xx), wt in (((y11, x11), w1), ((y11, x11 + 1), w2), ((y11 + 1, x11 + 1), w3), ((y11 + 1, x11), w4)):
        t = xp[:, yy][:, :, xx]
        v = f32(np.float64(t) * np.float64(wt) + np.float64(v)) if contract else (v + (t * wt).astype(f32)).astype(f32)
    return v


@pytest.mark.parametrize("scale", [2, 3, 1.5, 1.2, 2.5, 1.7])
def test_bilinear_restatement_holds_the_kernel_arithmetic(scale):
    rng = np.random.default_rng(int(scale * 10))
    x = exact.stored(rng.uniform(-1, 1, (2, 7, 9, 5)) * 255, False)
    out_hw = (int(7 * scale), int(9 * scale))
    ref, bound = exact.upsample_bilinear(x, scale, out_hw)
    for contract in (False, True):
        got = upsample_sim(x, scale, out_hw, contract)
        assert exact.check(got, ref, bound, "upsample")[1] == 0, (scale, contract)
    assert exact.check(upsample_sim(x, scale, out_hw, False, swap=True), ref, bound, "upsample")[1] > 0  # two tap weights swapped
    at = exact.sample_pixels(2, *out_hw, [(4, 4, 1)], seed=3)
    r2, b2 = exact.upsample_bilinear(x, scale, out_hw, at=at)
    assert np.array_equal(r2, ref[at]) and np.array_equal(b2, bound[at])


@pytest.mark.parametrize("scale", [2, 3, 1.5, 1.2])
def test_bilinear_restatement_agrees_with_the_oracle(built, scale):
    rng = np.random.default_rng(7)
    x = rng.uniform(-1, 1, (2, 6, 5, 12)).astype(f32)
    want = oracle.upsample(x, scale, bilinear=True)
    ref, bound = exact.upsample_bilinear(x, scale, want.shape[1:3])
    ratio, bad = exact.check(want, ref, bound, "upsample")
    assert bad == 0, (scale, ratio)


def test_nearest_index_is_the_fp32_product():
    """exact.upsample_nearest promises upsample_kernel's index floor(fl(o * fl(1 / scale))): floor(o / scale) at the integer scales,
    and not at 1.7 (fl(1/1.7) rounds down), where the GPU table's nearest case tells the two apart."""
    x = np.arange(64, dtype=f32).reshape(1, 1, 64, 1)
    o = np.arange(108)
    got = exact.upsample_nearest(x, (1, 108), scale=1.7)[0][0, 0, :, 0]
    assert np.array_equal(got, np.minimum(np.floor(o.astype(f32) * (f32(1) / f32(1.7))), 63))
    assert (got != np.minimum(o * 10 // 17, 63)).any()
    for s in (2, 3, 4):
        got = exact.upsample_nearest(x, (1, 64 * s), scale=s)[0][0, 0, :, 0]
        assert np.array_equal(got, np.arange(64 * s) // s)


# ---- the bounds are not vacuous ------------------------------------------------------------------------------------------------
def _split_input(rng, shape, scale=1.0):
    return exact.stored(rng.uniform(-1, 1, shape) * scale, False)  # hi + lo: a lost lo plane moves values by up to 2^-12 relative


def _exceeds(got, ref, bound):
    return exact.check(got, ref, bound, "mutation")[1] > 0


def test_depthwise_bound_catches_a_lost_lo_plane():
    rng = np.random.default_rng(1)
    x = _split_input(rng, (2, 9, 11, 20))
    wk = rng.standard_normal((20, 3, 3)).astype(f32)
    ref, bound = exact.depthwise(x, wk, None, None, 1, 1, 1, (9, 11))
    assert not _exceeds(exact.depthwise(x, wk, None, None, 1, 1, 1, (9, 11))[0], ref, bound)
    hi_only = exact.depthwise(exact.f16(x), wk, None, None, 1, 1, 1, (9, 11))[0]
    assert _exceeds(hi_only, ref, bound)


def avgpool_sim(x, k, s, out_hw, divisor=None):
    n, h, w, c = x.shape
    y = np.zeros((n,) + tuple(out_hw) + (c,), f32)
    for oy in range(out_hw[0]):
        for ox in range(out_hw[1]):
            win = x[:, oy * s:oy * s + k, ox * s:ox * s + k]
            acc = np.zeros((n, c), f32)
            for v in win.reshape(n, -1, c).transpose(1, 0, 2):
                acc = (acc + v).astype(f32)
            y[:, oy, ox] = acc / f32(divisor or win.shape[1] * win.shape[2])
    return y


def test_avgpool_bound_catches_a_lost_lo_plane_and_a_k2_divisor():
    rng = np.random.default_rng(2)
    out = (7, 7)  # 3x3 stride 2, the last window clipped
    for scale in (1.0, 1e-4):  # near zero, the lo plane of fp16 subnormals is mostly 0: the divisor alone is caught there
        x = _split_input(rng, (2, 13, 14, 20), scale)
        ref, bound = exact.avgpool(x, 3, 2, out)
        assert not _exceeds(avgpool_sim(x, 3, 2, out), ref, bound)
        assert _exceeds(avgpool_sim(x, 3, 2, out, divisor=9), ref, bound)
    x = _split_input(rng, (2, 13, 14, 20))
    ref, bound = exact.avgpool(x, 3, 2, out)
    assert _exceeds(avgpool_sim(exact.f16(x).astype(f32), 3, 2, out), ref, bound)


def instnorm_sim(x, g, b, unbiased=False, eps_outside=False):
    n, h, w, c = x.shape
    hw = h * w
    d = (x - x[:, :1, :1]).astype(f32).reshape(n, hw, c)
    s1 = d.sum(axis=1, dtype=f32)
    s2 = (d * d).sum(axis=1, dtype=f32)
    m = s1 / f32(hw)
    var = np.maximum(s2 / f32(hw) - m * m, f32(0))
    if unbiased:
        var = var * f32(hw) / f32(hw - 1)
    rstd = f32(1) / (np.sqrt(var) + f32(1e-5)) if eps_outside else f32(1) / np.sqrt(var + f32(1e-5))
    mean = x[:, 0, 0] + m
    return ((x - mean[:, None, None]) * (g * rstd)[:, None, None] + b).astype(f32)


def test_instancenorm_bound_catches_the_unbiased_variance_and_eps_outside_the_root():
    rng = np.random.default_rng(3)
    x = _split_input(rng, (2, 12, 13, 8), 0.01)  # variance 3e-5: eps matters
    x[..., 1] += 1000  # a large mean: the shift keeps the variance accurate
    g, b = rng.uniform(0.5, 1.5, 8).astype(f32), rng.uniform(-0.1, 0.1, 8).astype(f32)
    ref, bound = exact.instancenorm(x, g, b)
    assert not _exceeds(instnorm_sim(x, g, b), ref, bound)
    assert _exceeds(instnorm_sim(x, g, b, unbiased=True), ref, bound)
    assert _exceeds(instnorm_sim(x, g, b, eps_outside=True), ref, bound)


def test_softmax_bound_catches_a_missing_max_subtraction():
    """expf(60) is finite in fp32, so at logits of +-60 the sum without the max subtraction loses nothing; at +-100 (the GPU table's
    spread) it overflows to infinity."""
    rng = np.random.default_rng(4)
    z = exact.stored(rng.uniform(-100, 100, (3, 1000)), False).astype(f32)
    ref, bound = exact.softmax(z)
    with np.errstate(over="ignore", invalid="ignore"):
        e = np.exp(z - z.max(axis=1, keepdims=True))
        assert not _exceeds(e / e.sum(axis=1, keepdims=True, dtype=f32), ref, bound)
        e = np.exp(z)
        assert _exceeds(e / e.sum(axis=1, keepdims=True, dtype=f32), ref, bound)
