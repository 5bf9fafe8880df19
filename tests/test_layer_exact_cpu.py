"""CPU checks of oracle/exact.py, the float64 layer restatements test_layer_exact_gpu.py holds every layer to.

- Restatement sanity: the compiled fp32 oracle, an independent fp32 evaluation of the same layers, lies within exact.py's bound of
  the restatement (the bounds of the CUDA-core forms hold for any fp32 summation order), and the data-movement layers agree bit for bit.
- Mutations: plausible kernel defects, simulated in numpy on shapes of the GPU test's instantiation table, each land outside the
  bound somewhere - so the GPU test would catch them.
- Coverage: every conv_umma_kernel / conv_rowwin_kernel instantiation in the built library is named by the GPU test's table.
"""
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import exact, oracle

pytestmark = pytest.mark.usefixtures("built")


def _case(n, h, w, ic, oc, k, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    x = exact.stored(rng.uniform(-1, 1, (n, h, w, ic)) * scale, False)  # what a split-fp16 tensor holds
    wt = (rng.standard_normal((oc, ic, k, k)) * np.sqrt(2.0 / (k * k * ic))).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, oc).astype(np.float32)
    bn = {"gamma": rng.uniform(0.5, 1.5, oc).astype(np.float32), "beta": rng.uniform(-0.1, 0.1, oc).astype(np.float32),
          "mean": rng.uniform(-0.1, 0.1, oc).astype(np.float32), "var": rng.uniform(0.5, 1.5, oc).astype(np.float32)}
    return x, wt, b, bn


def _dims(h, w, k, s):
    o = oracle.same_padding(k, True)
    return o, (oracle.conv_out_dim(h, k, s, o[0], o[1]), oracle.conv_out_dim(w, k, s, o[0], o[1]))


def _direct_conv(x, w, s, pad_x, pad_y, ohw):
    """Plain loops over output pixels, in float64."""
    x = np.asarray(x, np.float64)
    n, h, wd, ic = x.shape
    oc, _, k, _ = w.shape
    y = np.zeros((n, ohw[0], ohw[1], oc))
    for oy in range(ohw[0]):
        for ox in range(ohw[1]):
            for ky in range(k):
                for kx in range(k):
                    iy, ix = oy * s + ky - pad_y, ox * s + kx - pad_x
                    if 0 <= iy < h and 0 <= ix < wd:
                        y[:, oy, ox] += x[:, iy, ix] @ w[:, :, ky, kx].T
    return y


def test_check_rejects_nan_and_inf():
    ref, bound = np.ones(4), np.full(4, 1e-6)
    for bad in (np.nan, np.inf, -np.inf):
        ratio, n_bad = exact.check(np.array([1.0, bad, 1.0, 1.0]), ref, bound, "")
        assert n_bad == 1 and ratio == np.inf
    assert exact.check(np.array([1.0, np.nan]), np.zeros(2), np.zeros(2), "")[1] == 2  # bit-identical layers too


def test_instancenorm_agrees_with_oracle():
    rng = np.random.default_rng(4)
    g, b = rng.uniform(0.5, 1.5, 20).astype(np.float32), rng.uniform(-0.1, 0.1, 20).astype(np.float32)
    for scale, offset in ((1.0, 0.0), (50.0, 100.0), (1e-3, 5.0)):
        x = exact.stored(rng.uniform(-1, 1, (2, 11, 13, 20)) * scale + offset, False)
        for act in ("", "relu", "tanh"):
            _within(oracle.instancenorm(x, g, b, act), *exact.instancenorm(x, g, b, act))


def test_k_order_of_the_row_window_kernels():
    # make_row_plan / make_feed_plan (snnb_internal.h): the 7x7 stride-2 stem, pad 3
    assert exact.row_plan_steps(7, 2, 3) == [[1, 3], [5], [0, 2], [4, 6]]
    assert exact.feed_plan_steps(7, 3) == [[0, 1, 2], [3, 4, 5, 6]]  # d = 1: taps at window pixels 1 .. 7
    assert exact.feed_rows_per_stage(7) == 4 and exact.feed_rows_per_stage(9) == 3 and exact.feed_rows_per_stage(3) == 3
    import ctypes as C
    from shadernn_b200 import _lib
    out = (C.c_int * 5)()
    for k in range(2, 10):
        for pad in range(0, 5):
            assert _lib.lib().snnb_debug_feed_plan(k, 2, pad, 3, out) and out[3] == len(exact.feed_plan_steps(k, pad)), (k, pad)


def _within(got, ref, bound):
    ratio, bad = exact.check(got, ref, bound, "")
    assert bad == 0, ratio
    return ratio


@pytest.mark.parametrize("n,h,w,ic,oc,k,s,act,kernel", [
    (2, 9, 11, 20, 24, 3, 1, "relu", "igemm"), (1, 7, 7, 70, 40, 3, 2, "tanh", "igemm"), (2, 5, 6, 16, 8, 1, 1, "SiLU", "igemm"),
    (2, 10, 12, 3, 16, 5, 1, "", "rowwin"), (1, 8, 8, 16, 8, 3, 1, "sigmoid", "simt"), (1, 6, 9, 24, 12, 3, 1, "leakyRelu", "simt")])
def test_conv_restatement_agrees_with_oracle(n, h, w, ic, oc, k, s, act, kernel):
    x, wt, b, bn = _case(n, h, w, ic, oc, k, h + ic)
    o, ohw = _dims(h, w, k, s)
    want = oracle.conv2d(x, wt, b, bn, s, o[0], o[2], "constant", act, 0.1, ohw)
    ref, bound = exact.conv2d(x, wt, b, bn, s, o[0], o[2], ohw, act, 0.1, form="simt", kernel="simt")
    _within(want, ref, bound)
    # the tensor-core forms against a direct float64 convolution with the operands each form multiplies
    wv, shift = exact.fold(wt, b, bn)
    for form in ("fp32x3", "fp16w", "fp16"):
        r2, b2 = exact.conv2d(x, wt, b, bn, s, o[0], o[2], ohw, act, 0.1, form=form, kernel=kernel)
        direct = exact.act64(_direct_conv(x, exact.weight_operand(wv, form)[0], s, o[0], o[2], ohw) + shift, act, 0.1)
        assert np.all(b2 > 0) and np.allclose(r2, direct, rtol=1e-12, atol=1e-12), form
    # the residual and the replicate / reflect pads restate the oracle too
    res = exact.stored(np.random.default_rng(1).uniform(-1, 1, ref.shape), False)
    want = oracle.add(oracle.conv2d(x, wt, b, bn, s, o[0], o[2], "reflect", "", 0.1, ohw), res, act, 0.1)
    ref, bound = exact.conv2d(x, wt, b, bn, s, o[0], o[2], ohw, act, 0.1, residual=res, form="simt", kernel="simt", pad_mode="reflect")
    _within(want, ref, bound)


def test_other_layers_agree_with_oracle():
    rng = np.random.default_rng(3)
    x = exact.stored(rng.uniform(-2, 2, (2, 9, 10, 20)), False)
    y = exact.stored(rng.uniform(-2, 2, (2, 9, 10, 20)), False)
    bn = {"gamma": rng.uniform(0.5, 1.5, 20).astype(np.float32), "beta": rng.uniform(-0.1, 0.1, 20).astype(np.float32),
          "mean": rng.uniform(-0.1, 0.1, 20).astype(np.float32), "var": rng.uniform(0.5, 1.5, 20).astype(np.float32)}
    wd = rng.standard_normal((20, 3, 3)).astype(np.float32)
    for act in ("", "relu", "relu6", "leakyRelu", "tanh", "sigmoid", "SiLU"):
        _within(oracle.add(x, y, act, 0.1), *exact.add(x, y, act, 0.1))
        _within(oracle.activation(x, act, 0.1), *exact.activation(x, act, 0.1))
        _within(oracle.batchnorm(x, bn, act, 0.1), *exact.batchnorm(x, bn, act, 0.1))
        for s in (1, 2):
            _, ohw = _dims(9, 10, 3, s)
            o = oracle.same_padding(3, True)
            ohw = (oracle.depthwise_out_dim(9, 3, s, o[1], o[3]), oracle.depthwise_out_dim(10, 3, s, o[0], o[2]))
            _within(oracle.depthwise(x, wd, None, bn, s, o[0], o[2], act, 0.1, ohw), *exact.depthwise(x, wd, None, bn, s, o[0], o[2], ohw, act, 0.1))
    for k, s in ((2, 2), (3, 2), (3, 1)):
        ohw = (oracle.pool_out_dim(9, k, s, True), oracle.pool_out_dim(10, k, s, True))
        ref, bound = exact.maxpool(x, k, s, ohw)
        assert np.array_equal(oracle.pool2d(x, k, s, False, ohw), ref.astype(np.float32))
        _within(oracle.pool2d(x, k, s, True, ohw), *exact.avgpool(x, k, s, ohw))
    _within(oracle.softmax(x), *exact.softmax(x))
    dk = rng.standard_normal((7, 9 * 10 * 20)).astype(np.float32) * 0.05
    _within(oracle.dense(x, dk, bn["beta"][:7]), *exact.dense(oracle.flatten(x), dk, bn["beta"][:7], form="fp32x3"))
    gk = rng.standard_normal((7, 20)).astype(np.float32) * 0.2
    pooled = x.mean(axis=(1, 2), keepdims=True, dtype=np.float64).astype(np.float32)
    _within(oracle.softmax(oracle.dense(pooled, gk, bn["beta"][:7])), *exact.gap_dense(x, gk, bn["beta"][:7], softmax_out=True))
    for mode in ("constant", "replicate", "reflect"):
        assert np.array_equal(oracle.pad(x, 2, 1, (12, 14), mode), exact.pad(x, 2, 1, (12, 14), mode)[0].astype(np.float32))
    assert np.array_equal(oracle.concat(x, y), exact.concat(x, y)[0].astype(np.float32))
    assert np.array_equal(oracle.flatten(x), exact.flatten(x)[0].astype(np.float32))
    assert np.array_equal(oracle.upsample(x, 2.0), exact.upsample_nearest(x, (18, 20))[0].astype(np.float32))
    _within(oracle.subpixel(x[..., :4], 2), *exact.subpixel(x[..., :4], 2))
    assert np.array_equal(exact.model_input(x, True)[0], x.astype(np.float16).astype(np.float64))


def test_storage_bound_covers_the_split():
    v = np.random.default_rng(5).standard_normal(100000).astype(np.float32) * np.float32(10.0) ** np.random.default_rng(6).integers(-9, 4, 100000)
    for half in (False, True):
        assert np.all(np.abs(exact.stored(v, half).astype(np.float64) - v) <= exact.store_bound(v, half))


# ---- mutations -----------------------------------------------------------------------------------------------------------------
MUT_SHAPES = [(3, 9, 11, 40, 56, 3, 1), (2, 15, 13, 20, 24, 3, 1), (2, 29, 31, 64, 96, 3, 2)]  # test_layer_exact_gpu.TABLE rows
# row-window shapes of the GPU table (kernel, shape): stride-1 8-channel windows, and the feed stems (7x7 is ResNet-18's, 8x8 and 9x9
# have three K steps per filter row)
ROWWIN_MUT_SHAPES = [("rowwin", (2, 40, 52, 3, 24, 3, 1)), ("rowwin", (1, 21, 60, 8, 40, 5, 1)), ("feed", (2, 41, 45, 3, 64, 7, 2)),
                     ("feed", (1, 33, 61, 3, 40, 8, 2)), ("feed", (2, 37, 41, 3, 24, 9, 2)), ("feed", (2, 27, 45, 3, 24, 2, 2))]


def _conv(x, wt, shift_bias, k, s, o, ohw, form, bias=True):
    return exact.conv2d(x, wt, shift_bias if bias else None, None, s, o[0], o[2], ohw, "", 0.0, form=form, kernel="igemm")


def _mutants(shape):
    n, h, w, ic, oc, k, s = shape
    x, wt, b, bn = _case(n, h, w, ic, oc, k, ic + oc)
    o, ohw = _dims(h, w, k, s)
    wv, shift = exact.fold(wt, b, bn)
    ref, bound = _conv(x, wv, shift, k, s, o, ohw, "fp32x3")
    hi = exact.f16(wv).astype(np.float32)
    lo = exact.f16(wv - hi).astype(np.float32)
    x_hi = exact.f16(x)
    muts = {}
    # A_lo * B_hi dropped: the activations' lo plane never multiplied
    muts["drop A_lo*B_hi"] = _conv(x_hi, wv, shift, k, s, o, ohw, "fp32x3")[0]
    # A_hi * B_lo dropped: (A_hi + A_lo) * B_hi, which is also what fp32x3 computes with w_hi alone (the 2-term product in its place)
    muts["drop A_hi*B_lo / w_hi alone"] = _conv(x, hi, shift, k, s, o, ohw, "simt")[0]
    # the weights' lo plane multiplied by the activations' lo plane instead of their hi plane
    muts["A_lo*B_lo instead of A_hi*B_lo"] = muts["drop A_hi*B_lo / w_hi alone"] + _conv(x - x_hi, lo, np.zeros_like(shift), k, s, o, ohw, "simt")[0]
    # the last K block (the last tap's last 64 input channels) never accumulated
    w_kb = wv.copy()
    w_kb[:, (ic - 1) // 64 * 64:, k - 1, k - 1] = 0
    muts["last K block dropped"] = _conv(x, w_kb, shift, k, s, o, ohw, "fp32x3")[0]
    # an 8-channel tail lost (channels [8 floor((ic - 1) / 8), ic))
    w_tail = wv.copy()
    w_tail[:, (ic - 1) // 8 * 8:] = 0
    muts["8-channel tail dropped"] = _conv(x, w_tail, shift, k, s, o, ohw, "fp32x3")[0]
    # one tap read one pixel off at the tiles' right edge (the last output column)
    xs = np.roll(x, -1, axis=2)
    w_tap = np.zeros_like(wv)
    w_tap[:, :, 0, 0] = wv[:, :, 0, 0]
    shifted = ref.copy()
    zero = np.zeros_like(shift)
    shifted[:, :, -1] += (_conv(xs, w_tap, zero, k, s, o, ohw, "fp32x3")[0] - _conv(x, w_tap, zero, k, s, o, ohw, "fp32x3")[0])[:, :, -1]
    muts["tap shifted at the tile edge"] = shifted
    # BN not folded into one channel
    w_bn, sh_bn = wv.copy(), shift.copy()
    w_bn[3], sh_bn[3] = wt[3], b[3]
    muts["BN fold skipped in one channel"] = _conv(x, w_bn, sh_bn, k, s, o, ohw, "fp32x3")[0]
    # the fp32x3 output stored as fp16
    muts["output rounded to fp16"] = exact.f16(ref)
    # the bias (folded shift) omitted
    muts["bias omitted"] = _conv(x, wv, shift, k, s, o, ohw, "fp32x3", bias=False)[0]
    return ref, bound, muts


@pytest.mark.parametrize("shape", MUT_SHAPES)
def test_conv_mutants_exceed_the_bound(shape):
    ref, bound, muts = _mutants(shape)
    for name, got in muts.items():
        ratio = float(np.max(np.abs(got - ref) / bound))
        print("%-32s %s: worst |err|/bound %.3g" % (name, shape, ratio))
        assert ratio > 1.0, (name, shape, ratio)


@pytest.mark.parametrize("form", ["fp32x3", "fp16w"])
@pytest.mark.parametrize("kernel,shape", ROWWIN_MUT_SHAPES)
def test_rowwin_dropped_lo_plane_exceeds_the_bound(kernel, shape, form):
    # conv_rowwin_kernel with the activations' lo plane missing (the A_lo * B_hi term dropped, or a zeroed feed_lo copy)
    n, h, w, ic, oc, k, s = shape
    x, wt, b, bn = _case(n, h, w, ic, oc, k, ic + oc + k)
    o, ohw = _dims(h, w, k, s)
    ref, bound = exact.conv2d(x, wt, b, bn, s, o[0], o[2], ohw, "", 0.0, form=form, kernel=kernel)
    got, _ = exact.conv2d(exact.f16(x), wt, b, bn, s, o[0], o[2], ohw, "", 0.0, form=form, kernel=kernel)
    ratio = float(np.max(np.abs(got - ref) / bound))
    print("lo plane dropped, %s %s %s: worst |err|/bound %.3g" % (kernel, shape, form, ratio))
    assert ratio > 1.0, (kernel, shape, form, ratio)


def test_avgpool_wrong_border_count_exceeds_the_bound():
    x = exact.stored(np.random.default_rng(9).uniform(0.5, 1.5, (2, 13, 13, 16)), False)
    ohw = (oracle.pool_out_dim(13, 3, 2, False), oracle.pool_out_dim(13, 3, 2, False))  # the last windows are clipped
    want = oracle.pool2d(x, 3, 2, True, ohw)
    ref, bound = exact.avgpool(x, 3, 2, ohw)
    _within(want, ref, bound)
    sums = ref
    cnt = np.zeros(ohw)
    for ky in range(3):
        for kx in range(3):
            cnt += np.outer(np.arange(ohw[0]) * 2 + ky < 13, np.arange(ohw[1]) * 2 + kx < 13)
    wrong = sums * cnt[None, :, :, None] / 9.0  # divided by k * k at the clipped border too
    assert float(np.max(np.abs(wrong - ref) / bound)) > 1.0


# ---- coverage ------------------------------------------------------------------------------------------------------------------
def test_instantiation_table_names_every_kernel():
    import test_layer_exact_gpu as gpu_test
    from test_wgmma_sass_cpu import _cuobjdump
    from shadernn_b200 import _lib
    tool = _cuobjdump()
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libsnn_b200.so has not been built")
    if tool is None:
        pytest.skip("cuobjdump not found")
    r = subprocess.run([tool, "-symbols", _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    found = set()
    for t, nb, sk in re.findall(r"conv_umma_kernelILi(\d+)ELi(\d+)ELb([01])E", r.stdout):
        found.add("conv_umma_kernel<%s, %s, %s>" % (t, nb, "true" if sk == "1" else "false"))
    for t, f, nb in re.findall(r"conv_rowwin_kernelILi(\d+)ELi(\d+)ELi(\d+)E", r.stdout):
        found.add("conv_rowwin_kernel<%s, %s, %s>" % (t, f, nb))
    table = set(gpu_test.expected_instantiations())
    import ctypes as C
    out = (C.c_int * 5)()
    reach = {out[3] for ic in (1, 2, 3, 4) for k in range(1, 33) for pad in range(0, 17) if _lib.lib().snnb_debug_feed_plan(k, 2, pad, ic, out)}
    assert reach == {1, 2, 3}  # the feed mode's K steps per filter row: conv_rowwin_kernel is instantiated for exactly these
    print("%d instantiations in the library, %d named by the table" % (len(found), len(found & table)))
    assert found == table, (sorted(found - table), sorted(table - found))
