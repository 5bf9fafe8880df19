"""GPU parity tests for the wgmma + TMA implicit-GEMM convolution (kernels_umma.cu), forced with algo="tcgen05" (the API name of that path),
against the oracle — and against the CUDA-core kernel on the same inputs, which isolates the 3-term split-bf16 product.
Shapes are the tensor-path layers of the BASELINE graphs (ResNet-18 3x3s, MobileNetV2 1x1 expand/project,
YOLOv3-tiny 13x13 / heads) plus ragged edges: tiles that overhang the image, channel tails that are not multiples of
64 / 16 / 8, several images stacked in one 128-row tile.
"""
import os

import numpy as np
import pytest

from oracle import oracle
from shadernn_b200 import core

pytestmark = pytest.mark.gpu
EPS = 1e-3


def run_case(ctx, n, h, w, ic, oc, k, s=1, padding="same", act="", alpha=0.1, bias=True, bn=True, residual=False, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (n, h, w, ic)).astype(np.float32)
    wt = (rng.standard_normal((oc, ic, k, k)) * np.sqrt(2.0 / (k * k * ic))).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, oc).astype(np.float32) if bias else None
    bnd = None
    if bn:
        bnd = {"gamma": rng.uniform(0.5, 1.5, oc), "beta": rng.uniform(-0.1, 0.1, oc), "mean": rng.uniform(-0.1, 0.1, oc), "var": rng.uniform(0.5, 1.5, oc)}
    o = oracle.same_padding(k, padding == "same") if isinstance(padding, str) else list(padding)
    oh, ow = oracle.conv_out_dim(h, k, s, o[0], o[1]), oracle.conv_out_dim(w, k, s, o[0], o[1])
    px, py = (0, 0) if k == 1 else (o[0], o[2])
    want = oracle.conv2d(x, wt, b, bnd, s, px, py, "constant", "" if residual else act, alpha, (oh, ow))
    res = None
    if residual:
        res = rng.uniform(-1, 1, want.shape).astype(np.float32)
        want = oracle.add(want, res, act, alpha)
    got = core.conv2d(ctx, x, wt, b, bnd, s, px, py, "constant", act, alpha, (oh, ow), residual=res, algo="tcgen05")
    simt = core.conv2d(ctx, x, wt, b, bnd, s, px, py, "constant", act, alpha, (oh, ow), residual=res, algo="simt")
    what = "tcgen05 conv n%d %dx%d ic%d oc%d k%d s%d %s" % (n, h, w, ic, oc, k, s, act)
    assert got.shape == want.shape
    bad = oracle.compare(got, want, EPS)
    err = float(np.max(np.abs(got - want) / np.maximum(np.abs(want), 1.0)))
    err_simt = float(np.max(np.abs(got - simt) / np.maximum(np.abs(simt), 1.0)))
    assert bad == 0, "%s: %d/%d outside eps (max rel err %.3g)" % (what, bad, got.size, err)
    assert err < 1e-4 and err_simt < 1e-4, (what, err, err_simt)  # hi*hi + lo*hi + hi*lo keeps ~16 bits
    return err


def run_case_fp16w(ctx, n, h, w, ic, oc, k, s=1, padding="same", act="relu", seed=0, residual=False):
    """The 2-term product (SNNB_PRECISION_FP16W): split-bf16 activations x ONE fp16 weight plane. Two checks: (a) against the
    oracle fed with the SAME fp16-rounded folded weights the difference is fp32-accumulation noise (the kernel computes exactly
    (A_hi + A_lo) * fp16(W)); (b) against the oracle with the original weights the error is the weight rounding (2^-12 relative
    per weight), inside the 1e-3 per-layer budget."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (n, h, w, ic)).astype(np.float32)
    wt = (rng.standard_normal((oc, ic, k, k)) * np.sqrt(2.0 / (k * k * ic))).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, oc).astype(np.float32)
    bnd = {"gamma": rng.uniform(0.5, 1.5, oc).astype(np.float32), "beta": rng.uniform(-0.1, 0.1, oc).astype(np.float32),
           "mean": rng.uniform(-0.1, 0.1, oc).astype(np.float32), "var": rng.uniform(0.5, 1.5, oc).astype(np.float32)}
    o = oracle.same_padding(k, padding == "same") if isinstance(padding, str) else list(padding)
    oh, ow = oracle.conv_out_dim(h, k, s, o[0], o[1]), oracle.conv_out_dim(w, k, s, o[0], o[1])
    px, py = (0, 0) if k == 1 else (o[0], o[2])
    res = rng.uniform(-1, 1, (n, oh, ow, oc)).astype(np.float32) if residual else None
    # BN folded the way csrc/pack.cpp does it, then the weights rounded to fp16
    sc = bnd["gamma"] / np.maximum(np.sqrt(bnd["var"] + np.float32(0.001)), np.float32(0.0001))
    w16 = (wt * sc[:, None, None, None]).astype(np.float16).astype(np.float32)
    shift = ((b - bnd["mean"]) * sc + bnd["beta"]).astype(np.float32)
    want16 = oracle.conv2d(x, w16, shift, None, s, px, py, "constant", "" if residual else act, 0.1, (oh, ow))
    want = oracle.conv2d(x, wt, b, bnd, s, px, py, "constant", "" if residual else act, 0.1, (oh, ow))
    if residual:
        want16, want = oracle.add(want16, res, act, 0.1), oracle.add(want, res, act, 0.1)
    ctx.set_precision("fp16w")
    try:
        got = core.conv2d(ctx, x, wt, b, bnd, s, px, py, "constant", act, 0.1, (oh, ow), residual=res, algo="tcgen05")
    finally:
        ctx.set_precision("fp32x3")
    scale = float(np.abs(want).max())
    e_exact = float(np.abs(got - want16).max()) / scale
    e_round = float(np.abs(got - want).max()) / scale
    what = "fp16w conv n%d %dx%d ic%d oc%d k%d s%d" % (n, h, w, ic, oc, k, s)
    assert e_exact < 3e-5, (what, "kernel vs oracle on fp16-rounded weights", e_exact)
    assert e_round < 1e-3, (what, "weight rounding error relative to the tensor's range", e_round)
    return e_exact, e_round


@pytest.mark.parametrize("n,h,w,ic,oc,k,s", [(2, 56, 56, 64, 64, 3, 1), (2, 28, 28, 128, 128, 3, 1), (3, 14, 14, 256, 256, 3, 1), (5, 7, 7, 512, 512, 3, 1),
                                             (2, 56, 56, 64, 128, 3, 2), (2, 28, 28, 144, 24, 1, 1), (2, 7, 7, 320, 1280, 1, 1), (1, 13, 13, 512, 1024, 3, 1),
                                             (2, 224, 224, 3, 64, 7, 2), (1, 15, 13, 32, 48, 3, 1), (4, 1, 1, 1280, 1000, 1, 1)])
def test_fp16w_two_term_product(ctx, n, h, w, ic, oc, k, s):
    run_case_fp16w(ctx, n, h, w, ic, oc, k, s, padding="same" if k > 1 else "valid", seed=ic + oc + k)


def test_fp16w_residual_and_wide_tiles(ctx):
    run_case_fp16w(ctx, 2, 14, 14, 128, 80, 3, residual=True, seed=5)
    run_case_fp16w(ctx, 8, 14, 14, 256, 512, 3, seed=6)    # n_blk = 256: one accumulator block of 256 columns
    run_case_fp16w(ctx, 8, 28, 28, 64, 200, 1, padding="valid", seed=7)  # channel tail in a wide tile


def test_first_light_1x1(ctx):
    # the smallest complete case: one M tile, one K block, one N tile
    run_case(ctx, 1, 8, 16, 64, 64, 1, padding="valid", bias=False, bn=False)


@pytest.mark.parametrize("n,h,w,ic,oc", [(2, 56, 56, 16, 96), (2, 28, 28, 144, 24), (3, 14, 14, 96, 576), (2, 7, 7, 320, 1280), (4, 1, 1, 1280, 1000),
                                         (1, 13, 13, 256, 255), (2, 26, 26, 384, 256), (1, 9, 11, 24, 40)])
def test_conv1x1(ctx, n, h, w, ic, oc):
    run_case(ctx, n, h, w, ic, oc, 1, padding="valid", act="relu6", seed=ic + oc)


@pytest.mark.parametrize("n,h,w,ic,oc", [(2, 56, 56, 64, 64), (2, 28, 28, 128, 128), (3, 14, 14, 256, 256), (5, 7, 7, 512, 512), (1, 13, 13, 512, 1024),
                                         (2, 15, 13, 32, 48), (1, 52, 52, 64, 128), (1, 30, 45, 128, 128)])
def test_conv3x3(ctx, n, h, w, ic, oc):
    run_case(ctx, n, h, w, ic, oc, 3, act="relu", seed=h + ic)


@pytest.mark.parametrize("act", ["", "relu", "relu6", "leakyRelu", "tanh", "sigmoid", "SiLU"])
def test_epilogues_and_residual(ctx, act):
    run_case(ctx, 2, 14, 14, 128, 80, 3, act=act, seed=3)
    run_case(ctx, 2, 14, 14, 128, 80, 3, act=act, residual=True, seed=4)


def test_other_kernel_sizes_and_asymmetric_padding(ctx):
    run_case(ctx, 1, 20, 20, 32, 32, 5, act="relu")
    run_case(ctx, 1, 24, 24, 32, 16, 9, padding=(4, 4, 4, 4))       # candy's 9x9 (constant padding flavour)
    run_case(ctx, 2, 12, 12, 64, 64, 3, padding=(1, 0, 1, 0))       # T,B,L,R
    run_case(ctx, 2, 12, 12, 64, 64, 2, act="relu")                 # even kernel: top/left = k/2-1
    run_case(ctx, 1, 16, 16, 64, 64, 3, padding="valid")            # reference dims quirk: output stays 16x16


@pytest.mark.parametrize("n,h,w,ic,oc,k,s,padding,act", [
    (2, 224, 224, 3, 64, 7, 2, "same", "relu"),      # ResNet-18 stem
    (2, 97, 97, 3, 32, 3, 2, "valid", "relu6"),      # MobileNetV2 stem (after ZeroPadding2D)
    (1, 64, 80, 3, 16, 3, 1, "same", "leakyRelu"),   # YOLOv3-tiny first conv
    (1, 40, 40, 1, 16, 5, 1, "same", "relu"),        # ESPCN first conv: 1 input channel
    (1, 33, 29, 4, 24, 3, 1, (1, 0, 1, 0), "tanh"),  # 4 channels, asymmetric padding, transcendental epilogue
    (3, 9, 9, 8, 40, 1, 1, "valid", ""),             # 8 channels 1x1, OC not a multiple of 16
    (2, 40, 52, 3, 32, 9, 1, (4, 4, 4, 4), "relu"),  # style-transfer 9x9 stem: 5 K steps = two weight panels per filter row
    (1, 37, 41, 3, 24, 9, 2, (4, 4, 4, 4), ""),      # 9x9 stride 2: both column parities, 5 K steps
    (1, 30, 30, 2, 16, 8, 1, "same", "relu6"),       # even 8x8: exactly one full panel
])
def test_small_channel_rowgemm(ctx, n, h, w, ic, oc, k, s, padding, act):
    run_case(ctx, n, h, w, ic, oc, k, s=s, padding=padding, act=act, seed=k + ic)


def test_many_tiles_persistent_loop(ctx):
    # more tiles than SMs, several N tiles, accumulator double-buffering exercised for many iterations
    run_case(ctx, 8, 56, 56, 64, 192, 3, act="relu", seed=9)


@pytest.mark.parametrize("k,ic,oc,h", [(3, 64, 128, 56), (1, 64, 128, 56), (3, 128, 256, 29), (3, 256, 512, 14), (1, 256, 512, 14), (5, 32, 32, 21)])
def test_stride2_tma_traversal_stride(ctx, k, ic, oc, h):
    run_case(ctx, 2, h, h, ic, oc, k, s=2, padding="same" if k > 1 else "valid", act="relu")


@pytest.mark.parametrize("n,h,w,ic,oc,k,residual,act", [
    (32, 7, 7, 512, 512, 3, False, "relu"),   # ResNet-18 layer4 at bench size: 128 tiles x 72 K blocks -> split-K
    (32, 7, 7, 512, 512, 3, True, "relu"),    # ... with the fused residual (Conv2D -> Add -> relu)
    (8, 7, 7, 320, 96, 3, False, ""),         # uneven K ranges (45 K blocks), one oc tile
    (2, 14, 14, 448, 64, 3, True, "relu6"),   # 63 K blocks, few tiles
    (1, 13, 13, 1024, 512, 1, False, "leakyRelu"),  # long-K 1x1 (YOLO head): 16 K blocks
])
def test_split_k(ctx, n, h, w, ic, oc, k, residual, act):
    # layers with too few output tiles for 132 SMs: K is split over several CTAs, fp32 partials are reduced by the last
    # arriver in split order. Run twice: the second launch checks that the arrival counters were left at zero.
    run_case(ctx, n, h, w, ic, oc, k, act=act, residual=residual, seed=ic + h)
    run_case(ctx, n, h, w, ic, oc, k, act=act, residual=residual, seed=ic + h + 1)


@pytest.mark.parametrize("n,h,w,ic,oc,k,s,residual", [
    (32, 28, 28, 128, 128, 3, 1, True),   # 196 tiles on 132 SMs: one whole wave + 64 tiles cut into K-block ranges
    (32, 14, 14, 256, 256, 3, 1, False),  # fewer tiles than SMs: every tile cut
    (8, 7, 7, 512, 512, 3, 1, True),      # long K, few tiles
    (5, 33, 21, 64, 96, 3, 2, False),     # ragged
])
def test_stream_k_decomposition(ctx, n, h, w, ic, oc, k, s, residual):
    # SNNB_ALGO_TCGEN05_STREAMK: whole tiles for the full waves, the K loops of the remaining tiles cut evenly across the SMs; a cut
    # tile's fp32 partials are summed in piece order by its last arriver -> deterministic, and equal to the oracle within the bar
    rng = np.random.default_rng(11)
    x = rng.uniform(-1, 1, (n, h, w, ic)).astype(np.float32)
    wt = (rng.standard_normal((oc, ic, k, k)) * np.sqrt(2.0 / (k * k * ic))).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, oc).astype(np.float32)
    o = oracle.same_padding(k, True)
    oh, ow = oracle.conv_out_dim(h, k, s, o[0], o[1]), oracle.conv_out_dim(w, k, s, o[0], o[1])
    want = oracle.conv2d(x, wt, b, None, s, o[0], o[2], "constant", "" if residual else "relu", 0.1, (oh, ow))
    res = None
    if residual:
        res = rng.uniform(-1, 1, want.shape).astype(np.float32)
        want = oracle.add(want, res, "relu", 0.1)
    got = core.conv2d(ctx, x, wt, b, None, s, o[0], o[2], "constant", "relu", 0.1, (oh, ow), residual=res, algo="tcgen05-streamk")
    again = core.conv2d(ctx, x, wt, b, None, s, o[0], o[2], "constant", "relu", 0.1, (oh, ow), residual=res, algo="tcgen05-streamk")
    assert np.array_equal(got, again)  # the reduction order does not depend on which CTA arrives last
    assert not oracle.compare(got, want, EPS), "stream-K conv differs from the oracle"
    plain = core.conv2d(ctx, x, wt, b, None, s, o[0], o[2], "constant", "relu", 0.1, (oh, ow), residual=res, algo="tcgen05")
    assert float(np.max(np.abs(got - plain))) <= 1e-4 * max(1.0, float(np.abs(plain).max()))
