"""The CUDA-core layer kernels held to oracle/exact.py's float64 restatements at the shapes where they break: depthwise (TMA ring and
CUDA-core kernels), pooling, classifier heads, soft-max, instance norm, the elementwise family, upsampling and the layout kernels.

Each case is a one-layer model (two for the fused heads) run in all three precisions (fp16 is the half-storage mode, where the
one-plane code paths run); the layer's output is checked against the restatement fed the engine's own stored input, within the
per-element bound (bit-identical for the data moves). Each case asserts, through snnb_debug_launches, which kernel instantiation
it launched; the depthwise cases run again in a child process with SNNB_DW_SIMT=1, so that depthwise_kernel<3, S, 4> runs on
split storage at large shapes. The test prints the worst |err| / bound of every instantiation and fails if one of
COVERED was never launched (test_cuda_core_exact_cpu.py holds COVERED to the library's kernels).
"""
import fnmatch
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import exact, oracle
from shadernn_b200 import core, modelzoo
from shadernn_b200._lib import SnnbError

import test_layer_exact_gpu as tl

pytestmark = pytest.mark.gpu

FORMS = ("fp32x3", "fp16w", "fp16")
HERE = os.path.dirname(os.path.abspath(__file__))
INSTNORM_MAX_CHUNKS = 64  # snnb_internal.h
GD_THREADS = 1024         # gap_dense_kernel

# every layer kernel instantiation outside the convolutions, frame, region, YOLO, device I/O and count-select paths
COVERED = ["depthwise_tma_kernel<1>", "depthwise_tma_kernel<2>", "depthwise_kernel<3, 1, 4>", "depthwise_kernel<3, 2, 4>",
           "depthwise_generic_kernel", "pool_kernel<2>", "pool_kernel<3>", "pool_kernel<0>", "global_avgpool_kernel", "gap_dense_kernel",
           "softmax_kernel", "add_kernel", "chanwise_kernel", "instnorm_partial_kernel", "instnorm_finalize_kernel", "instnorm_apply_kernel",
           "upsample_kernel", "pad_kernel", "subpixel_kernel", "concat_kernel", "flatten_kernel"]
ACTS = ["", "relu", "relu6", "leakyRelu", "tanh", "sigmoid", "SiLU"]


def _act(d, act):
    d["activation"] = act or "linear"
    if act == "leakyRelu":
        d["leakyReluAlpha"] = 0.1
    return d


def _img(rng, shape, scale=1.0, kind="uniform"):
    x = rng.uniform(-1, 1, shape) * scale
    if kind == "shift" and shape[-1] >= 2:  # channel 0 constant, channel 1 of mean 1000 with unit noise
        x[..., 0] = 0.375
        x[..., 1] = 1000 + rng.standard_normal(shape[:-1])
    if kind == "logits":  # spread over +-100: only the max subtraction keeps expf finite (expf(60) still is)
        x = rng.uniform(-100, 100, shape)
    return x.astype(np.float32)


# ---- the cases: build(b, rng) adds the model's layers and returns (input images, target layer) --------------------------------
def dw_case(n, h, w, c, k, s, padding, act, bias, bn, scale):
    def build(b, rng):
        x = b.input(w, h, c)
        i = b.depthwise(x, k, s, padding, "linear", bias=bias, bn=bn)
        _act(b.layers[i], act)
        return [_img(rng, (n, h, w, c), scale)], i
    return build


def dw_expect(h, w, k, s, padding, half, simt):
    """The depthwise launch: launch_depthwise's choice, with depthwise_tma_supported's tile rule."""
    p = oracle.Model._offsets({"padding": padding}, k)
    oh, ow = (h - k + p[0] + p[1]) // s + 1, (w - k + p[2] + p[3]) // s + 1
    if k == 3 and s in (1, 2):
        tw, th = (16, 8) if s == 1 else (8, 4)
        full = -(-ow // tw) * tw * -(-oh // th) * th
        if not half and not simt and ow * oh >= 0.5 * full:
            return "depthwise_tma_kernel<%d>" % s
        return "depthwise_kernel<3, %d, 4>" % s
    return "depthwise_generic_kernel"


def dw_tiles(n, h, w, c, s):
    tw, th = (16, 8) if s == 1 else (8, 4)
    oh, ow = -(-h // s), -(-w // s)
    return n * -(-oh // th) * -(-ow // tw) * -(-(-(-c // 8) * 8) // 64)


# (n, h, w, c, k, stride, padding, act, bias, bn, input scale)
DW = [
    (2, 29, 37, 20, 3, 1, "same", "relu6", False, True, 1.0),      # tiles overhang right and bottom, channels inside one 8-group
    (2, 29, 37, 136, 3, 2, "same", "", True, True, 1.0),           # 64-channel chunk tail (136 = 2 x 64 + 8)
    (3, 23, 45, 200, 3, 1, "same", "leakyRelu", True, False, 255.0),
    (2, 21, 19, 20, 3, 1, "same", "tanh", False, True, 1e-4),      # fp16 subnormal range; tanh through umma_act_call
    (2, 31, 27, 136, 3, 2, "same", "sigmoid", True, True, 1.0),
    (2, 25, 33, 200, 3, 2, "same", "SiLU", False, True, 255.0),
    (2, 30, 34, 20, 3, 1, "valid", "", True, True, 1.0),
    (4, 111, 111, 136, 3, 1, "same", "relu", False, True, 1.0),    # >= 3 x (2 SMs) tiles: ring stages reused, chunks crossed
    (4, 111, 111, 136, 3, 2, "same", "relu6", True, True, 1.0),
    (2, 7, 7, 20, 3, 1, "same", "relu", True, True, 1.0),          # under half a tile: the CUDA-core kernel
    (2, 5, 9, 136, 3, 2, "same", "leakyRelu", False, True, 255.0),
    (2, 12, 13, 20, 1, 1, "valid", "relu6", True, True, 1.0),      # depthwise_generic_kernel: k != 3, stride 3
    (2, 12, 13, 20, 2, 1, "same", "", False, True, 1e-4),
    (2, 17, 15, 136, 5, 2, "same", "leakyRelu", True, True, 1.0),
    (1, 19, 21, 20, 7, 1, "same", "SiLU", False, True, 255.0),
    (2, 20, 22, 24, 3, 3, "same", "tanh", True, False, 1.0),
    (2, 20, 22, 20, 5, 3, "valid", "sigmoid", False, True, 1.0),
]


def pool_case(n, h, w, c, k, s, avg, padding, scale, glob=False):
    def build(b, rng):
        x = b.input(w, h, c)
        i = b.global_avgpool(x, h) if glob else (b.avgpool(x, k, s, padding) if avg else b.maxpool(x, k, s, padding))
        return [_img(rng, (n, h, w, c), scale)], i
    return build


# (n, h, w, c, k, stride, avg, padding, scale, expected kernel): "same" keeps the last, clipped window
POOL = [
    (2, 13, 15, 3, 2, 2, False, "same", 1.0, "pool_kernel<2>"),
    (2, 9, 11, 12, 2, 1, True, "same", 1e-4, "pool_kernel<2>"),
    (2, 13, 14, 20, 3, 2, False, "same", 255.0, "pool_kernel<3>"),
    (2, 13, 14, 130, 3, 2, True, "same", 1e-4, "pool_kernel<3>"),  # near zero, clipped windows: a k*k divisor shows
    (2, 14, 16, 20, 3, 3, True, "same", 1.0, "pool_kernel<3>"),
    (1, 10, 10, 130, 3, 1, False, "same", 1.0, "pool_kernel<3>"),
    (2, 14, 17, 12, 4, 3, False, "same", 1.0, "pool_kernel<0>"),
    (2, 13, 12, 20, 5, 2, True, "same", 1.0, "pool_kernel<0>"),
    (1, 16, 20, 3, 7, 3, True, "same", 1e-4, "pool_kernel<0>"),
    (2, 9, 9, 130, 7, 1, False, "valid", 1.0, "pool_kernel<0>"),
]
GLOBAL_POOL = [(2, 5, 130, "global_avgpool_kernel"), (2, 4, 3, "global_avgpool_kernel"), (3, 12, 20, "global_avgpool_kernel"),
               (2, 3, 20, "pool_kernel<3>"), (2, 2, 12, "pool_kernel<2>")]  # (n, side, c, kernel): unfused, HW >= 16 or not


def head_case(n, side, cin, cout, act, flatten, scale=1.0):
    def build(b, rng):
        x = b.input(side, side, cin)
        p = b.global_avgpool(x, side)
        if flatten:
            p = b.flatten(p, cin)
        i = b.dense(p, cin, cout, act or "linear")
        return [_img(rng, (n, side, side, cin), scale)], i
    return build


def gap_dense_parts(cin, cout):
    """launch_gap_dense's pixel ranges per channel group (0: the head does not fit in 48 KB of shared memory)."""
    icp, ocp = -(-cin // 8) * 8, -(-cout // 8) * 8
    fits = lambda parts: (parts * icp + (GD_THREADS // 32 + 1) * ocp) * 4 <= 48 * 1024  # noqa: E731
    parts = max(1, min(GD_THREADS // (icp // 8), 8))
    while parts > 1 and not fits(parts):
        parts -= 1
    return parts if fits(parts) else 0


# fused global pool -> [Flatten] -> Dense: (n, side, in C, out C, act, flatten)
HEADS = [
    (2, 2, 20, 1, "relu", True),
    (2, 3, 512, 31, "softmax", False),
    (2, 7, 1000, 33, "", True),
    (2, 7, 1000, 200, "softmax", False),
    (1, 56, 512, 256, "relu", True),
    (2, 3, 4096, 200, "softmax", True),
    (2, 2, 4096, 31, "", False),
    (2, 7, 20, 256, "softmax", True),
    (2, 2, 4096, 256, "softmax", False),  # past the shared-memory limit: the pool and the Dense run apart
]


def flatten_case(n, h, w, c, act, kind="uniform"):
    def build(b, rng):
        x = b.input(w, h, c)
        i = b.flatten(x, h * w * c)
        _act(b.layers[i], act)
        return [_img(rng, (n, h, w, c), kind=kind)], i
    return build


def dense_case(n, cin, cout, scale):
    def build(b, rng):
        x = b.input(1, 1, cin)
        return [_img(rng, (n, 1, 1, cin), scale)], b.dense(x, cin, cout, "softmax")
    return build


def instnorm_chunks(n, h, w, c, sms):
    """launch_instancenorm's chunk count."""
    groups, hw = n * (-(-c // 8)), h * w
    chunks = min(INSTNORM_MAX_CHUNKS, max(1, -(-4 * sms // groups)))
    chunks = max(1, min(chunks, -(-hw // 2048)))
    chunk_px = -(-hw // chunks)
    return -(-hw // chunk_px)


def instnorm_case(n, h, w, c, act, kind):
    def build(b, rng):
        x = b.input(w, h, c)
        i = b.instancenorm(x)
        _act(b.layers[i], act)
        return [_img(rng, (n, h, w, c), kind=kind)], i
    return build


# (n, h, w, c, act, input): chunk counts 1, a few, 16 .. 32, and INSTNORM_MAX_CHUNKS on a 132-SM H100
INSTNORM = [
    (1, 40, 40, 20, "", "shift"),
    (2, 100, 100, 20, "relu", "shift"),
    (2, 90, 91, 24, "leakyRelu", "uniform"),
    (1, 360, 360, 3, "tanh", "shift"),
    (2, 181, 181, 12, "sigmoid", "shift"),
    (3, 200, 200, 8, "SiLU", "uniform"),
    (2, 255, 255, 8, "relu6", "shift"),
]


def elementwise_case(kind, n, h, w, c, act, scale):
    def build(b, rng):
        x = b.input(w, h, c)
        if kind == "add":
            y = b.input(w, h, c, index=1)
            i = b.add(x, y)
            _act(b.layers[i], act)
            return [_img(rng, (n, h, w, c), scale), _img(rng, (n, h, w, c), scale)], i
        if kind == "bn":
            i = b.batchnorm(x)
        else:
            i = b._add({"type": "Activation", "name": "activation_%d" % len(b.layers), "inputPlanes": c, "outputPlanes": c}, [x])
        _act(b.layers[i], act)
        return [_img(rng, (n, h, w, c), scale)], i
    return build


ELEMENTWISE = [(n, h, w, c, act, scale) for (n, h, w, c, scale), act in zip(
    [(2, 9, 11, 20, 1.0), (2, 5, 7, 3, 255.0), (1, 8, 8, 130, 1e-4), (2, 6, 6, 12, 1.0), (2, 6, 5, 20, 255.0), (2, 4, 4, 24, 1e-4), (1, 7, 3, 9, 1.0)], ACTS)]


def upsample_case(n, h, w, c, scale, bilinear):
    def build(b, rng):
        x = b.input(w, h, c)
        return [_img(rng, (n, h, w, c))], b.upsample(x, scale, "bilinear" if bilinear else "nearest")
    return build


# (n, h, w, c, scale, bilinear)
UPSAMPLE = [(2, 5, 7, 20, 2, False), (2, 4, 3, 3, 3, False), (1, 3, 5, 12, 4, False), (1, 1, 1, 12, 2, False),
            (2, 6, 7, 20, 1.5, False), (2, 11, 9, 3, 1.2, False), (2, 5, 6, 12, 2.5, False), (1, 23, 21, 9, 1.7, False),
            (2, 5, 7, 20, 2, True), (2, 4, 5, 3, 3, True), (2, 1, 6, 20, 2, True), (2, 5, 1, 3, 3, True),
            (2, 6, 7, 20, 1.5, True), (2, 11, 9, 12, 1.2, True), (1, 5, 6, 20, 2.5, True), (1, 23, 21, 9, 1.7, True)]


def pad_case(n, h, w, c, t, bt, l, r, mode):
    def build(b, rng):
        x = b.input(w, h, c)
        return [_img(rng, (n, h, w, c))], b.pad(x, t, bt, l, r, None if mode == "constant" else mode)
    return build


# (n, h, w, c, T, B, L, R, mode): the kernel shifts columns by T and rows by L (the reference's uPad = (T, L), exact.pad)
PAD = [(2, 6, 7, 20, 1, 2, 3, 0, "constant"), (2, 6, 7, 3, 2, 1, 0, 3, "replicate"), (2, 6, 7, 12, 1, 3, 2, 1, "reflect"),
       (1, 5, 6, 20, 5, 4, 4, 5, "reflect"), (1, 4, 4, 3, 6, 6, 6, 6, "reflect"), (1, 3, 5, 12, 7, 2, 1, 6, "replicate")]


def concat_case(n, h, w, ca, cb):
    def build(b, rng):
        x = b.input(w, h, ca)
        y = b.input(w, h, cb, index=1)
        return [_img(rng, (n, h, w, ca)), _img(rng, (n, h, w, cb))], b.concat(x, y)
    return build


def subpixel_case(n, h, w, r):
    def build(b, rng):
        x = b.input(w, h, r * r)
        return [_img(rng, (n, h, w, r * r), 3.0)], b.subpixel(x, r)
    return build


def cases(sms):
    """(why, build, fuse, expected launches) of the whole table: the launches are fnmatch patterns, or a function of the precision and
    of SNNB_DW_SIMT that gives them."""
    out = []
    for row in DW:
        n, h, w, c, k, s, padding, act, bias, bn, scale = row
        why = "depthwise n%d %dx%d c%d k%d s%d %s %s bias=%d bn=%d x%g" % (n, h, w, c, k, s, padding, act, bias, bn, scale)
        out.append((why, dw_case(*row), False, lambda prec, simt, a=(h, w, k, s, padding): [dw_expect(*a, prec == "fp16", simt)]))
    for n, h, w, c, k, s, avg, padding, scale, kern in POOL:
        out.append(("%s pool n%d %dx%d c%d k%d s%d %s x%g" % ("avg" if avg else "max", n, h, w, c, k, s, padding, scale),
                    pool_case(n, h, w, c, k, s, avg, padding, scale), False, [kern]))
    for n, side, c, kern in GLOBAL_POOL:
        out.append(("global avg pool n%d %dx%d c%d" % (n, side, side, c), pool_case(n, side, side, c, side, side, True, "valid", 1.0, glob=True), False, [kern]))
    for n, side, cin, cout, act, flat in HEADS:
        parts = gap_dense_parts(cin, cout)
        why = "head n%d %dx%d %d->%d %s flatten=%d parts=%d" % (n, side, side, cin, cout, act, flat, parts)
        # past the shared-memory limit the pool and the Dense (a 1x1 convolution, then the soft-max) launch apart
        out.append((why, head_case(n, side, cin, cout, act, flat), True, ["gap_dense_kernel"] if parts else ["pool_kernel<%d>" % side, "conv_*", "softmax_kernel"]))
    out.append(("flatten softmax logits +-100 c1000", flatten_case(2, 1, 1, 1000, "softmax", "logits"), False, ["flatten_kernel", "softmax_kernel"]))
    out.append(("flatten softmax logits +-100 c37", flatten_case(3, 1, 1, 37, "softmax", "logits"), False, ["flatten_kernel", "softmax_kernel"]))
    out.append(("flatten 3x5x20 (channel tail)", flatten_case(2, 3, 5, 20, ""), False, ["flatten_kernel"]))
    out.append(("flatten 2x3x13", flatten_case(2, 2, 3, 13, ""), False, ["flatten_kernel"]))
    out.append(("dense 64->1000 softmax, inputs x100 (logits over +-60 and more)", dense_case(2, 64, 1000, 100.0), False, ["conv_*", "softmax_kernel"]))
    for row in INSTNORM:
        n, h, w, c, act, kind = row
        why = "instnorm n%d %dx%d c%d %s %s chunks=%d" % (n, h, w, c, act, kind, instnorm_chunks(n, h, w, c, sms))
        out.append((why, instnorm_case(*row), False, ["instnorm_partial_kernel", "instnorm_finalize_kernel", "instnorm_apply_kernel"]))
    for kind, kern in (("add", "add_kernel"), ("bn", "chanwise_kernel"), ("act", "chanwise_kernel")):
        for n, h, w, c, act, scale in ELEMENTWISE:
            out.append(("%s n%d %dx%d c%d %s x%g" % (kind, n, h, w, c, act, scale), elementwise_case(kind, n, h, w, c, act, scale), False, [kern]))
    for row in UPSAMPLE:
        out.append(("upsample %s n%d %dx%d c%d x%g" % ("bilinear" if row[5] else "nearest", *row[:5]), upsample_case(*row), False, ["upsample_kernel"]))
    for row in PAD:
        out.append(("pad %s n%d %dx%d c%d T%d B%d L%d R%d" % (row[8], *row[:8]), pad_case(*row), False, ["pad_kernel"]))
    for ca, cb in ((3, 5), (20, 255), (3, 255), (20, 5)):
        out.append(("concat %d + %d" % (ca, cb), concat_case(2, 5, 6, ca, cb), False, ["concat_kernel"]))
    out.append(("subpixel r2", subpixel_case(2, 5, 6, 2), False, ["subpixel_kernel"]))
    out.append(("subpixel r3 (C 9, Cp 16)", subpixel_case(2, 4, 7, 3), False, ["subpixel_kernel"]))
    return out


# ---- running one case --------------------------------------------------------------------------------------------------------
WHOLE = ("Pad", "Concatenate", "Flatten", "Dense", "MaxPooling2D", "Subpixel", "UpSampling2D")  # data moves and heads: always whole
SAMPLE_ABOVE = 20000  # output pixels above which a layer is restated at exact.sample_pixels points


def run_case(ctx, tmp, idx, why, build, fuse, precision):
    """Runs one case; returns (launched kernel names, worst |err| / bound)."""
    b = modelzoo.Builder(idx)
    rng = np.random.default_rng(1000 + idx)
    imgs, target = build(b, rng)
    path = os.path.join(tmp, "case%d_%s.json" % (idx, precision))
    modelzoo.write_model(b.layers, path, split=True)
    n = imgs[0].shape[0]
    m = core.MixedInferenceCore(ctx, path, batch=n, fuse=fuse, precision=precision)
    om = oracle.Model(path)
    try:
        for j, img in enumerate(imgs):
            m.set_input(img, j)
        ctx.debug_launches(clear=True)
        m.forward()
        ctx.sync()
        launched = ctx.debug_launches(clear=True)
        outs = []
        for i in range(m.num_layers):
            if fuse and om.type_of(om.layers[i]) == "Flatten":
                outs.append(None)  # fused, a Flatten of a 1 x 1 map is an alias of its producer's tensor
                continue
            try:
                outs.append(m.layer_output(i))
            except SnnbError:
                assert fuse, m.layer_info(i)[0]  # only fusion may hide a layer: the pool of the fused head
                outs.append(None)
        shapes = [m.layer_info(i)[2] for i in range(m.num_layers)]
    finally:
        m.close()
    half = precision == "fp16"
    got = outs[target]
    t = om.type_of(om.layers[target])
    nn, oh, ow, _ = got.shape
    at = None
    if t not in WHOLE and nn * oh * ow > SAMPLE_ABOVE:
        at = exact.sample_pixels(nn, oh, ow, [(16, 8, 1), (8, 4, 1)], seed=idx)
        got = got[at]
    r = tl.restate(om, target, outs, {"names": [""] * len(shapes), "shapes": shapes}, precision, half, imgs[0], at)
    assert r is not None, (why, "no restatement")
    ref, bound = r
    assert got.shape == ref.shape, (why, got.shape, ref.shape)
    ratio, bad = exact.check(got, ref, bound, t)
    if bad:
        err = np.abs(got.astype(np.float64) - ref)
        k = np.unravel_index(np.argmax(np.where(err <= bound, 0, err / np.maximum(bound, 1e-300))), err.shape)
        raise AssertionError("%s %s: %d elements outside the bound, worst |err|/bound %.3g; at %s got %r ref %r bound %.3g (launched %s)" % (
            why, precision, bad, ratio, k, float(got[k]), float(ref[k]), float(bound[k]), launched))
    return launched, ratio


def run_all(ctx, tmp, precisions, only_dw=False, simt=False):
    import torch
    sms = torch.cuda.get_device_properties(ctx.device).multi_processor_count
    seen = {}
    chunk_counts = set()
    for idx, (why, build, fuse, want) in enumerate(cases(sms)):
        if only_dw and not why.startswith("depthwise"):
            continue
        for precision in precisions:
            launched, ratio = run_case(ctx, tmp, idx, why, build, fuse, precision)
            expect = want(precision, simt) if callable(want) else want
            assert len(launched) == len(expect) and all(fnmatch.fnmatchcase(k, e) for k, e in zip(launched, expect)), (why, precision, launched, expect)
            for k in launched:
                if seen.get(k, (None, -1.0))[1] < ratio:
                    seen[k] = ("%s %s" % (why, precision), ratio)
        if why.startswith("instnorm"):
            chunk_counts.add(int(why.rsplit("=", 1)[1]))
    if not only_dw:
        big = [r for r in DW if dw_tiles(r[0], r[1], r[2], r[3], r[5]) >= 3 * 2 * sms and dw_expect(r[1], r[2], r[4], r[5], r[6], False, False).startswith("depthwise_tma")]
        assert {r[5] for r in big} == {1, 2}, "no depthwise case walks >= 3 tiles per CTA at %d SMs in both strides" % sms
        assert 1 in chunk_counts and INSTNORM_MAX_CHUNKS in chunk_counts and len(chunk_counts) >= 4, sorted(chunk_counts)
        parts = {gap_dense_parts(h[2], h[3]) for h in HEADS}
        assert {0, 1, 2}.issubset(parts) and max(parts) == 8, sorted(parts)
    return seen


def child_main():
    """SNNB_DW_SIMT=1 child: the depthwise cases on the CUDA-core kernels in the split-storage forms; prints what it launched."""
    import tempfile
    ctx = core.GpuContext(0)
    with tempfile.TemporaryDirectory() as tmp:
        seen = run_all(ctx, tmp, ("fp32x3", "fp16w"), only_dw=True, simt=True)
    ctx.close()
    print("SEEN " + json.dumps({"%s (SNNB_DW_SIMT=1)" % k: v for k, v in seen.items()}))


def test_every_cuda_core_instantiation(ctx, tmp_path):
    seen = run_all(ctx, str(tmp_path), FORMS)
    env = dict(os.environ, SNNB_DW_SIMT="1")
    code = "import sys; sys.path[:0] = [%r, %r]; import test_cuda_core_exact_gpu as t; t.child_main()" % (HERE, os.path.dirname(HERE))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("SEEN ")][-1]
    child = json.loads(line[5:])
    for key, val in child.items():
        seen[key] = tuple(val)
    for key in COVERED + sorted(child):
        print("%-44s %s" % (key, "worst |err|/bound %.3g (%s)" % (seen[key][1], seen[key][0]) if key in seen else "NOT LAUNCHED"))
    missing = [k for k in COVERED if k not in seen]
    assert not missing, missing
    assert any(k.startswith("depthwise_kernel<3, 1, 4>") for k in child) and any(k.startswith("depthwise_kernel<3, 2, 4>") for k in child), sorted(child)


def test_launch_record_keeps_the_latest_names(ctx, tmp_path):
    """snnb_debug_launches past its cap: whole names, the most recent kept, and a clear empties it."""
    b = modelzoo.Builder(0)
    b.maxpool(b.input(6, 6, 8), 2)
    path = os.path.join(str(tmp_path), "pool.json")
    modelzoo.write_model(b.layers, path, split=True)
    m = core.MixedInferenceCore(ctx, path, batch=1)
    try:
        m.set_input(np.zeros((1, 6, 6, 8), np.float32))
        ctx.debug_launches(clear=True)
        for _ in range(5000):  # 15 bytes per name: past the 64 KB cap
            m.forward()
        ctx.sync()
        names = ctx.debug_launches(clear=True)
        assert set(names) == {"pool_kernel<2>"} and 32 * 1024 // 15 <= len(names) <= 64 * 1024 // 15, len(names)
        m.forward()
        assert ctx.debug_launches(clear=True) == ["pool_kernel<2>"]
        assert ctx.debug_launches() == []
    finally:
        m.close()
