"""The fused residual (Conv2D -> Add) of every tensor-core convolution instantiation, held to oracle/exact.py's float64 restatement.

Each case is a three-layer model: a residual source convolution of the input, then the convolution under test (linear) of the same
input, then add(conv, source, act). The source comes first, so the fuser folds the tested convolution into the Add: its epilogue loads
the source's tensor as the residual, adds it and applies the Add's activation. The Add's output is restated in full by
test_layer_exact_gpu.restate from the engine's own input and residual, and must hold to the bound everywhere.

Every case runs twice on one loaded model with different inputs, and both runs are restated: the second catches split-K / stream-K
counters left non-zero and stale partial or staging data. Each launch must be the one snnb_debug_conv_launch gives for the case with a
residual at the device's SM count. Between them the cases must reach every key of case_keys in every product form: all 18
conv_umma_kernel<TERMS, NB, SK> instantiations with a residual (the stream-K ones in a child process with SNNB_SK=1, which makes the
planner consider it), split-K in each TERMS, channel tails inside the last tile, stacked images, boxes over the image edge, several
work items per CTA, stride 2, the activations of the Add, residuals at 255 scale and in fp16's subnormal range, and replicate / reflect
padding, including the <= 8-channel convolution that runs the implicit GEMM on a pre-padded copy of its input. test_residual_exact_cpu.py
checks on the host that the table reaches them and that the restatement catches the epilogue's plausible defects.

The launch record (snnb_debug_last_conv_variant) names the path, product form, channel tile, K split and stream-K of a launch, not its
tile box: the keys about the box (stacked images, boxes over the edge, work items per CTA) rest on the launch being the host plan, whose
box test_conv_plan.py holds to the rules it restates. The residual-scale keys are earned by the residual the case restates (residual_keys),
not by the row's input scale.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import test_conv_plan as cp
from oracle import exact, oracle
from shadernn_b200 import core, modelzoo
from test_layer_exact_gpu import FORMS, KERNEL_OF_PATH, conv_kernel, plan_variant, restate, variant_key

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
SRC, CONV, ADD = 1, 2, 3  # layer ids of a case model (0: the input)
PAD_MODE = {None: cp.PAD_NONE, "constant": cp.PAD_CONSTANT, "reflect": cp.PAD_REFLECT, "replicate": cp.PAD_REPLICATE}


def P(k):
    """Explicit symmetric padding of a k x k window, as the converter writes a replicate / reflect pad folded into its convolution."""
    return [[k // 2, k // 2], [k // 2, k // 2]]


# (n, h, w, ic, oc, k, s, padding, pad mode, Add activation, input scale). The planner picks the channel tile from its cost model per
# product form; test_residual_exact_cpu.py checks which rows reach which key.
TABLE = [
    # channel tails: OC < 32 on a narrow slab, OC not a multiple of 8
    (3, 9, 11, 40, 20, 3, 1, "same", None, "", 1.0),
    # OC 80 on 64-channel tiles (the second tile holds 16 channels), with the transcendental epilogue and leakyRelu
    (4, 40, 44, 32, 80, 3, 1, "same", None, "tanh", 1.0),
    (4, 40, 44, 32, 80, 3, 1, "same", None, "sigmoid", 1.0),
    (4, 40, 44, 32, 80, 3, 1, "same", None, "SiLU", 1.0),
    (4, 40, 44, 32, 80, 3, 1, "same", None, "leakyRelu", 1.0),
    # 128-channel tiles, four work items per CTA: slab 1 of the last tile partly (OC 200) and wholly (OC 180) outside the tensor
    (33, 32, 32, 64, 200, 1, 1, "valid", None, "tanh", 1.0),
    (33, 32, 32, 64, 180, 1, 1, "valid", None, "sigmoid", 1.0),
    (33, 32, 32, 64, 200, 1, 1, "valid", None, "SiLU", 1.0),
    # stacked images: five 5 x 5 maps to a 128-channel tile
    (500, 5, 5, 64, 200, 1, 1, "valid", None, "leakyRelu", 1.0),
    # stride 2 with odd sizes, boxes over the edges
    (2, 29, 31, 64, 96, 3, 2, "same", None, "relu6", 1.0),
    # split-K: few tiles, the zoo's longest K (3x3x512)
    (2, 7, 7, 512, 136, 3, 1, "same", None, "", 1.0),
    # inputs, biases and BatchNorm shifts at Candy's 0..255 scale, and at 1e-4, where about half the residual is subnormal in fp16
    (2, 30, 30, 32, 48, 3, 1, "same", None, "relu", 255.0),
    (2, 12, 17, 48, 136, 3, 1, "same", None, "", 1e-4),
    # replicate / reflect padding: the implicit GEMM on a pre-padded copy, with >= 16 and <= 8 input channels
    (2, 18, 21, 24, 40, 3, 1, P(3), "reflect", "relu", 1.0),
    (2, 18, 21, 24, 40, 3, 1, P(3), "replicate", "", 1.0),
    (2, 19, 23, 3, 32, 3, 1, P(3), "reflect", "", 1.0),
    (1, 21, 17, 8, 64, 5, 1, P(5), "replicate", "leakyRelu", 1.0),
]
# stream-K (SNNB_SK=1): tile counts that leave a partial last wave on 132 SMs
SK_TABLE = [
    (9, 14, 14, 256, 256, 3, 1, "same", None, "relu", 1.0),
    (9, 14, 14, 256, 56, 3, 1, "same", None, "", 1.0),
    (9, 14, 14, 256, 96, 3, 1, "same", None, "tanh", 1.0),
    (17, 16, 32, 64, 256, 3, 1, "same", None, "relu", 1.0),
]


def out_hw(row):
    n, h, w, ic, oc, k, s, padding, mode, act, scale = row
    o = oracle.Model._offsets({"padding": padding}, k)
    return oracle.conv_out_dim(h, k, s, o[0], o[1]), oracle.conv_out_dim(w, k, s, o[2], o[3])


def src_mode(row):
    """The residual source's padding mode: zero padding, named explicitly where the row gives its padding as a list (the model
    format requires a mode there)."""
    return "constant" if isinstance(row[7], list) else None


def case_plan(row, precision, sms, stream_k=False, layer=CONV):
    """snnb_debug_conv_launch of the tested convolution (with its residual) or of the residual source (layer=SRC), as the engine plans
    them (stream_k: as SNNB_SK=1 makes it)."""
    n, h, w, ic, oc, k, s, padding, mode, act, scale = row
    o = oracle.Model._offsets({"padding": padding}, k)
    px, py = (0, 0) if k == 1 else (o[0], o[2])
    if layer == SRC:
        return cp.plan((h, w, ic), (*out_hw(row), oc), k, s, px, py, pad_mode=PAD_MODE[src_mode(row)], may_feed=True, n=n, precision=precision,
                       stream_k=stream_k, sms=sms)
    return cp.plan((h, w, ic), (*out_hw(row), oc), k, s, px, py, pad_mode=PAD_MODE[mode], residual=True, may_feed=True, n=n,
                   precision=precision, stream_k=stream_k, sms=sms)


def case_keys(row, precision, p):
    """What a case with plan p covers: its instantiation, split-K, and the properties of its tiles named in the module docstring
    (those other than the instantiation and split-K carry the product form)."""
    n, h, w, ic, oc, k, s, padding, mode, act, scale = row
    oh, ow = out_hw(row)
    keys = [variant_key(plan_variant(p))]
    if p["ksplit"] > 1:
        keys.append("split-K TERMS=%d" % p["terms"])
    nb = p["n_blk"]
    own = []
    if nb == 32 and oc < 32:
        own.append("OC < 32 on a 32-channel tile")
    if nb == 64 and oc == 80:
        own.append("OC 80 on 64-channel tiles")
    if nb == 128 and oc % 128 > 64:
        own.append("128-channel tile, slab 1 partly outside")
    if nb == 128 and 0 < oc % 128 <= 64:
        own.append("128-channel tile, slab 1 wholly outside")
    if oc % 8:
        own.append("OC not a multiple of 8")
    if p["tn"] > 1:
        own.append("stacked images")
    if p["tiles_x"] * p["tw"] > ow or p["tiles_y"] * p["th"] > oh or p["tiles_n"] * p["tn"] > n:
        own.append("boxes over the edge")
    items = p["tiles_x"] * p["tiles_y"] * p["tiles_n"] * p["tiles_oc"] * p["ksplit"]
    if not p["sk"] and items >= 3 * p["grid"]:
        own.append(">= 3 work items per CTA")
    if s == 2:
        own.append("stride 2")
    if act in ("tanh", "sigmoid", "SiLU", "leakyRelu") and nb in (64, 128):
        own.append("%s on %d-channel tiles" % (act, nb))
    if mode is not None:
        own.append("%s padding, IC %s" % (mode, ">= 16" if ic >= 16 else "<= 8 on a pre-padded copy"))
    return keys + ["%s [%s]" % (key, precision) for key in own]


RES_255, RES_SUBNORMAL = "residual at 255 scale", "residual at 1e-4 scale, >= 25% subnormal in fp16"


def residual_keys(res, precision):
    """The residual-scale keys a residual earns, as stored by the engine: 255 scale when its median magnitude is at least 32; fp16's
    subnormal range when all of it stays below 2^-8 and at least a quarter of it is non-zero and below 2^-14, fp16's smallest normal."""
    a = np.abs(np.asarray(res, np.float64))
    keys = []
    if np.median(a) >= 32:
        keys.append(RES_255)
    if a.max() < 2.0 ** -8 and np.mean((a > 0) & (a < 2.0 ** -14)) >= 0.25:
        keys.append(RES_SUBNORMAL)
    return ["%s [%s]" % (key, precision) for key in keys]


def required_keys():
    umma = ["conv_umma_kernel<%d, %d, %s>" % (t, nb, sk) for t in (1, 2, 3) for nb in (32, 64, 128) for sk in ("false", "true")]
    own = ["OC < 32 on a 32-channel tile", "OC 80 on 64-channel tiles", "128-channel tile, slab 1 partly outside",
           "128-channel tile, slab 1 wholly outside", "OC not a multiple of 8", "stacked images", "boxes over the edge",
           ">= 3 work items per CTA", "stride 2", RES_255, RES_SUBNORMAL]
    own += ["%s on %d-channel tiles" % (act, nb) for act in ("tanh", "sigmoid", "SiLU", "leakyRelu") for nb in (64, 128)]
    own += ["%s padding, IC %s" % (mode, ic) for mode in ("reflect", "replicate") for ic in (">= 16", "<= 8 on a pre-padded copy")]
    return umma + ["split-K TERMS=%d" % t for t in (1, 2, 3)] + ["%s [%s]" % (key, f) for f in FORMS for key in own]


def write_case(row, path, seed):
    """The case model of `row`: the residual source (constant padding, linear), the tested convolution (BatchNorm folded in, the row's
    padding mode) and the Add with the row's activation. Separate weights keep the two operands uncorrelated, of the same magnitude.
    The biases and the BatchNorm shift scale with the row's input scale, so that the products, not the shifts, set the magnitude of
    the residual and of the output."""
    n, h, w, ic, oc, k, s, padding, mode, act, scale = row
    b = modelzoo.Builder(seed)
    x = b.input(w, h, ic)
    src = b.conv(x, oc, k, s, padding, "linear", bias=True, mode=src_mode(row))
    conv = b.conv(x, oc, k, s, padding, "linear", bias=True, bn=True, mode=mode)
    add = b.add(conv, src, act)
    for i in (src, conv):
        b.layers[i]["_w"]["bias"] = (b.layers[i]["_w"]["bias"] * scale).astype(np.float32)
    for key in ("beta", "moving_mean"):
        b.layers[conv]["_bn"][key] = (b.layers[conv]["_bn"][key] * scale).astype(np.float32)
    if act == "leakyRelu":
        b.layers[add]["leakyReluAlpha"] = 0.1
    modelzoo.write_model(b.layers, path, split=True)


def case_input(row, seed):
    n, h, w, ic = row[:4]
    return (np.random.default_rng(seed).uniform(-1, 1, (n, h, w, ic)) * row[10]).astype(np.float32)


def restate_case(om, x_stored, residual, conv_kernel_name, shape, precision, at=None):
    """exact.conv2d of the Add's output (fused conv + residual + activation) through test_layer_exact_gpu.restate; at: the output
    pixels to restate (exact.py)."""
    outs = [x_stored, residual, None, None]
    kernels = {"names": ["", "", conv_kernel_name, ""], "shapes": [None, None, None, shape]}
    return restate(om, ADD, outs, kernels, precision, precision == "fp16", None, at=at)


def kernel_name(p):
    return "conv_umma_kernel<stream-K>" if p["sk"] else ("conv_umma_kernel<split-K>" if p["ksplit"] > 1 else "conv_umma_kernel")


def run_case(ctx, tmp, row, precision, sms, seed, stream_k=False):
    """Both runs of one case; returns (plan, worst |err| / bound, what, the residual-scale keys both runs' residuals earn)."""
    n, h, w, ic, oc, k, s, padding, mode, act, scale = row
    what = "n%d %dx%d ic%d oc%d k%d s%d %s %s %s x%g" % (n, h, w, ic, oc, k, s, mode or "zero", act or "linear", precision, scale)
    path = os.path.join(tmp, "res_%d_%s_%d.json" % (seed, precision, int(stream_k)))
    write_case(row, path, seed)
    p = case_plan(row, precision, sms, stream_k)
    ps = case_plan(row, precision, sms, stream_k, layer=SRC)
    assert p["path"] == cp.IGEMM, (what, p["path"])
    m = core.MixedInferenceCore(ctx, path, batch=n, precision=precision, fuse=True)
    runs = []
    try:
        for r in range(2):
            img = case_input(row, 1000 * seed + r)
            m.set_input(img)
            m.forward()
            ctx.sync()
            v = ctx.last_conv_variant()
            assert v == plan_variant(p), (what, "run %d" % r, v, plan_variant(p))
            runs.append((img, m.layer_output(0), m.layer_output(SRC), m.layer_output(ADD)))
        m.time_layers()
        names = [m.layer_kernel(i) for i in range(m.num_layers)]
        shape = m.layer_info(ADD)[2]
    finally:
        m.close()
    assert names[CONV] == kernel_name(p) and names[ADD] == "", (what, names)
    assert conv_kernel(names[SRC]) == KERNEL_OF_PATH[plan_variant(ps)["path"]], (what, names[SRC], ps["path"])
    om = oracle.Model(path)
    worst = 0.0
    res_keys = set(residual_keys(runs[0][2], precision)) & set(residual_keys(runs[1][2], precision))
    for r, (img, xin, res, got) in enumerate(runs):
        assert np.array_equal(xin, exact.model_input(img, precision == "fp16")[0]), (what, "input upload")
        ref, bound = restate_case(om, xin, res, names[CONV], shape, precision)
        assert got.shape == ref.shape, (what, got.shape, ref.shape)
        ratio, bad = exact.check(got, ref, bound, "Add")
        assert bad == 0, "%s (%s), run %d: %d elements outside the bound, worst |err|/bound %.3g" % (what, variant_key(plan_variant(p)), r, bad, ratio)
        worst = max(worst, ratio)
    return p, worst, what, sorted(res_keys)


def run_table(ctx, tmp, table, precisions, stream_k=False):
    import torch
    sms = torch.cuda.get_device_properties(ctx.device).multi_processor_count
    seen = {}
    for precision in precisions:
        for i, row in enumerate(table):
            p, ratio, what, res_keys = run_case(ctx, tmp, row, precision, sms, seed=i, stream_k=stream_k)
            for key in case_keys(row, precision, p) + res_keys:
                seen.setdefault(key, (what, ratio))
    return seen


def child_main():
    """SNNB_SK=1 child: run SK_TABLE in every product form and print what it covered as one JSON line."""
    import tempfile
    ctx = core.GpuContext(0)
    with tempfile.TemporaryDirectory() as tmp:
        seen = run_table(ctx, tmp, SK_TABLE, FORMS, stream_k=True)
    ctx.close()
    print("SEEN " + json.dumps(seen))


def test_every_residual_instantiation(ctx, tmp_path):
    seen = run_table(ctx, str(tmp_path), TABLE, FORMS)
    env = dict(os.environ, SNNB_SK="1")
    code = "import sys; sys.path[:0] = [%r, %r]; import test_residual_exact_gpu as t; t.child_main()" % (HERE, os.path.dirname(HERE))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("SEEN ")][-1]
    for key, val in json.loads(line[5:]).items():
        seen.setdefault(key, tuple(val))
    want = required_keys()
    for key in want:
        print("%-58s %s" % (key, "%s (worst |err|/bound %.3g)" % seen[key] if key in seen else "NOT COVERED"))
    missing = [k for k in want if k not in seen]
    assert not missing, missing
