"""Layer-local, teacher-forced checks: every layer's output held to oracle/exact.py's float64 restatement of that one layer, fed
the engine's own inputs (the layer outputs of its producers), within a per-element bound derived from the operands. Nothing
accumulates with depth, so the bounds are those of one layer's arithmetic.

- Instantiation table: single-convolution models that between them launch all 18 conv_umma_kernel<TERMS, NB, SK> and all 24
  conv_rowwin_kernel<TERMS, FKS, NB> instantiations, and split-K in each TERMS. Each case asserts through
  snnb_debug_last_conv_variant the path, product form and whatever of the tile width, feed K steps and K split its shape decides;
  together they must launch every instantiation. The engine never asks for stream-K, so those cases run in a child process with
  SNNB_SK=1, which makes the planner consider it.
- Whole zoo models in fp32x3, fp16w and fp16, fused and unfused, and on the CUDA-core convolution: every layer with a tensor of
  its own is restated (only YOLO's host decode is not).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import exact, oracle
from shadernn_b200 import core, modelzoo

pytestmark = pytest.mark.gpu

FORMS = ("fp32x3", "fp16w", "fp16")
HERE = os.path.dirname(os.path.abspath(__file__))


def variant_key(v):
    """The kernel instantiation a variant record names, as it appears in the library's symbols."""
    if v["path"] == "igemm":
        return "conv_umma_kernel<%d, %d, %s>" % (v["terms"], v["n_blk"], "true" if v["stream_k"] else "false")
    if v["path"] in ("rowwin", "rowwin-feed"):
        return "conv_rowwin_kernel<%d, %d, %d>" % (v["terms"], v["fks"], v["n_blk"])
    return v["path"]


def conv_params(layer, k):
    """(pad_x, pad_y, pad_mode) the engine gives the kernels for a Conv2D layer, as the oracle's walker reads them."""
    o = oracle.Model._offsets(layer, k)
    mode = layer.get("mode", "") if isinstance(layer.get("padding"), list) and isinstance(layer["padding"][0], list) else ""
    px, py = (0, 0) if k == 1 else (o[0], o[2])
    return px, py, mode or "constant"


def conv_form(kernel_name, precision):
    return "simt" if kernel_name.startswith("conv2d_simt") else precision


def conv_kernel(kernel_name):
    """exact.conv2d's kernel argument for the kernel a layer launched (MixedInferenceCore.layer_kernel)."""
    if kernel_name.startswith("conv_umma"):
        return "igemm"
    if kernel_name == "conv_rowwin_kernel<feed>":
        return "feed"
    if kernel_name.startswith("conv_rowwin"):
        return "rowwin"
    return "simt"


KERNEL_OF_PATH = {"igemm": "igemm", "rowwin": "rowwin", "rowwin-feed": "feed", "simt": "simt"}


def run_single_conv(ctx, tmp, n, h, w, ic, oc, k, s, padding, act, precision, scale=1.0, seed=0, bn=True):
    """One Conv2D model: returns (variant, worst |err| / bound, what)."""
    b = modelzoo.Builder(seed)
    x = b.input(w, h, ic)
    b.conv(x, oc, k, s, padding, act, bias=True, bn=bn)
    path = os.path.join(tmp, "conv_%d_%d_%d_%d_%d_%d_%d_%d_%s_%s.json" % (n, h, w, ic, oc, k, s, seed, act, precision))
    modelzoo.write_model(b.layers, path, split=True)
    rng = np.random.default_rng(seed + 1)
    img = (rng.uniform(-1, 1, (n, h, w, ic)) * scale).astype(np.float32)
    m = core.MixedInferenceCore(ctx, path, batch=n, precision=precision)
    try:
        m.set_input(img)
        m.forward()
        ctx.sync()
        v = ctx.last_conv_variant()
        xin, got = m.layer_output(0), m.layer_output(1)
    finally:
        m.close()
    half = precision == "fp16"
    ref_in, _ = exact.model_input(img, half)
    assert np.array_equal(xin, ref_in), "input upload"
    om = oracle.Model(path)
    lw = om.w[1]
    px, py, mode = conv_params(om.layers[1], k)
    ref, bound = exact.conv2d(xin, lw["kernel"], lw.get("bias"), lw.get("bn"), s, px, py, got.shape[1:3], act, 0.1,
                              form=precision if v["path"] != "simt" else "simt", kernel=KERNEL_OF_PATH[v["path"]], half_out=half, pad_mode=mode)
    ratio, bad = exact.check(got, ref, bound, "conv")
    what = "n%d %dx%d ic%d oc%d k%d s%d %s %s x%g" % (n, h, w, ic, oc, k, s, act, precision, scale)
    assert bad == 0, "%s (%s): %d elements outside the bound, worst |err|/bound %.3g" % (what, variant_key(v), bad, ratio)
    return v, ratio, what


def feed_k(fks):
    """A stride-2, 'same'-padded stem kernel size whose feed plan has `fks` K steps per filter row (3 input channels)."""
    import ctypes as C
    from shadernn_b200._lib import lib
    for k in range(2, 16):
        pad = oracle.same_padding(k, True)[0]
        out = (C.c_int * 5)()
        if lib().snnb_debug_feed_plan(k, 2, pad, 3, out) and out[3] == fks:
            return k
    return None


# (n, h, w, ic, oc, k, s, padding, act, input scale): shapes where kernels break - channel tails, overhanging tiles and images stacked
# in one tile, 1x1 maps, stride 2 with odd sizes, the zoo's longest K (3x3x512), inputs at Candy's 0..255 scale and in fp16's
# subnormal range
TABLE = [
    (2, 15, 13, 20, 24, 3, 1, "same", "relu", 1.0),
    (3, 9, 11, 40, 56, 3, 1, "same", "leakyRelu", 1.0),
    (4, 28, 28, 64, 56, 1, 1, "valid", "relu6", 1.0),
    (2, 29, 31, 64, 96, 3, 2, "same", "relu", 1.0),
    (2, 28, 28, 72, 200, 1, 1, "valid", "tanh", 1.0),
    (4, 1, 1, 1280, 200, 1, 1, "valid", "", 1.0),
    (2, 7, 7, 512, 512, 3, 1, "same", "relu", 1.0),
    (1, 14, 14, 520, 72, 3, 1, "same", "SiLU", 1.0),
    (2, 30, 30, 32, 48, 3, 1, "same", "sigmoid", 255.0),
    (2, 12, 17, 48, 136, 3, 1, "same", "", 1e-4),
    (2, 56, 56, 64, 128, 3, 1, "same", "relu", 1.0),
    (8, 14, 14, 256, 24, 3, 2, "same", "relu", 1.0),
    (33, 32, 32, 64, 256, 1, 1, "valid", "relu", 1.0),  # several waves of tiles: the widest tile (NB = 128) pays off in every form
    # conv_rowwin_kernel (<= 8 input channels), stride 1 (FKS = 0) and 2
    (2, 40, 52, 3, 24, 3, 1, "same", "relu", 1.0),
    (1, 33, 29, 4, 48, 3, 1, "same", "tanh", 1.0),
    (1, 21, 300, 8, 40, 5, 1, "same", "", 255.0),
    (2, 37, 41, 3, 24, 9, 2, "same", "relu", 1.0),
    (1, 30, 30, 1, 64, 5, 1, "same", "leakyRelu", 1e-4),
]
# stream-K (SNNB_SK=1): tile counts that leave a partial last wave on 132 SMs
SK_TABLE = [
    (32, 28, 28, 128, 128, 3, 1, "same", "relu", 1.0),
    (32, 28, 28, 128, 48, 3, 1, "same", "relu", 1.0),
    (32, 28, 28, 128, 24, 3, 1, "same", "", 1.0),
    (9, 14, 14, 256, 256, 3, 1, "same", "relu", 1.0),
    (5, 33, 21, 64, 96, 3, 2, "same", "relu", 1.0),
    (9, 14, 14, 256, 56, 3, 1, "same", "", 1.0),
    (9, 14, 14, 256, 24, 3, 1, "same", "", 1.0),
    (34, 32, 32, 64, 256, 3, 1, "same", "relu", 1.0),
    (34, 32, 32, 64, 96, 3, 1, "same", "", 1.0),
    (9, 14, 14, 256, 96, 3, 1, "same", "relu", 1.0),
    (17, 16, 32, 64, 256, 3, 1, "same", "relu", 1.0),  # ~136 tiles of 128 channels: one wave and a few, cut into K pieces
    (35, 16, 16, 64, 256, 3, 1, "same", "", 1.0),
]


def feed_table():
    rows = []
    for fks in (1, 2, 3):
        k = feed_k(fks)
        assert k is not None, "no stem kernel size has %d feed K steps" % fks
        rows += [(2, 2 * k + 23, 2 * k + 41, 3, 24, k, 2, "same", "relu", 1.0), (1, 2 * k + 17, 131, 3, 40, k, 2, "same", "", 1.0)]
    return rows


def expected_variant(row, precision, stream_k):
    """What a single-convolution case must launch, as far as its shape decides it (the tile width of conv_umma_kernel is the
    planner's cost model's choice, and differs between product forms, unless OC <= 32 leaves only 32)."""
    n, h, w, ic, oc, k, s, padding, act, scale = row
    want = {"terms": exact.TERMS[precision]}
    if ic <= 8:
        feed = s == 2 and ic <= 4
        want["path"] = "rowwin-feed" if feed else "rowwin"
        want["n_blk"] = 32 if oc <= 32 else 64  # rowwin_nblk
        want["fks"] = len(exact.feed_plan_steps(k, oracle.same_padding(k, True)[0])) if feed else 0
    else:
        want["path"] = "igemm"
        if oc <= 32:
            want["n_blk"] = 32
        if not stream_k and ic * k * k >= 4608 and n * h * w <= 128:  # the zoo's longest K on one 128-row tile: split-K in every form
            want["ksplit_gt1"] = True
    return want


def run_table(ctx, tmp, table, precisions, stream_k=False):
    seen = {}
    for precision in precisions:
        for i, row in enumerate(table):
            n, h, w, ic, oc, k, s, padding, act, scale = row
            v, ratio, what = run_single_conv(ctx, tmp, n, h, w, ic, oc, k, s, padding, act, precision, scale, seed=i)
            want = expected_variant(row, precision, stream_k)
            got = {key: (v["ksplit"] > 1 if key == "ksplit_gt1" else v[key]) for key in want}
            assert got == want, (what, v, want)
            key = variant_key(v)
            seen.setdefault(key, (what, ratio))
            if v["ksplit"] > 1:
                seen.setdefault("split-K TERMS=%d" % v["terms"], (what, ratio))
    return seen


def child_main():
    """SNNB_SK=1 child: run SK_TABLE in every product form and print what it launched as one JSON line."""
    import tempfile
    ctx = core.GpuContext(0)
    with tempfile.TemporaryDirectory() as tmp:
        seen = run_table(ctx, tmp, SK_TABLE, FORMS, stream_k=True)
    ctx.close()
    print("SEEN " + json.dumps(seen))


def expected_instantiations():
    umma = ["conv_umma_kernel<%d, %d, %s>" % (t, nb, sk) for t in (1, 2, 3) for nb in (32, 64, 128) for sk in ("false", "true")]
    rowwin = ["conv_rowwin_kernel<%d, %d, %d>" % (t, f, nb) for t in (1, 2, 3) for f in range(4) for nb in (32, 64)]
    return umma + rowwin


def test_every_tensor_core_instantiation(ctx, tmp_path):
    seen = run_table(ctx, str(tmp_path), TABLE + feed_table(), FORMS)
    env = dict(os.environ, SNNB_SK="1")
    code = "import sys; sys.path[:0] = [%r, %r]; import test_layer_exact_gpu as t; t.child_main()" % (HERE, os.path.dirname(HERE))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("SEEN ")][-1]
    for key, val in json.loads(line[5:]).items():
        seen.setdefault(key, tuple(val))
    want = expected_instantiations()
    for key in want + ["split-K TERMS=%d" % t for t in (1, 2, 3)]:
        print("%-36s %s" % (key, "%s (worst |err|/bound %.3g)" % seen[key] if key in seen else "NOT LAUNCHED"))
    missing = [k for k in want if k not in seen]
    assert not missing, missing
    assert all(("split-K TERMS=%d" % t) in seen for t in (1, 2, 3)), sorted(seen)


# ---- whole models, teacher-forced -------------------------------------------------------------------------------------------
def restate(om, i, outs, kernels, precision, half, x):
    """exact.* for layer i of oracle.Model om from the engine outputs `outs` of its producers (None where fusion hid them).
    Returns (ref, bound), or None when a hidden producer makes the layer one this restatement does not cover."""
    l = om.layers[i]
    t = om.type_of(l)
    w = om.w[i]
    act = l.get("activation", "linear")
    ins = [int(v) for v in l.get("inputId", [])][:int(l.get("numInputs", 0))]
    if t == "InputLayer":
        return exact.model_input(x, half)
    outs = list(outs)
    for j in ins:  # a constant Pad folded into its consumer: zero padding composes, so restate it as a tensor (pure data movement)
        p = om.layers[j]
        if outs[j] is None and om.type_of(p) == "Pad" and p.get("mode", "constant") in ("constant", ""):
            up = int(p["inputId"][0])
            if outs[up] is not None:
                o = om._offsets(p, 0, False) if "pads" not in p else [int(p["pads"][2]), int(p["pads"][6]), int(p["pads"][3]), int(p["pads"][7])]
                outs[j] = exact.pad(outs[up], o[0], o[2], kernels["shapes"][j][1:3])[0]
    if t == "Add" and any(outs[j] is None for j in ins):
        # a Conv2D fused into this Add: its epilogue adds the other operand and applies the Add's activation
        j = [j for j in ins if outs[j] is None][0]
        other = [q for q in ins if q != j][0]
        if om.type_of(om.layers[j]) != "Conv2D" or outs[other] is None:
            return None
        return restate_conv(om, j, outs, kernels, precision, half, act=act, alpha=float(l.get("leakyReluAlpha", l.get("alpha", 0.3))),
                            residual=outs[other], shape_of=i)
    if t == "Dense" and any(outs[j] is None for j in ins):
        # the fused global average pool + dense (+ soft-max) head
        j = ins[0]
        src = om.layers[j]
        while outs[j] is None and om.type_of(src) in ("Flatten", "AveragePooling2D"):
            j = [int(v) for v in src["inputId"]][0]
            src = om.layers[j]
        if outs[j] is None:
            return None
        return exact.gap_dense(outs[j], w["kernel"], w.get("bias"), "" if act == "softmax" else act, softmax_out=act == "softmax", half_out=half)
    if t == "Conv2D":
        return restate_conv(om, i, outs, kernels, precision, half, act=act, alpha=float(l.get("leakyReluAlpha", l.get("alpha", 0.0))))
    if any(outs[j] is None for j in ins):
        return None
    a = outs[ins[0]]
    n, h, wd, c = a.shape
    shape = kernels["shapes"][i]
    if t == "SeparableConv2D":
        k, s = int(l["kernel_size"]), int(l["strides"])
        o = om._offsets(l, k)
        return exact.depthwise(a, w["kernel"], w.get("bias"), w.get("bn"), s, o[0], o[2], shape[1:3], act, float(l.get("leakyReluAlpha", l.get("alpha", 0.0))), half)
    if t == "MaxPooling2D":
        pool = l.get("pool", l.get("pool_size"))
        k = int(pool[0] if isinstance(pool, list) else pool)
        s = l.get("stride", l.get("strides", k))
        return exact.maxpool(a, k, int(s[0] if isinstance(s, list) else s), shape[1:3])
    if t == "AveragePooling2D":
        pool = l.get("pool", l.get("pool_size"))
        k = int(pool[0] if isinstance(pool, list) else pool)
        s = l.get("stride", k)
        return exact.avgpool(a, k, int(s[0] if isinstance(s, list) else s), shape[1:3], half)
    if t == "Add":
        return exact.add(a, outs[ins[1]], act, float(l.get("leakyReluAlpha", l.get("alpha", 0.3))), half)
    if t == "InstanceNorm":
        return exact.instancenorm(a, w["gamma"], w["beta"], act, float(l.get("leakyReluAlpha", 0.0)), half)
    if t == "BatchNormalization":
        return exact.batchnorm(a, w["bn"], act, float(l.get("leakyReluAlpha", l.get("alpha", 0.0))), half)
    if t == "Activation":
        return exact.activation(a, act, float(l.get("leakyReluAlpha", 0.3)), half)
    if t == "Flatten":
        if act not in ("", "linear"):
            return None
        return exact.flatten(a)
    if t == "Dense":
        if act not in ("", "linear", "relu", "softmax"):
            return None
        ref, bound = exact.dense(a, w["kernel"], w.get("bias"), "" if act == "softmax" else act, form=precision, half_out=half)
        if act == "softmax":  # launch_dense stores the logits in the output tensor's format, then the soft-max reads them back
            ref, bound = exact.softmax_rows(ref.reshape(n, -1), bound.reshape(n, -1))
            ref, bound = ref.reshape(n, 1, 1, -1), bound.reshape(n, 1, 1, -1) + exact.store_bound(ref.reshape(n, 1, 1, -1), half)
        return ref, bound
    if t == "Concatenate":
        return exact.concat(a, outs[ins[1]])
    if t == "UpSampling2D":
        if l.get("interpolation") == "bilinear":
            return None
        return exact.upsample_nearest(a, shape[1:3])
    if t == "Pad":
        if "pads" in l:
            p = l["pads"]
            o = [int(p[2]), int(p[6]), int(p[3]), int(p[7])]
        else:
            o = om._offsets(l, 0, False)
        return exact.pad(a, o[0], o[2], shape[1:3], l.get("mode", "constant"))
    if t == "Subpixel":
        return exact.subpixel(a, int(l.get("kernel_size", 2)), half)
    return None


def restate_conv(om, j, outs, kernels, precision, half, act, alpha, residual=None, shape_of=None):
    l = om.layers[j]
    k, s = int(l["kernel_size"]), int(l["strides"])
    src = [int(v) for v in l["inputId"]][0]
    x = outs[src]
    px, py, mode = conv_params(l, k)
    if x is None:
        return None
    kern = conv_kernel(kernels["names"][j])
    w = om.w[j]
    shape = kernels["shapes"][shape_of if shape_of is not None else j]
    return exact.conv2d(x, w["kernel"], w.get("bias"), w.get("bn"), s, px, py, shape[1:3], act, alpha, residual=residual,
                        form=conv_form(kernels["names"][j], precision), kernel=kern, half_out=half, pad_mode=mode)


def teacher_forced(ctx, name, hw, batch, model_dir, precision, fuse, conv_algo="auto", **kw):
    from shadernn_b200._lib import SnnbError
    path, _ = modelzoo.build(name, model_dir, input_hw=hw, **kw)
    x = modelzoo.synthetic_input(name, batch, hw)
    om = oracle.Model(path)
    m = core.MixedInferenceCore(ctx, path, batch=batch, input_hw=hw, fuse=fuse, conv_algo=conv_algo, precision=precision)
    try:
        m.set_input(x)
        m.forward()
        ctx.sync()
        outs = []
        for i in range(m.num_layers):
            t = om.type_of(om.layers[i])
            if t == "YOLO" or (fuse and t in ("Pad", "Flatten")):
                outs.append(None)  # no tensor of its own; fused, a Pad or Flatten is an alias of its producer's tensor or folded away
                continue
            try:
                outs.append(m.layer_output(i))
            except SnnbError:
                assert fuse, m.layer_info(i)[0]  # only fusion may hide a layer
                outs.append(None)
        m.time_layers()
        kernels = {"names": [m.layer_kernel(i) for i in range(m.num_layers)], "shapes": [m.layer_info(i)[2] for i in range(m.num_layers)]}
    finally:
        m.close()
    half = precision == "fp16"
    worst, checked, skipped = 0.0, 0, []
    for i in range(om.count):
        t = om.type_of(om.layers[i])
        if outs[i] is None or t == "YOLO":
            continue
        r = restate(om, i, outs, kernels, precision, half, x)
        if r is None:
            skipped.append("%d:%s" % (i, t))
            continue
        ref, bound = r
        got = outs[i]
        assert got.shape == ref.shape, (name, i, t, got.shape, ref.shape)
        ratio, bad = exact.check(got, ref, bound, t)
        assert bad == 0, "%s %s fuse=%d %s: layer %d (%s, %s): %d elements outside the bound, worst |err|/bound %.3g" % (
            name, precision, int(fuse), conv_algo, i, t, kernels["names"][i], bad, ratio)
        worst = max(worst, ratio)
        checked += 1
    print("%-12s %4dx%-4d batch %2d %-6s fuse=%d %-4s: %3d layers, worst |err|/bound %.3g%s" % (
        name, hw[0], hw[1], batch, precision, int(fuse), conv_algo, checked, worst, (" (not restated: %s)" % ", ".join(skipped)) if skipped else ""))
    assert not skipped, "layers without a restatement: %s" % skipped
    return worst


ZOO = [("resnet18", (64, 64), 2, {}), ("mobilenetv2", (64, 64), 2, {"classes": 100}), ("yolov3tiny", (128, 128), 1, {}),
       ("candy", (48, 48), 1, {}), ("espcn", (48, 48), 2, {}), ("unet", (64, 64), 1, {})]


@pytest.mark.parametrize("precision", FORMS)
@pytest.mark.parametrize("fuse", [False, True])
@pytest.mark.parametrize("name,hw,batch,kw", ZOO, ids=[z[0] for z in ZOO])
def test_zoo_teacher_forced(ctx, model_dir, name, hw, batch, kw, precision, fuse):
    teacher_forced(ctx, name, hw, batch, model_dir, precision, fuse, **kw)


@pytest.mark.parametrize("precision", FORMS)
def test_zoo_teacher_forced_simt(ctx, model_dir, precision):
    for name, hw, batch, kw in ZOO:
        teacher_forced(ctx, name, hw, batch, model_dir, precision, False, conv_algo="simt", **kw)


@pytest.mark.parametrize("precision", FORMS)
def test_resnet18_baseline_size_teacher_forced(ctx, model_dir, precision):
    teacher_forced(ctx, "resnet18", (224, 224), 2, model_dir, precision, True)
