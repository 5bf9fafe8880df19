"""Partial batches without a GPU (snnb_model_set_batch): the entry point is exported and refuses a null model, the Python wrapper fails
as every other call does, and the planner gives the convolutions of the models tests/test_partial_batch_gpu.py switches between batch
sizes a launch configuration per batch size with the path, pre-padded copy and feed copy of the loaded batch's plan, which is what
MixedInferenceCore::setBatch asserts before it switches."""
import numpy as np
import pytest

import test_conv_plan as cp
from shadernn_b200 import _lib, modelzoo

# the first ten fields of snnb_debug_conv_launch: what the engine allocates and packs for at load (kernel, pre-padded copy, feed copy)
DECISION = cp.FIELDS[:10]
LAUNCH = ("n_blk", "tiles_x", "grid", "tw", "th", "tn", "tiles_y", "tiles_n", "tiles_oc", "ksplit", "kb_per_split")


def test_set_batch_refuses_a_null_model(built):
    lib = _lib.lib()
    assert lib.snnb_model_set_batch(None, 1) != 0
    assert b"snnb_model_set_batch: null model" in lib.snnb_last_error()


def test_python_set_batch_fails_loudly_without_a_model(built):
    from shadernn_b200.core import MixedInferenceCore
    m = MixedInferenceCore.__new__(MixedInferenceCore)
    m.h, m.batch, m.max_batch = None, 8, 8
    with pytest.raises(_lib.SnnbError) as e:
        m.set_batch(2)
    assert "snnb_model_set_batch: null model" in str(e.value)
    assert m.batch == 8  # a refused call changes nothing


def model_convs(name, hw, **kw):
    """(input hwc, output hwc, k, stride, pad_x, pad_y, pad mode, reads a model input) of every Conv2D of a zoo model at `hw`."""
    layers = modelzoo.MODELS[name][0](hw, **kw)
    x = modelzoo.synthetic_input(name, 1, hw)
    last = max(i for i, l in enumerate(layers) if l["type"] == "Conv2D")
    outs = modelzoo.torch_forward(layers, x, upto=last)
    convs = []
    for i, l in enumerate(layers[:last + 1]):
        if l["type"] != "Conv2D":
            continue
        src = l["inputId"][0]
        k, s = int(l["kernel_size"]), int(l["strides"])
        o = modelzoo._pad4(l, k)
        mode = {"constant": cp.PAD_CONSTANT, "reflect": cp.PAD_REFLECT, "replicate": cp.PAD_REPLICATE}[l.get("mode", "constant")] if "mode" in l \
            else cp.PAD_NONE
        convs.append((np.shape(outs[src])[1:], np.shape(outs[i])[1:], k, s, 0 if k == 1 else o[0], 0 if k == 1 else o[2], mode,
                      layers[src]["type"] == "InputLayer"))
    return convs


# (model, input size, loaded batch, builder arguments): the models of the GPU tests, and ResNet-18 at its benchmark size and batch
MODELS = [("resnet18", (64, 64), 8, {}), ("resnet18", (224, 224), 32, {}), ("yolov3tiny", (416, 416), 4, {}), ("candy", (48, 64), 4, {}),
          ("espcn", (24, 40), 4, {}), ("unet", (64, 64), 4, {"classes": 1}), ("unet", (64, 64), 4, {"classes": 21})]


@pytest.mark.parametrize("name,hw,batch,kw", MODELS, ids=["%s-%dx%d-b%d%s" % (m[0], m[1][0], m[1][1], m[2], "".join("-%s%s" % i for i in m[3].items()))
                                                          for m in MODELS])
def test_every_batch_size_keeps_the_loaded_decision(built, name, hw, batch, kw):
    convs = model_convs(name, hw, **kw)
    assert convs
    for in_hwc, out_hwc, k, s, px, py, mode, from_input in convs:
        for precision in cp.FORMS:
            args = dict(pad_mode=mode, may_feed=from_input, precision=precision)
            at_b = cp.plan(in_hwc, out_hwc, k, s, px, py, n=batch, **args)
            for n in sorted({1, 2, 3, batch - 1}):
                got = cp.plan(in_hwc, out_hwc, k, s, px, py, n=n, **args)
                assert {f: got[f] for f in DECISION} == {f: at_b[f] for f in DECISION}, (name, in_hwc, out_hwc, k, s, precision, n)
                assert got["n"] == n


def test_resnet18_deep_convolutions_are_planned_per_batch():
    # ResNet-18 224 x 224: the 3x3 convolutions of 512 channels on 7 x 7 maps (9 x 8 = 72 K blocks). The restatement of plan_tiles /
    # plan_oc_ksplit (test_conv_plan.py) and the library agree: 64-channel tiles without a K split at 32 images, 32-channel tiles split
    # four ways at 1 image, whose one 49-pixel tile would otherwise keep few of the 132 SMs busy.
    want = {32: (64, 1), 1: (32, 4)}
    for n, (n_blk, ksplit) in want.items():
        tp = cp.plan_tiles(n, 7, 7, 1)
        op = cp.plan_oc_ksplit(512, tp["tiles_x"] * tp["tiles_y"] * tp["tiles_n"], tp["tw"] * tp["th"] * tp["tn"], 9 * 512 // 64, cp.SMS, 3, False)
        assert (op["n_blk"], op["ksplit"]) == (n_blk, ksplit), n
        got = cp.plan((7, 7, 512), (7, 7, 512), 3, 1, 1, 1, pad_mode=cp.PAD_NONE, n=n)
        assert (got["n_blk"], got["ksplit"]) == (n_blk, ksplit), n
        assert got["path"] == cp.IGEMM
    one, full = (cp.plan((7, 7, 512), (7, 7, 512), 3, 1, 1, 1, pad_mode=cp.PAD_NONE, n=n) for n in (1, 32))
    assert {f: one[f] for f in DECISION} == {f: full[f] for f in DECISION}
    assert {f: one[f] for f in LAUNCH} != {f: full[f] for f in LAUNCH}
