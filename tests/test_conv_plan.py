"""The convolution planner (csrc/conv_plan.cpp, plan_conv), evaluated on the host through snnb_debug_conv_plan: which kernel runs a
convolution, whether it reads a pre-padded copy of its input and whether a model input gets the compact feed copy.

The expected values restate the rules the engine and the C-ABI applied before the decision was moved into one planner: the
tensor-core support predicates of kernels_umma.cu (rowwin_supported, feed_usable and the implicit-GEMM limits), the packing predicates
of pack.cpp (pack_rowwin_host, pack_feed_host), Conv2DLayer's pre-pad probe and the feed conditions and feed-copy geometry of
MixedInferenceCore::init. `reference_plan` below is that rule set; the tables pin each limit on both sides with literal paths too."""
import ctypes as C

import numpy as np
import pytest

from shadernn_b200 import modelzoo
from shadernn_b200._lib import lib

REFUSED, SIMT, IGEMM, ROWWIN, FEED = 0, 1, 2, 3, 4
AUTO, ALGO_SIMT, TCGEN05, STREAMK = 0, 1, 2, 3
PAD_NONE, PAD_CONSTANT, PAD_REPLICATE, PAD_REFLECT = 0, 1, 2, 3
RW_BOXW, RW_ARR_BYTES, RW_B_MAX_BYTES = 144, 144 * 16, 227 * 1024 - 1024 - 512 - 2 * 128 * 128 - 4 * 4 * 144 * 16


def plan(in_hwc, out_hwc, k, stride, pad_x, pad_y, pad_mode=PAD_CONSTANT, residual=False, algo=AUTO, may_prepad=True, may_feed=False,
         row=None, feed_pad=None):
    """snnb_debug_conv_plan. row / feed_pad default to what the engine packs (Conv2DLayer::plan); pass them for C-ABI weights."""
    zero = pad_mode in (PAD_NONE, PAD_CONSTANT)
    row = (stride, pad_x if zero else 0) if row is None else row
    feed_pad = pad_x if feed_pad is None else feed_pad
    q = [*in_hwc, *out_hwc, k, stride, pad_x, pad_y, pad_mode, int(residual), algo, int(may_prepad), int(may_feed), row[0], row[1], feed_pad]
    out = (C.c_int * 10)()
    assert lib().snnb_debug_conv_plan((C.c_int * 18)(*q), out) == 0
    return dict(zip(["path", "pad_x", "pad_y", "pad_mode", "prepad_h", "prepad_w", "feed_h", "feed_w", "feed_py", "feed_px"], list(out)))


# ---- the rules before the planner ------------------------------------------------------------------------------------------
def _row_plan(k, stride, pad_x):  # make_row_plan: (K steps, span) or None
    if k < 1 or k > 9 or stride not in (1, 2):
        return None
    ksteps = span = 0
    for par in range(stride):
        t = sum(1 for j in range(k) if (j - pad_x) % stride == par)
        if t:
            ksteps += (t + 1) // 2
            span = max(span, 2 * ((t + 1) // 2))
    return (ksteps, span) if 0 < ksteps <= 8 else None


def _feed_plan(k, stride, pad_x, ic):  # make_feed_plan: (px, nch, rows_per_panel) or None
    if stride != 2 or ic > 4 or k < 2 or k > 9 or pad_x < 0 or pad_x > 8:
        return None
    px = (pad_x + 1) & ~1
    nch = ((px - pad_x + k + 1) // 2 + 1) & ~1
    ks = nch // 2
    return (px, nch, 4 if ks == 1 else (2 if ks == 2 else 1)) if ks <= 4 else None


def reference_plan(in_hwc, out_hwc, k, stride, pad_x, pad_y, pad_mode=PAD_CONSTANT, residual=False, algo=AUTO, may_prepad=True, may_feed=False,
                   row=None, feed_pad=None):
    (ih, iw, ic), (oh, ow, oc) = in_hwc, out_hwc
    zero = pad_mode in (PAD_NONE, PAD_CONSTANT)
    row = (stride, pad_x if zero else 0) if row is None else row
    feed_pad = pad_x if feed_pad is None else feed_pad
    has_row = ic <= 8 and oc <= 64 and _row_plan(k, row[0], row[1]) is not None   # pack_rowwin_host

    def rowwin(px, res, fp):  # rowwin_supported
        rp = _row_plan(k, stride, px)
        if not (ic <= 8 and has_row and row == (stride, px) and oc <= 64 and not res and rp and 128 + rp[1] <= RW_BOXW):
            return False
        wrows = -(-k // fp[2]) if fp else k * ((rp[0] + 3) // 4)
        return wrows * 2 * (32 if oc <= 32 else 64) * 128 <= RW_B_MAX_BYTES

    def igemm(px, py):
        return stride in (1, 2) and ic >= 16 and 1 <= k <= 11 and px <= 127 and py <= 127

    want = {"path": SIMT, "pad_x": pad_x, "pad_y": pad_y, "pad_mode": pad_mode, "prepad_h": 0, "prepad_w": 0, "feed_h": 0, "feed_w": 0, "feed_py": 0,
            "feed_px": 0}
    forced = algo in (TCGEN05, STREAMK)  # (the engine plans SNNB_ALGO_TCGEN05_STREAMK as AUTO: Conv2DLayer::plan)
    if algo == ALGO_SIMT:
        return want
    if not zero:
        if may_prepad and k > 1 and (rowwin(0, False, None) or igemm(0, 0)):  # the pre-pad probe: pads 0, no residual
            want.update(path=ROWWIN if rowwin(0, residual, None) else IGEMM, pad_x=0, pad_y=0, pad_mode=PAD_CONSTANT,
                        prepad_h=(oh - 1) * stride + k, prepad_w=(ow - 1) * stride + k)
            return want
        want["path"] = REFUSED if forced else SIMT
        return want
    fp = _feed_plan(k, stride, pad_x, ic) if (may_feed and not residual and oc <= 64) else None  # MixedInferenceCore::init
    if fp and feed_pad == pad_x and has_row and (254 + 2 * fp[1]) * 8 <= RW_ARR_BYTES and rowwin(pad_x, residual, fp):
        need_w = 2 * (-(-ow // 128) * 128 - 1) + 2 * fp[1]
        want.update(path=FEED, feed_w=(max(iw + fp[0], need_w) + 1) & ~1, feed_h=max(ih + pad_y, 2 * (oh - 1) + k), feed_py=pad_y, feed_px=fp[0])
    elif rowwin(pad_x, residual, None):
        want["path"] = ROWWIN
    elif igemm(pad_x, pad_y):
        want["path"] = IGEMM
    else:
        want["path"] = REFUSED if forced else SIMT
    return want


def _out(n, k, s, p):
    return (n + 2 * p - k) // s + 1


def _conv(ic, oc, k=3, s=1, p=None, n=32, **kw):
    p = k // 2 if p is None else p
    o = _out(n, k, s, p)
    return (n, n, ic), (o, o, oc), k, s, p, p, kw


# (description, case, expected path) - each limit with a case on both sides
LIMITS = [
    ("IC 8: row window", _conv(8, 32), ROWWIN),
    ("IC 9: neither tensor kernel", _conv(9, 32), SIMT),
    ("IC 9 forced", _conv(9, 32, algo=TCGEN05), REFUSED),
    ("IC 16: implicit GEMM", _conv(16, 32), IGEMM),
    ("OC 64: row window", _conv(3, 64), ROWWIN),
    ("OC 65: no row-window operand", _conv(3, 65), SIMT),
    ("k 9 IC 32", _conv(32, 32, k=9), IGEMM),
    ("k 11 IC 32", _conv(32, 32, k=11), IGEMM),
    ("k 12 IC 32", _conv(32, 32, k=12, p=5), SIMT),
    ("k 9 IC 3 OC 32: two panels per row still resident", _conv(3, 32, k=9), ROWWIN),
    ("k 9 IC 3 OC 64: weight panels too large", _conv(3, 64, k=9), SIMT),
    ("k 11 IC 3: no row plan", _conv(3, 32, k=11), SIMT),
    ("stride 1", _conv(32, 64, s=1), IGEMM),
    ("stride 2", _conv(32, 64, s=2), IGEMM),
    ("stride 3", _conv(32, 64, s=3), SIMT),
    ("stride 2 IC 3", _conv(3, 64, s=2), ROWWIN),
    ("stride 3 IC 3", _conv(3, 64, s=3), SIMT),
    ("pad 127", ((8, 8, 32), (260, 260, 32), 3, 1, 127, 127, {}), IGEMM),
    ("pad_x 128", ((8, 8, 32), (262, 260, 32), 3, 1, 128, 127, {}), SIMT),
    ("pad_y 128", ((8, 8, 32), (260, 262, 32), 3, 1, 127, 128, {}), SIMT),
    ("reflect, pre-pad allowed", _conv(32, 64, pad_mode=PAD_REFLECT), IGEMM),
    ("replicate, pre-pad allowed", _conv(32, 64, pad_mode=PAD_REPLICATE), IGEMM),
    ("reflect, no pre-pad", _conv(32, 64, pad_mode=PAD_REFLECT, may_prepad=False), SIMT),
    ("reflect, no pre-pad, forced", _conv(32, 64, pad_mode=PAD_REFLECT, may_prepad=False, algo=TCGEN05), REFUSED),
    ("reflect stem 9x9 (Candy)", _conv(3, 32, k=9, pad_mode=PAD_REFLECT), ROWWIN),
    ("reflect 1x1", _conv(32, 64, k=1, pad_mode=PAD_REFLECT), SIMT),
    ("reflect IC 9", _conv(9, 64, pad_mode=PAD_REFLECT), SIMT),
    ("reflect stem with residual: implicit GEMM on the padded copy", _conv(3, 32, pad_mode=PAD_REFLECT, residual=True), IGEMM),
    ("constant with residual IC 3", _conv(3, 32, residual=True), SIMT),
    ("constant with residual IC 32", _conv(32, 32, residual=True), IGEMM),
    ("SIMT requested", _conv(32, 64, algo=ALGO_SIMT), SIMT),
    ("SIMT requested, reflect", _conv(32, 64, pad_mode=PAD_REFLECT, algo=ALGO_SIMT), SIMT),
    ("tcgen05 requested", _conv(32, 64, algo=TCGEN05), IGEMM),
    ("stream-K requested, IC 9", _conv(9, 32, algo=STREAMK, may_prepad=False), REFUSED),
    ("feed IC 1", _conv(1, 64, k=7, s=2, n=224, may_feed=True), FEED),
    ("feed IC 3", _conv(3, 64, k=7, s=2, n=224, may_feed=True), FEED),
    ("feed IC 4", _conv(4, 64, k=7, s=2, n=224, may_feed=True), FEED),
    ("feed IC 5: row window only", _conv(5, 64, k=7, s=2, n=224, may_feed=True), ROWWIN),
    ("feed 3x3 stem", _conv(3, 32, k=3, s=2, n=224, may_feed=True), FEED),
    ("feed refused for stride 1", _conv(3, 32, k=3, s=1, n=224, may_feed=True), ROWWIN),
    ("feed refused with residual", _conv(3, 64, k=7, s=2, n=224, may_feed=True, residual=True), SIMT),
    ("feed refused under SIMT", _conv(3, 64, k=7, s=2, n=224, may_feed=True, algo=ALGO_SIMT), SIMT),
    ("input not a model input", _conv(3, 64, k=7, s=2, n=224), ROWWIN),
    ("row-window operand packed for another pad", _conv(3, 32, row=(1, 0)), SIMT),
    ("row-window operand packed for another stride", _conv(3, 32, s=2, row=(1, 1)), SIMT),
    ("no row-window operand", _conv(3, 32, row=(0, 0)), SIMT),
    ("feed operand packed for another pad", _conv(3, 64, k=7, s=2, n=224, may_feed=True, feed_pad=2), ROWWIN),
    ("no feed operand", _conv(3, 64, k=7, s=2, n=224, may_feed=True, feed_pad=-1), ROWWIN),
]


@pytest.mark.parametrize("desc,case,path", LIMITS, ids=[c[0] for c in LIMITS])
def test_decision_table(desc, case, path):
    in_hwc, out_hwc, k, s, px, py, kw = case
    got = plan(in_hwc, out_hwc, k, s, px, py, **kw)
    assert got["path"] == path, (desc, got)
    assert got == reference_plan(in_hwc, out_hwc, k, s, px, py, **kw), desc


def test_plan_carries_what_the_kernel_sees():
    # ResNet-18's 7x7 stem on a 224x224 model input: the feed copy's geometry (MixedInferenceCore::init before the planner)
    got = plan((224, 224, 3), (112, 112, 64), 7, 2, 3, 3, may_feed=True)
    assert got == {"path": FEED, "pad_x": 3, "pad_y": 3, "pad_mode": PAD_CONSTANT, "prepad_h": 0, "prepad_w": 0, "feed_h": 229, "feed_w": 262,
                   "feed_py": 3, "feed_px": 4}
    # Candy's reflect-padded 9x9 stem: the row-window kernel reads a 728x728 pre-padded copy with zero padding
    got = plan((720, 720, 3), (720, 720, 32), 9, 1, 4, 4, pad_mode=PAD_REFLECT)
    assert (got["path"], got["pad_x"], got["pad_y"], got["pad_mode"], got["prepad_h"], got["prepad_w"]) == (ROWWIN, 0, 0, PAD_CONSTANT, 728, 728)


def _model_convs(name):
    """(input hwc, output hwc, k, stride, pad_x, pad_y, pad mode, reads a model input) of every Conv2D of a BASELINE model at its bench size."""
    fn, hw, _, _ = modelzoo.MODELS[name]
    layers = fn(hw)
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
        mode = {"constant": PAD_CONSTANT, "reflect": PAD_REFLECT, "replicate": PAD_REPLICATE}[l.get("mode", "constant")] if "mode" in l else PAD_NONE
        pin, pout = np.shape(outs[src]), np.shape(outs[i])  # NHWC
        convs.append((pin[1:], pout[1:], k, s, 0 if k == 1 else o[0], 0 if k == 1 else o[2], mode,
                      layers[src]["type"] == "InputLayer"))
    return convs


@pytest.mark.parametrize("name", ["resnet18", "mobilenetv2", "yolov3tiny", "candy", "espcn"])
def test_every_baseline_convolution(name):
    pytest.importorskip("torch")
    convs = _model_convs(name)
    assert convs
    seen = set()
    for in_hwc, out_hwc, k, s, px, py, mode, from_input in convs:
        for algo in (AUTO, ALGO_SIMT, TCGEN05):
            kw = dict(pad_mode=mode, algo=algo, may_feed=from_input)
            got = plan(in_hwc, out_hwc, k, s, px, py, **kw)
            assert got == reference_plan(in_hwc, out_hwc, k, s, px, py, **kw), (name, in_hwc, out_hwc, k, s, algo)
            if algo == AUTO:
                seen.add(got["path"])
    # the tensor-core paths the unfused models exercise under AUTO (MobileNetV2 reads its input through a ZeroPadding2D layer)
    assert seen == {"resnet18": {FEED, IGEMM}, "mobilenetv2": {ROWWIN, IGEMM}, "yolov3tiny": {ROWWIN, IGEMM}, "candy": {ROWWIN, IGEMM},
                    "espcn": {ROWWIN, IGEMM}}[name], seen


@pytest.mark.gpu
@pytest.mark.parametrize("workload", ["candy", "espcn", "mobilenetv2", "resnet18", "yolov3tiny"])
def test_engine_runs_the_recorded_plan(ctx, tmp_path, workload):
    # tests/golden/conv_plan_golden.json (generator beside it) holds, for every fuse / algo / precision configuration, the kernel of every
    # layer, the weight arena's size and the launches per forward pass as the engine ran them before the planner existed
    import json
    import os
    import sys
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    sys.path.insert(0, golden)
    from make_plan_golden import record
    want = json.load(open(os.path.join(golden, "conv_plan_golden.json")))[workload]
    got = record(ctx, workload, str(tmp_path))
    assert sorted(got) == sorted(want)
    for cfg in want:
        assert got[cfg]["arena_bytes"] == want[cfg]["arena_bytes"], cfg
        assert got[cfg]["launches"] == want[cfg]["launches"], cfg
        assert got[cfg]["kernels"] == want[cfg]["kernels"], cfg
