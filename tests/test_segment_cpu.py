"""snnb_model_segment_frames without a GPU: the entry point is exported and refuses a null model, the numpy restatement of its label
plane (oracle/seg.py), which the GPU tests hold the kernel to, gives the values worked out by hand below, and the U-Net of the model zoo
is a graph worth segmenting with: the oracle agrees with torch on every layer, activations stay O(1), the calibrated heads give mixed
labels, and its convolutions are planned onto the tensor-core kernels."""
import ctypes as C

import numpy as np
import pytest

from oracle import seg
from shadernn_b200 import _lib

NAN, INF = np.float32(np.nan), np.float32(np.inf)


def test_segment_frames_is_exported_and_refuses_a_null_model(built):
    lib = _lib.lib()
    assert "snnb_model_segment_frames" in _lib.SIGNATURES
    f, o = _lib.Frames(), _lib.LabelsOut()
    assert lib.snnb_model_segment_frames(None, None, 0, None, None) != 0
    assert b"snnb_model_segment_frames: null model" in lib.snnb_last_error()
    assert lib.snnb_model_segment_frames(None, C.byref(f), 1, C.byref(o), None) != 0
    assert b"snnb_model_segment_frames: null model" in lib.snnb_last_error()


def t4(a):
    """[h][w][C] nested lists -> [1, h, w, C] float32"""
    return np.array(a, np.float32)[None]


def test_equal_size_is_the_per_pixel_argmax():
    rng = np.random.default_rng(0)
    t = rng.standard_normal((3, 5, 7, 21)).astype(np.float32)
    for linear in (True, False):
        assert np.array_equal(seg.scores(t, (5, 7), linear), t)
        assert np.array_equal(seg.segment(t, (5, 7), linear), t.argmax(-1).astype(np.uint8))


def test_nearest_is_the_argmax_at_model_size_then_a_nearest_resize():
    rng = np.random.default_rng(1)
    t = rng.standard_normal((2, 4, 6, 5)).astype(np.float32)
    small = t.argmax(-1).astype(np.uint8)
    # 2x: output pixel o samples (o + 0.5) / 2, i.e. source o // 2
    assert np.array_equal(seg.segment(t, (8, 12), linear=False), np.repeat(np.repeat(small, 2, 1), 2, 2))
    # 3 x 5 from 4 x 6: rows (0.5, 1.5, 2.5) * 4 / 3 -> 0, 2, 3; columns (o + 0.5) * 6 / 5 -> 0, 1, 3, 4, 5
    assert np.array_equal(seg.segment(t, (3, 5), linear=False), small[:, [0, 2, 3]][:, :, [0, 1, 3, 4, 5]])


def test_linear_blends_the_scores_before_the_argmax():
    # 1 x 2 -> 1 x 4: x = -0.25, 0.25, 0.75, 1.25 -> weights of the right texel 0 (clamped), 0.25, 0.75, 1 (clamped)
    t = t4([[[1.0, 0.0], [0.0, 1.0]]])
    s = seg.scores(t, (1, 4), True)[0, 0]
    assert np.array_equal(s, np.array([[1.0, 0.0], [0.75, 0.25], [0.25, 0.75], [0.0, 1.0]], np.float32))
    assert seg.segment(t, (1, 4), True).tolist() == [[[0, 0, 1, 1]]]
    # the arg-max of blended scores is not a blend of labels: channel 2 wins nowhere at the taps but wins in between
    t = t4([[[1.0, 0.0, 0.9], [0.0, 1.0, 0.9]]])
    assert seg.segment(t, (1, 4), True).tolist() == [[[0, 2, 2, 1]]]


def test_linear_2x2_to_1x1_blends_the_four_taps():
    # 2 x 2 -> 1 x 1: the source position 0.5 on both axes, weights 0.5. Channel 0: top 2, bottom 2 + 0.5 (0 - 2) = 1, 1.5; channel 1:
    # top 0, bottom 2, 1. Nearest takes texel (1, 1) alone.
    t = t4([[[2.0, 0.0], [2.0, 0.0]], [[2.0, 0.0], [0.0, 4.0]]])
    assert np.array_equal(seg.scores(t, (1, 1), True)[0, 0, 0], np.array([1.5, 1.0], np.float32))
    assert seg.segment(t, (1, 1), True).tolist() == [[[0]]]
    assert seg.scores(t, (1, 1), False)[0, 0, 0].tolist() == [0.0, 4.0]
    assert seg.segment(t, (1, 1), False).tolist() == [[[1]]]


def test_ties_go_to_the_lowest_channel():
    t = t4([[[1.0, 3.0, 3.0, 2.0], [5.0, 5.0, 5.0, 5.0], [-INF, -INF, -INF, -INF], [0.0, -0.0, 0.0, 0.0]]])
    assert seg.segment(t, (1, 4)).tolist() == [[[1, 0, 0, 0]]]
    t = t4([[[-0.0, 0.0]]])  # -0 == +0
    assert seg.segment(t, (1, 1)).tolist() == [[[0]]]


def test_nan_scores_never_win_and_all_nan_is_zero():
    t = t4([[[NAN, 1.0, 2.0], [3.0, NAN, 2.0], [NAN, NAN, NAN], [NAN, -INF, NAN], [1.0, 1.0, NAN]]])
    assert seg.segment(t, (1, 5)).tolist() == [[[2, 0, 0, 1, 0]]]
    # a NaN tap makes every blend that reads it NaN (even with weight 0): pixels 1 to 3 are left with channel 1
    t = t4([[[2.0, 1.0], [NAN, 0.0]]])
    assert seg.segment(t, (1, 4), True).tolist() == [[[0, 1, 1, 1]]]


def test_threshold_at_exactly_the_threshold():
    t = t4([[[0.25], [0.5], [np.nextafter(np.float32(0.5), np.float32(0))], [0.75], [NAN], [INF], [-INF]]])
    assert seg.segment(t, (1, 7), threshold=0.5).tolist() == [[[0, 1, 0, 1, 0, 1, 0]]]
    assert seg.segment(t, (1, 7), threshold=0.25).tolist() == [[[1, 1, 1, 1, 0, 1, 0]]]
    # linear threshold of blended scores: 0 and 1 blended to 0.25, 0.75 at 2x
    t = t4([[[0.0], [1.0]]])
    assert seg.segment(t, (1, 4), True, threshold=0.5).tolist() == [[[0, 0, 1, 1]]]
    assert seg.segment(t, (1, 4), True, threshold=0.75).tolist() == [[[0, 0, 1, 1]]]
    assert seg.segment(t, (1, 4), True, threshold=0.7500001).tolist() == [[[0, 0, 0, 1]]]


@pytest.mark.parametrize("hw,out_hw", [((1, 1), (1, 1)), ((1, 1), (5, 3)), ((5, 3), (1, 1)), ((7, 9), (13, 4)), ((16, 16), (1, 31)),
                                       ((3, 5), (1080, 1920)), ((64, 96), (17, 23))])
def test_odd_one_pixel_up_and_down_sizes(hw, out_hw):
    rng = np.random.default_rng(5)
    t = rng.standard_normal((2,) + hw + (3,)).astype(np.float32)
    for linear in (True, False):
        lab = seg.segment(t, out_hw, linear)
        assert lab.shape == (2,) + out_hw and lab.dtype == np.uint8 and lab.max() <= 2
        s = seg.scores(t, out_hw, linear)
        # the corners clamp onto the source's corners when upsampling; nearest only ever takes source values
        if out_hw[0] >= hw[0] and out_hw[1] >= hw[1]:
            assert np.array_equal(s[:, 0, 0], t[:, 0, 0]) and np.array_equal(s[:, -1, -1], t[:, -1, -1])
        if not linear:
            assert np.isin(s, t).all()
    if hw == (1, 1):  # one texel resized to anything is constant
        assert (seg.segment(t, out_hw) == t[:, 0, 0].argmax(-1)[:, None, None]).all()


# ---- U-Net ---------------------------------------------------------------------------------------------------------------------
torch = pytest.importorskip("torch")
from oracle import oracle  # noqa: E402
from shadernn_b200 import modelzoo  # noqa: E402


@pytest.mark.parametrize("classes,hw,batch", [(1, (256, 256), 1), (21, (64, 96), 2)])
def test_unet_oracle_agrees_with_torch_on_every_layer(tmp_path, classes, hw, batch):
    path, layers = modelzoo.build("unet", str(tmp_path), input_hw=hw, classes=classes)
    assert [l["type"] for l in layers].count("Conv2D") == (24 if classes == 1 else 23)
    x = modelzoo.synthetic_input("unet", batch, hw)
    want = oracle.Model(path).run(x, return_all=True)
    got = modelzoo.torch_forward(layers, x)
    assert want[-1].shape == (batch,) + hw + (classes,)
    for i, l in enumerate(layers):
        assert want[i].shape == got[i].shape, (i, l["type"], want[i].shape, got[i].shape)
        scale = float(np.abs(want[i]).max())
        err = float(np.abs(want[i] - got[i]).max())
        assert err <= 5e-5 * max(scale, 1e-6), "layer %d (%s): oracle vs torch %.3g of range %.3g" % (i, l["type"], err, scale)
        if l["type"] == "Conv2D" and i < len(layers) - 1:
            rms = float(np.sqrt(np.mean(want[i].astype(np.float64) ** 2)))
            assert 0.05 < rms < 8.0, "layer %d (%s): activations left O(1): rms %.3g" % (i, l["type"], rms)


def test_unet_calibration_gives_mixed_labels(tmp_path):
    # one class: sigmoid scores on both sides of 0.5 in every image; 21 classes: at least 4 labels in every image
    path, _ = modelzoo.build("unet", str(tmp_path / "k1"), input_hw=(64, 64))
    x = modelzoo.synthetic_input("unet", 3, (64, 64))
    lab = seg.segment(oracle.Model(path).run(x), (64, 64))
    for n in range(3):
        assert 0.05 < float(lab[n].mean()) < 0.95, lab[n].mean()
    path, _ = modelzoo.build("unet", str(tmp_path / "k21"), input_hw=(64, 64), classes=21)
    lab = seg.segment(oracle.Model(path).run(x), (64, 64))
    for n in range(3):
        assert len(np.unique(lab[n])) >= 4, np.unique(lab[n])


IGEMM, ROWWIN, PAD_NONE = 2, 3, 0  # snnb_debug_conv_plan's path codes and SNNB_PAD_NONE


def plan_path(in_hwc, out_hwc, k, pad_x, pad_y, may_feed):
    """snnb_debug_conv_plan of a stride-1 convolution with unnamed ('same' / 'valid') padding under SNNB_ALGO_AUTO, with the weights'
    row-window and feed operands packed for it as the engine packs them: the path."""
    q = [*in_hwc, *out_hwc, k, 1, pad_x, pad_y, PAD_NONE, 0, 0, 1, int(may_feed), 1, pad_x, pad_x]
    out = (C.c_int * 10)()
    assert _lib.lib().snnb_debug_conv_plan((C.c_int * 18)(*q), out) == 0
    return out[0]


def test_unet_convolutions_go_to_the_tensor_cores(built):
    # every convolution with >= 16 input channels (the 2x2 decoder convolutions too) on the implicit GEMM, the 1 -> 64 stem and the
    # 2 -> 1 head on the row window
    layers = modelzoo.unet((256, 256), calibrate=False)
    outs = modelzoo.torch_forward(layers, modelzoo.synthetic_input("unet", 1, (256, 256)))
    paths = []
    for i, l in enumerate(layers):
        if l["type"] != "Conv2D":
            continue
        k = int(l["kernel_size"])
        o = modelzoo._pad4(l, k)
        pin, pout = np.shape(outs[l["inputId"][0]])[1:], np.shape(outs[i])[1:]
        px, py = (0, 0) if k == 1 else (o[0], o[2])
        got = plan_path(pin, pout, k, px, py, layers[l["inputId"][0]]["type"] == "InputLayer")
        assert got == (IGEMM if pin[2] >= 16 else ROWWIN), (i, pin, pout, k, got)
        paths.append((pin[2], k, got))
    assert len(paths) == 24
    assert sum(1 for ic, k, p in paths if k == 2 and p == IGEMM) == 4
    assert [ic for ic, _, p in paths if p == ROWWIN] == [1, 2]
