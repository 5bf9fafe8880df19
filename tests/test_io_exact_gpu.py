"""The model's input and output transfers held to oracle/exact.py's float64 restatements: the resize and normalisation of 8-bit images
(resize_u8_kernel, and frame_input_kernel on RGBA8 and NV12 frames), the plain uploads (split_kernel, split_u8_kernel and the
device-buffer inputs in both layouts), the stem's feed copy, the downloads (merge_kernel, merge_u8_kernel, the device-buffer
outputs) with their 8-bit quantisation, and the arg-max of the classes (argmax_kernel, result_small_kernel).

The input side is observed through layer_output(0), the stored model input, of one-layer models; the output side through models whose
one layer only moves data (a zero pad, or a Flatten for the classifiers), whose output is therefore the stored input, so every output
kernel has a reference computed from the host-side input alone. Each case asserts from snnb_debug_launches which instantiation ran.
Every case runs in the three precisions. The test prints the worst |err| / bound of every instantiation and fails if one of COVERED
was never launched (test_io_exact_cpu.py holds COVERED to the library's kernels). Data moves and quantised bytes must match exactly.
"""
import ctypes as C
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
SMALL_RESULT_BYTES = 64 * 1024  # MixedInferenceCore::SMALL_RESULT_BYTES (engine.h)

COVERED = ["resize_u8_kernel", "frame_input_kernel<rgba8, batch>", "frame_input_kernel<nv12, batch>", "split_kernel", "split_u8_kernel",
           "device_input_kernel<f32>", "device_input_kernel<f16>", "device_input_kernel<u8>", "device_input_nchw_tiled_kernel<f32>",
           "device_input_nchw_tiled_kernel<f16>", "device_input_nchw_tiled_kernel<u8>", "merge_kernel", "merge_u8_kernel",
           "device_output_kernel<f32>", "device_output_kernel<f16>", "device_output_kernel<u8>", "argmax_kernel", "result_small_kernel"]
SEEN = {}  # instantiation -> (case, worst |err| / bound), over the whole module
MEAN4, NORM4 = [10.0, 100.5, 30.25, 200.0], [0.0125, 0.5, 2.0, 1.0 / 3.0]  # per channel, none exact in both


def record(kernel, why, ratio):
    if SEEN.get(kernel, (None, -1.0))[1] < ratio:
        SEEN[kernel] = (why, ratio)


def hold(got, ref, bound, kernel, why):
    ratio, bad = exact.check(got, ref, bound, kernel)
    if bad:
        err = np.abs(np.asarray(got, np.float64) - ref)
        k = np.unravel_index(np.argmax(np.where(err <= bound, 0, np.where(np.isnan(err), np.inf, err) / np.maximum(bound, 1e-300))), err.shape)
        raise AssertionError("%s (%s): %d of %d elements outside the bound, worst |err|/bound %.3g; at %s got %r ref %r bound %.3g" % (
            why, kernel, bad, err.size, ratio, k, float(np.asarray(got)[k]), float(ref[k]), float(bound[k])))
    record(kernel, why, ratio)


def torch():
    import torch as t
    return t


def cuda(a):
    return torch().from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch().cuda.synchronize()
    return t.cpu().numpy()


def launched(ctx):
    return ctx.debug_launches(clear=True)


def expect_first(ctx, kernel, why):
    names = launched(ctx)
    assert names and names[0] == kernel, (why, kernel, names)


def load(ctx, tmp, build, batch, precision, tag):
    b = modelzoo.Builder(11)
    build(b)
    path = os.path.join(tmp, "%s_%s.json" % (tag, precision))
    modelzoo.write_model(b.layers, path, split=True)
    return core.MixedInferenceCore(ctx, path, batch=batch, precision=precision), path


def padded(h, w, c):
    """Input -> zero pad by one pixel on every side: the output is the stored input, bordered with zeros."""
    return lambda b: b.pad(b.input(w, h, c), 1, 1, 1, 1)


def stem(h, w, c=3):
    """The ResNet-18 stem (7 x 7, stride 2, 64 channels, 'same'): its input's only reader is the feed-mode convolution, so the input is
    feed-only (the compact 4-channel copy, no regular planes)."""
    return lambda b: b.conv(b.input(w, h, c), 64, 7, 2, "same", "relu", bias=True)


def u8_images(rng, shape):
    return rng.integers(0, 256, shape, dtype=np.uint8)  # noise: a tap one texel off moves a value by ~85 on average


def u8_normalised(img, half):
    """(x - mean[c & 3]) * norm[c & 3] in fp32 (two roundings, exactly what the kernels compute) and its store: the restatement of an
    equal-size 8-bit input that the convolution restatement below is fed."""
    c = img.shape[-1]
    mean = np.array([MEAN4[i & 3] for i in range(c)], np.float32)
    norm = np.array([NORM4[i & 3] for i in range(c)], np.float32)
    return exact.stored((img.astype(np.float32) - mean) * norm, half).astype(np.float64)


def wide_f32(rng, shape):
    """fp32 inputs over fp16's whole range and past it: unit noise, values past 65504 and past 131008 (saturated), fp16 subnormals."""
    x = rng.uniform(-1, 1, shape)
    sel = rng.integers(0, 5, shape)
    x = np.where(sel == 1, x * 1e5, x)
    x = np.where(sel == 2, x * 1e6, x)
    x = np.where(sel == 3, x * 1e-6, x)
    return x.astype(np.float32)


def wide_f16(rng, shape):
    x = rng.uniform(-1, 1, shape)
    sel = rng.integers(0, 4, shape)
    x = np.where(sel == 1, x * 6e4, x)
    x = np.where(sel == 2, x * 1e-6, x)  # subnormal in fp16
    return x.astype(np.float16)


# ---- the input side ----------------------------------------------------------------------------------------------------------
def check_stem_conv(m, path, x_stored, precision, why):
    """The feed-mode convolution's output against exact.conv2d fed the host-side stored input: a feed written at the wrong offset, or
    a halo left non-zero, breaks it."""
    import test_layer_exact_gpu as tl
    om = oracle.Model(path)
    shapes = [m.layer_info(i)[2] for i in range(m.num_layers)]
    m.time_layers()  # one more pass on the same input: it records each layer's kernel
    kname = m.layer_kernel(1)
    assert kname == "conv_rowwin_kernel<feed>", (why, kname)
    got = m.layer_output(1)
    ref, bound = tl.restate(om, 1, [x_stored, None], {"names": ["", kname], "shapes": shapes}, precision, precision == "fp16", None)
    ratio, bad = exact.check(got, ref, bound, "conv")
    assert bad == 0, (why, "stem convolution", bad, ratio)


def hold_resize(got, img, out_hw, linear, half, kernel, why):
    """The resized model input within exact.resize_u8's bound; nearest: also bit-identical to one of the candidate taps' values."""
    hold(got, *exact.resize_u8(img, out_hw, MEAN4, NORM4, linear, half), kernel, why)
    if not linear:
        c = img.shape[-1]
        cands = exact.nearest_candidates(img, out_hw, [MEAN4[i & 3] for i in range(c)], [NORM4[i & 3] for i in range(c)], half)
        assert np.any([got == v for v in cands], axis=0).all(), (why, "a nearest value that is none of its candidate taps")


# (model input h, w, c; source h, w; batch; feed-only stem)
RESIZE = [((64, 80, 3), (150, 233), 2, False),  # downscale in y, mixed
          ((64, 80, 3), (40, 50), 2, False),    # upscale
          ((32, 48, 4), (64, 96), 2, False),    # exact 2x down: nearest positions fall on integers
          ((30, 33, 1), (90, 99), 2, False),    # exact 3x down: linear positions fall on integers
          ((40, 60, 3), (20, 30), 2, False),    # exact 2x up
          ((24, 36, 20), (8, 12), 2, False),    # exact 3x up; C = 20: mean and norm cycle, a tail channel group
          ((16, 24, 3), (1, 57), 2, False),     # 1 x N
          ((16, 24, 4), (45, 1), 2, False),     # N x 1
          ((16, 24, 3), (1, 1), 3, False),      # 1 x 1
          ((24, 40, 3), (2160, 3840), 1, False),  # coarse fp32 positions
          ((37, 53, 3), (120, 77), 2, True),    # feed-only stem input
          ((37, 53, 3), (20, 31), 2, True)]


@pytest.mark.parametrize("precision", FORMS)
def test_resize_u8(ctx, tmp_path, precision):
    half = precision == "fp16"
    for idx, ((h, w, c), (sh, sw), n, feed) in enumerate(RESIZE):
        m, _ = load(ctx, str(tmp_path), stem(h, w, c) if feed else padded(h, w, c), n, precision, "resize%d" % idx)
        try:
            for linear in (True, False):
                why = "resize %dx%d -> %dx%dx%d n%d %s%s %s" % (sh, sw, h, w, c, n, "linear" if linear else "nearest", " feed" if feed else "", precision)
                img = u8_images(np.random.default_rng(100 + idx + 50 * linear), (n, sh, sw, c))
                launched(ctx)
                m.run_image(img, MEAN4, NORM4, linear=linear)
                expect_first(ctx, "resize_u8_kernel", why)
                hold_resize(m.layer_output(0), img, (h, w), linear, half, "resize_u8_kernel", why)
        finally:
            m.close()


# (model input h, w, c; frame h, w; feed-only stem)
FRAMES = [((36, 52, 3), (96, 80), False), ((36, 52, 4), (30, 40), False), ((33, 47, 3), (96, 80), True)]


@pytest.mark.parametrize("precision", FORMS)
def test_frame_input(ctx, tmp_path, precision):
    """frame_input_kernel on RGBA8 and NV12, held to the same restatement as resize_u8_kernel: NV12 through oracle/yuv.py's libyuv
    RGBA (integer-exact), which anchors the 8-bit frame chain on its own."""
    from test_frames_gpu import expected_rgba, packed, random_yuv
    half = precision == "fp16"
    for idx, ((h, w, c), (fh, fw), feed) in enumerate(FRAMES):
        m, _ = load(ctx, str(tmp_path), stem(h, w, c) if feed else padded(h, w, c), 2, precision, "frames%d" % idx)
        try:
            for fmt in ("rgba8", "nv12"):
                for linear in (True, False):
                    why = "frames %s %dx%d -> %dx%dx%d %s%s %s" % (fmt, fh, fw, h, w, c, "linear" if linear else "nearest", " feed" if feed else "", precision)
                    y, u, v = random_yuv(2, fh, fw, seed=7 + idx)
                    rgba = expected_rgba("nv12", y, u, v, "bt601")
                    rgba[..., 3] = u8_images(np.random.default_rng(idx), rgba.shape[:3])  # a noisy alpha for the 4-channel model
                    if fmt == "nv12":
                        rgba[..., 3] = 255
                    frames = cuda(rgba) if fmt == "rgba8" else packed("nv12", y, u, v)
                    launched(ctx)
                    m.run_frames(frames, format=fmt, linear=linear, mean4=MEAN4, norm4=NORM4)
                    kern = "frame_input_kernel<%s, batch>" % fmt
                    expect_first(ctx, kern, why)
                    torch().cuda.synchronize()
                    hold_resize(m.layer_output(0), rgba[..., :c], (h, w), linear, half, kern, why)
        finally:
            m.close()


# (n, h, w, c): H x W below 32 and not a multiple of 32, channel counts around the 64-channel tile
DIRECT = [(2, 5, 6, 3), (2, 7, 9, 8), (3, 5, 6, 9), (2, 7, 9, 63), (2, 5, 6, 64), (3, 7, 9, 65), (2, 7, 9, 130)]


def device_kernel(layout, dtype, c, feed):
    tiled = layout == "nchw" and c > 8 and not feed
    return "device_input_%s<%s>" % ("nchw_tiled_kernel" if tiled else "kernel", dtype)


def direct_drivers(m, rng, shape, half, wide):
    """(name, call, expected kernel, host-side stored input) of every equal-size input path, each with its own images. wide: fp32 and
    fp16 inputs over and past fp16's range (else unit noise, for the stem, whose convolution restatement does not model saturation)."""
    n, h, w, c = shape
    nchw = lambda a: np.ascontiguousarray(a.transpose(0, 3, 1, 2))  # noqa: E731
    wide_f32_ = wide_f32 if wide else (lambda rng, shape: rng.uniform(-1, 1, shape).astype(np.float32))  # noqa: E731
    wide_f16_ = wide_f16 if wide else (lambda rng, shape: rng.uniform(-1, 1, shape).astype(np.float16))  # noqa: E731
    x = wide_f32_(rng, shape)
    yield "set_input f32", lambda: m.set_input(x), "split_kernel", exact.model_input(x, half)[0]
    u8 = u8_images(rng, shape)
    yield "run_u8", lambda: m.run_u8(u8, MEAN4, NORM4, want_classes=False), "split_u8_kernel", u8_normalised(u8, half)
    for layout in ("nhwc", "nchw"):
        lay = (lambda a: a) if layout == "nhwc" else nchw
        x = wide_f32_(rng, shape)
        yield "run_torch f32 " + layout, lambda x=x, lay=lay, layout=layout: m.run_torch(cuda(lay(x)), layout=layout), "f32", exact.model_input(x, half)[0]
        x16 = wide_f16_(rng, shape)
        yield ("run_torch f16 " + layout, lambda x16=x16, lay=lay, layout=layout: m.run_torch(cuda(lay(x16)), layout=layout), "f16",
               exact.model_input(x16.astype(np.float32), half)[0])
        u8 = u8_images(rng, shape)
        yield ("run_torch u8 " + layout, lambda u8=u8, lay=lay, layout=layout: m.run_torch(cuda(lay(u8)), layout=layout, mean4=MEAN4, norm4=NORM4), "u8",
               u8_normalised(u8, half))


@pytest.mark.parametrize("precision", FORMS)
def test_direct_inputs(ctx, tmp_path, precision):
    """split_kernel, split_u8_kernel, device_input_kernel and device_input_nchw_tiled_kernel: bit-identical to the stored host-side input.
    The 8-bit paths are also held to resize_u8 at equal size (direct sampling), whose normalisation is stated in float64."""
    half = precision == "fp16"
    for idx, shape in enumerate(DIRECT + [(2, 37, 53, 3, "feed")]):
        feed = len(shape) == 5
        n, h, w, c = shape[:4]
        m, path = load(ctx, str(tmp_path), stem(h, w, c) if feed else padded(h, w, c), n, precision, "direct%d" % idx)
        try:
            for name, call, kern, want in direct_drivers(m, np.random.default_rng(200 + idx), (n, h, w, c), half, not feed):
                layout = name.split()[-1]
                if kern in ("f32", "f16", "u8"):
                    kern = device_kernel(layout, kern, c, feed)
                why = "%s n%d %dx%dx%d%s %s" % (name, n, h, w, c, " feed" if feed else "", precision)
                launched(ctx)
                call()
                expect_first(ctx, kern, why)
                torch().cuda.synchronize()
                got = m.layer_output(0)  # feed-only: merge_kernel's load_feed branch
                hold(got, want, np.zeros(want.shape), kern, why)
                if feed:
                    if name == "set_input f32":
                        m.forward()
                    ctx.sync()
                    check_stem_conv(m, path, want, precision, why)
        finally:
            m.close()


@pytest.mark.parametrize("precision", FORMS)
def test_u8_direct_normalisation_matches_the_float64_statement(ctx, tmp_path, precision):
    """split_u8_kernel and device_input_kernel<u8> at equal size are resize_u8's direct sampling: held to the float64 statement too."""
    half = precision == "fp16"
    n, h, w, c = 2, 7, 9, 20
    m, _ = load(ctx, str(tmp_path), padded(h, w, c), n, precision, "u8direct")
    try:
        u8 = u8_images(np.random.default_rng(5), (n, h, w, c))
        ref, bound = exact.resize_u8(u8, (h, w), MEAN4, NORM4, True, half)
        m.run_u8(u8, MEAN4, NORM4, want_classes=False)
        hold(m.layer_output(0), ref, bound, "split_u8_kernel", "run_u8 as resize_u8 %s" % precision)
        m.run_torch(cuda(u8), mean4=MEAN4, norm4=NORM4)
        torch().cuda.synchronize()
        hold(m.layer_output(0), ref, bound, "device_input_kernel<u8>", "run_torch u8 as resize_u8 %s" % precision)
    finally:
        m.close()


# ---- the output side ---------------------------------------------------------------------------------------------------------
def straddling(rng, shape, scale, offset):
    """fp32 values whose v * scale + offset straddle half-integers from -20 to 280 (just below, on, just above), a share far outside
    [0, 255], and values around 65504 .. 65520, where __float2half_rn overflows to infinity."""
    k = rng.integers(-20, 281, shape) + 0.5
    v = (k - offset) / scale + rng.choice([-1e-3, -1e-5, 0.0, 1e-5, 1e-3], shape)
    sel = rng.integers(0, 6, shape)
    v = np.where(sel == 1, rng.uniform(-1e4, 1e4, shape), v)
    v = np.where(sel == 2, rng.uniform(65500, 65530, shape) * rng.choice([-1, 1], shape), v)
    return v.astype(np.float32)


OUT_SHAPES = [(2, 5, 6, 3), (2, 7, 9, 20), (3, 4, 5, 65)]
QUANT = [(0.7, 12.0), (2.0, 0.5), (2.0, -100.0)]  # scale 0.7 is not exact in fp32, scale 2 is


@pytest.mark.parametrize("precision", FORMS)
def test_outputs(ctx, tmp_path, precision):
    """merge_kernel, device_output_kernel<f32 | f16 | u8> in NHWC and NCHW, and merge_u8_kernel (submit_image's 8-bit output)."""
    half = precision == "fp16"
    for idx, (n, h, w, c) in enumerate(OUT_SHAPES):
        m, _ = load(ctx, str(tmp_path), padded(h, w, c), n, precision, "out%d" % idx)
        rng = np.random.default_rng(300 + idx)
        try:
            for scale, offset in QUANT:
                x = straddling(rng, (n, h, w, c), scale, offset)
                if scale == 2.0:  # every other image: exact .5 ties of v * 2 + offset
                    x[::2] = ((np.floor(x[::2] * 2 + offset) + 0.5 - offset) / 2).astype(np.float32)
                stored = np.pad(exact.stored(x, half), ((0, 0), (1, 1), (1, 1), (0, 0)))
                why = "out n%d %dx%dx%d scale %g offset %g %s" % (n, h, w, c, scale, offset, precision)
                launched(ctx)
                got, _ = m.run(x, want_classes=False)
                assert "merge_kernel" in launched(ctx), why
                hold(got, stored.astype(np.float64), np.zeros(stored.shape), "merge_kernel", why)
                q_ref, q_bound = exact.quant_u8(stored, scale, offset)
                for layout in ("nhwc", "nchw"):
                    tr = (lambda a: a) if layout == "nhwc" else (lambda a: a.transpose(0, 3, 1, 2))
                    for dt, name in ((torch().float32, "f32"), (torch().float16, "f16"), (torch().uint8, "u8")):
                        kern = "device_output_kernel<%s>" % name
                        launched(ctx)
                        out = host(m.run_torch(cuda(x), out_dtype=dt, out_layout=layout, out_scale=scale, out_offset=offset))
                        assert kern in launched(ctx), (why, kern)
                        if name == "f32":
                            hold(out, tr(stored).astype(np.float64), np.zeros(out.shape), kern, why + " " + layout)
                        elif name == "f16":
                            with np.errstate(over="ignore"):
                                want = tr(stored).astype(np.float16)
                            assert np.array_equal(out.view(np.uint16), want.view(np.uint16)), (why, layout, "f16 output")
                            assert half or np.isinf(want).any(), "no value rounds past 65504"
                            record(kern, why, 0.0)
                        else:
                            hold(out.astype(np.float64), tr(q_ref), tr(q_bound), kern, why + " " + layout)
            # 8-bit images in (split_u8_kernel), 8-bit images out (merge_u8_kernel); norm 0.37 puts the values between integers
            u8 = u8_images(rng, (n, h, w, c))
            for scale, offset in QUANT:
                mean4, norm4 = [3.0, 0.0, 100.0, 7.5], [0.37, 2.0, 1.25, -3.0]
                launched(ctx)
                got, _ = m.run_image(u8, mean4, norm4, out_u8=True, out_scale=scale, out_offset=offset)
                assert "merge_u8_kernel" in launched(ctx)
                mean = np.array([mean4[i & 3] for i in range(c)], np.float32)
                norm = np.array([norm4[i & 3] for i in range(c)], np.float32)
                stored = np.pad(exact.stored((u8.astype(np.float32) - mean) * norm, half), ((0, 0), (1, 1), (1, 1), (0, 0)))
                q_ref, q_bound = exact.quant_u8(stored, scale, offset)
                hold(got.astype(np.float64), q_ref, q_bound, "merge_u8_kernel", "run_image u8 out n%d %dx%dx%d scale %g offset %g %s" % (n, h, w, c, scale, offset, precision))
        finally:
            m.close()


# ---- the arg-max -------------------------------------------------------------------------------------------------------------
def scores(rng, n, c, kinds):
    """n images of c scores, image i of kind kinds[i % len(kinds)]."""
    x = rng.uniform(-5, 5, (n, c)).astype(np.float32)
    for i in range(n):
        kind = kinds[i % len(kinds)]
        top = float(np.abs(x[i]).max()) + 1
        j = int(rng.integers(0, c))
        if kind == "tie32" and c > 32:
            j = int(rng.integers(0, c - 32))
            x[i, j] = x[i, j + 32] = top
        elif kind == "tie1":
            j = int(rng.integers(0, c - 1))
            x[i, j] = x[i, j + 1] = top
        elif kind == "last":
            x[i, -1] = top
        elif kind == "equal":
            x[i] = 0.75
        elif kind == "nan0":
            x[i, 0] = np.nan
            x[i, j] = top
        elif kind == "nan_later":
            x[i, j] = np.nan
            x[i, (j + 1) % c] = top
            x[i, rng.integers(0, c, 3)] = np.nan
        elif kind == "nan_all":
            x[i] = np.nan
    return x


def classifier(c):
    return lambda b: b.flatten(b.input(1, 1, c), c)


def classes_of(ctx, m, x, via):
    """1-based classes of images x through one entry point, with the instantiations it launched and the values it returned."""
    n, c = x.shape
    launched(ctx)
    if via == "run":
        vals, cls = m.run(x.reshape(n, 1, 1, c))
    elif via == "submit":
        vals = np.empty((n, 1, 1, c), np.float32)
        cls_buf = (C.c_int * n)()
        t = m.submit_raw(np.ascontiguousarray(x).ctypes.data, vals.ctypes.data, vals.size, C.cast(cls_buf, C.c_void_p))
        m.wait(t)
        cls = np.array(list(cls_buf), np.int32)
    elif via == "torch":
        vals, cls = m.run_torch(cuda(x.reshape(n, 1, 1, c)), want_classes=True)
        vals, cls = host(vals), host(cls)
    return np.asarray(cls), vals, launched(ctx)


def hold_classes(ctx, m, x, via, half, why):
    cls, vals, names = classes_of(ctx, m, x, via)
    n, c = x.shape
    small = via == "submit" and vals.size * 4 + n * 4 <= SMALL_RESULT_BYTES and not os.environ.get("SNNB_NO_SMALL_RESULT")
    kern = "result_small_kernel" if small else "argmax_kernel"
    assert kern in names, (why, via, names)
    st = exact.stored(x, half)
    want, _ = exact.argmax(st)
    bad = np.nonzero(cls - 1 != want)[0]
    assert bad.size == 0, "%s via %s (%s): %d of %d classes differ; image %d: got %d, want %d" % (
        why, via, kern, bad.size, n, bad[0] if bad.size else -1, cls[bad[0]] if bad.size else 0, want[bad[0]] + 1 if bad.size else 0)
    assert np.array_equal(vals.reshape(n, c).view(np.uint32)[~np.isnan(st)], st.view(np.uint32)[~np.isnan(st)]) and np.isnan(vals.reshape(n, c)[np.isnan(st)]).all()
    record(kern, why + " via " + via, 0.0)
    return kern


ARGMAX_KINDS = ["random", "tie32", "tie1", "last", "equal"]


@pytest.mark.parametrize("precision", FORMS)
@pytest.mark.parametrize("c", [2, 31, 32, 33, 1000, 1001])
def test_argmax(ctx, tmp_path, c, precision):
    """argmax_kernel (snnb_argmax1, run, run_torch's device classes at base 1) and result_small_kernel (submit's mapped result), at
    batches of 5 and 130 (several warps per block, several blocks): ties between channels c and c + 32 (one lane) and c + 1, the
    maximum at the last channel, all-equal scores."""
    half = precision == "fp16"
    for n in (5, 130):
        m, _ = load(ctx, str(tmp_path), classifier(c), n, precision, "argmax%d_%d" % (c, n))
        try:
            x = scores(np.random.default_rng(c * 1000 + n), n, c, ARGMAX_KINDS)
            for via in ("run", "torch", "submit"):
                hold_classes(ctx, m, x, via, half, "argmax n%d c%d %s" % (n, c, precision))
        finally:
            m.close()
    if precision == "fp32x3":
        x = scores(np.random.default_rng(c), 130, c, ARGMAX_KINDS)
        got = core.argmax1(ctx, x.reshape(130, 1, 1, c))
        assert np.array_equal(got - 1, exact.argmax(exact.stored(x, False))[0]), c


@pytest.mark.parametrize("kind", ["nan0", "nan_later", "nan_all"])
@pytest.mark.parametrize("c", [2, 33, 1000])
def test_argmax_nan_scores(ctx, tmp_path, c, kind):
    """NaN scores (overflowed fp16 logits, a NaN input): std::max_element's index, 0 for an all-NaN image, through every path."""
    for precision in FORMS:
        m, _ = load(ctx, str(tmp_path), classifier(c), 5, precision, "nan%d_%s" % (c, kind))
        try:
            x = scores(np.random.default_rng(c + len(kind)), 5, c, [kind, "random"])
            for via in ("run", "torch", "submit"):
                hold_classes(ctx, m, x, via, precision == "fp16", "argmax %s c%d %s" % (kind, c, precision))
        finally:
            m.close()
    x = scores(np.random.default_rng(c), 5, c, [kind])
    assert np.array_equal(core.argmax1(ctx, x.reshape(5, 1, 1, c)) - 1, exact.argmax(exact.stored(x, False))[0]), (c, kind)


def small_result_cases(ctx, tmp):
    """1000 classes at batch 16 fit SMALL_RESULT_BYTES (result_small_kernel), at batch 17 they do not (merge_kernel + argmax_kernel).
    Returns the instantiation each batch launched."""
    kinds = {}
    for n in (16, 17):
        m, _ = load(ctx, tmp, classifier(1000), n, "fp32x3", "small%d" % n)
        try:
            x = scores(np.random.default_rng(n), n, 1000, ARGMAX_KINDS + ["nan0", "nan_later", "nan_all"])
            kinds[n] = hold_classes(ctx, m, x, "submit", False, "submit n%d c1000" % n)
        finally:
            m.close()
    return kinds


def test_small_result_threshold(ctx, tmp_path):
    assert small_result_cases(ctx, str(tmp_path)) == {16: "result_small_kernel", 17: "argmax_kernel"}


def child_main():
    """SNNB_NO_SMALL_RESULT=1 child (the variable is read once into a static): both batches take merge_kernel + argmax_kernel."""
    import tempfile
    ctx = core.GpuContext(0)
    with tempfile.TemporaryDirectory() as tmp:
        kinds = small_result_cases(ctx, tmp)
    ctx.close()
    print("KINDS " + json.dumps(kinds))


def test_small_result_switched_off(ctx):
    env = dict(os.environ, SNNB_NO_SMALL_RESULT="1")
    code = "import sys; sys.path[:0] = [%r, %r]; import test_io_exact_gpu as t; t.child_main()" % (HERE, os.path.dirname(HERE))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("KINDS ")][-1]
    assert json.loads(line[6:]) == {"16": "argmax_kernel", "17": "argmax_kernel"}


def test_every_transfer_kernel_was_launched():
    """Runs last: the worst |err| / bound of every instantiation over this module's cases."""
    for key in COVERED:
        print("%-40s %s" % (key, "worst |err|/bound %.3g (%s)" % (SEEN[key][1], SEEN[key][0]) if key in SEEN else "NOT LAUNCHED"))
    missing = [k for k in COVERED if k not in SEEN]
    assert not missing, missing
