"""snnb_model_segment_frames (MixedInferenceCore.segment_frames): device frames in, output 0's class scores resampled to a label plane of
any size and reduced to one byte per pixel; every byte exact.

The expected labels are oracle/seg.py (tests/test_segment_cpu.py) applied to the scores the same handle computes for the same input:
the F32 output of run_frames, or for luma input (the Y plane into a 1-channel model) the output of run_image fed the Y planes, which
tests/test_luma_gpu.py holds to be the model input transform_luma feeds."""
import ctypes as C

import numpy as np
import pytest

from oracle import seg
from shadernn_b200 import _lib, core, modelzoo
from shadernn_b200._lib import SnnbError
from test_frames_gpu import expected_rgba, host, laid_out, load, packed, random_yuv, raw_run, set_params
from test_models_gpu import LIMIT, baseline_size_check

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

YUV = ["nv12", "nv21", "i420"]
MEAN, NORM = 16.0, 1.0 / 219.0  # limited-range Y into a model trained on Y / 255
FILL = 0xA5
_paths = {}


def conv_model(ctx, model_dir, in_c, out_c, batch=2, hw=(24, 40), **kw):
    """A small Builder model: one 3x3 convolution from in_c to out_c channels at the input's size; its output is the class scores."""
    key = (in_c, out_c, hw)
    if key not in _paths:
        b = modelzoo.Builder(seed=71 + out_c)
        b.conv(b.input(hw[1], hw[0], in_c), out_c, 3)
        _paths[key] = modelzoo.write_model(b.layers, "%s/seg_%dto%d_%dx%d.json" % (model_dir, in_c, out_c, hw[0], hw[1]))
    return core.MixedInferenceCore(ctx, _paths[key], batch=batch, **kw)


def unet(ctx, model_dir, hw, classes, batch, **kw):
    key = ("unet", hw, classes)
    if key not in _paths:
        _paths[key], _ = modelzoo.build("unet", "%s/seg_unet%d_%dx%d" % (model_dir, classes, hw[0], hw[1]), input_hw=hw, classes=classes)
    return core.MixedInferenceCore(ctx, _paths[key], batch=batch, input_hw=hw, **kw)


def labels_out(n, h, w, pitch=None, gap=0, linear=True, threshold=0.5):
    """A label plane for n images of h x w in one device buffer filled with FILL: rows `pitch` bytes apart, `gap` spare bytes after each
    image. Returns (the buffer, its snnb_labels_out)."""
    pitch = w if pitch is None else pitch
    stride = pitch * h + gap
    buf = torch.full(((n - 1) * stride + (h - 1) * pitch + w + 64,), FILL, dtype=torch.uint8, device="cuda")
    o = _lib.LabelsOut()
    o.width, o.height, o.plane, o.pitch, o.image_stride = w, h, buf.data_ptr(), pitch, stride
    o.linear_filter, o.threshold = int(bool(linear)), float(threshold)
    return buf, o


def read_labels(buf, o, n):
    """(the labels [n, h, w], whether every byte outside the rows still holds FILL)."""
    b = host(buf)
    mask = np.zeros(b.shape, bool)
    for i in range(n):
        for y in range(o.height):
            s = i * o.image_stride + y * o.pitch
            mask[s:s + o.width] = True
    lab = b[mask].reshape(n, o.height, o.width)
    return lab, bool((b[~mask] == FILL).all())


def segment(m, f, o, luma=False, stream=None):
    _lib.check(_lib.lib().snnb_model_segment_frames(m.h, C.byref(f), int(luma), C.byref(o), stream if stream is not None else m._torch_stream()),
               "snnb_model_segment_frames")


def assert_labels(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.argwhere(got != want)
    assert bad.size == 0, "%s: %d of %d labels differ, first at %s: %d, want %d" % (what, len(bad), got.size, tuple(bad[0]), got[tuple(bad[0])],
                                                                                   want[tuple(bad[0])])


def y_scores(m, y, linear=True, mean=MEAN, norm=NORM):
    """Output 0 for the Y planes [N, H, W] as a 1-channel 8-bit image: the scores of luma input."""
    out, _ = m.run_image(np.ascontiguousarray(y[..., None]), [mean] * 4, [norm] * 4, linear=linear)
    return out


def median_threshold(t):
    return float(np.median(t))


SIZES = [(24, 40), (48, 80), (12, 20), (25, 41), (13, 7), (1, 1), (50, 70), (1, 97)]  # equal, above, below, odd, 1 x 1, the frames'


@pytest.mark.parametrize("classes", [1, 2, 21])
@pytest.mark.parametrize("fmt", ["nv12", "nv21", "i420", "rgba8"])
def test_formats_sizes_and_filters_bit_for_bit(ctx, model_dir, fmt, classes):
    m = conv_model(ctx, model_dir, 3, classes, fuse=True, use_cuda_graph=True)
    y, u, v = random_yuv(m.batch, 50, 70, seed=classes * 10 + len(fmt))
    rgba = expected_rgba("nv12", y, u, v, "bt601") if fmt == "rgba8" else None
    keep, f = laid_out(fmt, y, u, v, rgba=rgba)
    for linear in (True, False):
        set_params(f, linear=linear, mean4=(128.0,) * 4, norm4=(1.0 / 64.0,) * 4)
        t = host(raw_run(m, f))
        assert t.shape == (m.batch, 24, 40, classes)
        th = median_threshold(t)
        for hw in SIZES:
            for out_linear in (True, False):
                buf, o = labels_out(m.batch, hw[0], hw[1], linear=out_linear, threshold=th)
                segment(m, f, o)
                got, clean = read_labels(buf, o, m.batch)
                assert clean, (fmt, hw)
                want = seg.segment(t, hw, out_linear, th)
                assert_labels(got, want, (fmt, classes, linear, hw, out_linear))
                if hw[0] * hw[1] >= 100:
                    assert len(np.unique(want)) >= min(classes, 2) and (classes == 1 or len(np.unique(want)) > 1)


@pytest.mark.parametrize("classes", [1, 21])
@pytest.mark.parametrize("fmt", YUV)
def test_luma_input_bit_for_bit(ctx, model_dir, fmt, classes):
    m = conv_model(ctx, model_dir, 1, classes, fuse=True, use_cuda_graph=True)
    y, u, v = random_yuv(m.batch, 50, 70, seed=classes + len(fmt))
    keep, f = laid_out(fmt, y, u, v, pitch_align=128, uv_row_align=16, pad_image=1000 + 3)
    for linear in (True, False):
        set_params(f, linear=linear, mean4=(MEAN,) * 4, norm4=(NORM,) * 4)
        t = y_scores(m, y, linear)
        th = median_threshold(t)
        for hw in [(24, 40), (50, 70), (11, 13), (1, 1), (97, 150)]:
            for out_linear in (True, False):
                buf, o = labels_out(m.batch, hw[0], hw[1], linear=out_linear, threshold=th)
                segment(m, f, o, luma=True)
                got, clean = read_labels(buf, o, m.batch)
                assert clean
                assert_labels(got, seg.segment(t, hw, out_linear, th), (fmt, classes, linear, hw, out_linear))
        # the same frames without luma feed RGBA component R, another input
        if fmt == "nv12" and linear:
            buf, o = labels_out(m.batch, 24, 40, threshold=th)
            segment(m, f, o)
            assert_labels(read_labels(buf, o, m.batch)[0], seg.segment(host(raw_run(m, f)), (24, 40), True, th), "luma=0")


def test_pitched_planes_with_gaps_and_batch_3(ctx, model_dir):
    m = conv_model(ctx, model_dir, 3, 21, batch=3, fuse=True, use_cuda_graph=True)
    y, u, v = random_yuv(3, 90, 120, seed=9)
    keep, f = laid_out("nv12", y, u, v, pitch_align=256, uv_row_align=16, pad_image=4096 + 3)
    set_params(f)
    t = host(raw_run(m, f))
    for hw, pitch, gap in [((90, 120), 128, 77), ((45, 61), 64, 1), ((7, 3), 5, 0), ((1, 1), 1, 9)]:
        for linear in (True, False):
            buf, o = labels_out(3, hw[0], hw[1], pitch=pitch, gap=gap, linear=linear)
            segment(m, f, o)
            got, clean = read_labels(buf, o, 3)
            assert clean, "bytes outside the rows were written"
            assert_labels(got, seg.segment(t, hw, linear), (hw, pitch, gap, linear))
    # the Python wrapper with a strided out: the same bytes
    frames = packed("nv12", y, u, v)
    base = torch.full((3 * (128 * 90 + 77),), FILL, dtype=torch.uint8, device="cuda")
    out = torch.as_strided(base, (3, 90, 120), (128 * 90 + 77, 128, 1))
    assert m.segment_frames(frames, out=out) is out
    got = host(out)
    assert_labels(got, seg.segment(t, (90, 120), True), "strided out")
    b = host(base).reshape(3, -1)[:, :128 * 90].reshape(3, 90, 128)
    assert (b[:, :, 120:] == FILL).all() and (host(base).reshape(3, -1)[:, 128 * 90:] == FILL).all()
    dense = m.segment_frames(frames, out_hw=(45, 61), out_linear=False)
    assert dense.shape == (3, 45, 61) and dense.is_contiguous()
    assert_labels(host(dense), seg.segment(t, (45, 61), False), "dense out")


def test_256_channels(ctx, model_dir):
    m = conv_model(ctx, model_dir, 3, 256, hw=(16, 24), fuse=False)
    y, u, v = random_yuv(m.batch, 32, 48, seed=256)
    frames = packed("i420", y, u, v)
    t = host(m.run_frames(frames, format="i420", mean4=[128.0] * 4, norm4=[1.0 / 64.0] * 4, out_dtype=torch.float32))
    assert t.shape == (2, 16, 24, 256)
    for hw in [(16, 24), (37, 53), (5, 5)]:
        for linear in (True, False):
            got = host(m.segment_frames(frames, format="i420", mean4=[128.0] * 4, norm4=[1.0 / 64.0] * 4, out_hw=hw, out_linear=linear))
            want = seg.segment(t, hw, linear)
            assert_labels(got, want, (hw, linear))
    assert len(np.unique(want)) > 5 and int(np.max(seg.segment(t, (16, 24)))) > 128


@pytest.mark.parametrize("classes", [1, 21])
@pytest.mark.parametrize("fuse,graph,precision", [(False, False, None), (True, False, None), (False, True, None), (True, True, "fp16")])
def test_unet_fuse_graph_and_fp16(ctx, model_dir, classes, fuse, graph, precision):
    kw = {"precision": precision} if precision else {}
    m = unet(ctx, model_dir, (64, 64), classes, 2, fuse=fuse, use_cuda_graph=graph, **kw)
    y, u, v = random_yuv(m.batch, 96, 128, seed=classes)
    frames = packed("nv12", y, u, v)
    t = y_scores(m, y, True, 0.0, 1.0 / 255.0)
    th = median_threshold(t) if classes == 1 else 0.5
    for hw in [(64, 64), (96, 128), (31, 47)]:
        for linear in (True, False):
            got = host(m.segment_frames(frames, luma=True, mean4=[0.0] * 4, norm4=[1.0 / 255.0] * 4, out_hw=hw, out_linear=linear, threshold=th))
            want = seg.segment(t, hw, linear, th)
            assert_labels(got, want, (classes, fuse, graph, precision, hw, linear))
            assert len(np.unique(want)) >= 2
    m.close()


def test_ordering_on_the_callers_stream(ctx, model_dir):
    m = conv_model(ctx, model_dir, 3, 21, fuse=True, use_cuda_graph=True)
    frames = [packed("nv12", *random_yuv(m.batch, 60, 80, seed=s)) for s in (1, 2)]
    kw = dict(mean4=[128.0] * 4, norm4=[1.0 / 64.0] * 4, out_hw=(120, 160))
    want = [host(m.segment_frames(fr, **kw)) for fr in frames]
    assert not np.array_equal(want[0], want[1])
    torch.cuda.synchronize()

    def spin_write_segment_read(src, stream):
        with torch.cuda.stream(stream):
            torch.cuda._sleep(100_000_000)
            x = torch.empty_like(src)
            x.copy_(src)
            return m.segment_frames(x, **kw).clone()

    m.segment_frames(frames[0], **kw)
    assert np.array_equal(host(spin_write_segment_read(frames[1], torch.cuda.Stream())), want[1])
    # segment_frames between submit and wait of the same model: both results correct
    x0 = np.random.default_rng(4).uniform(0.0, 1.0, m.input_shape(0)).astype(np.float32)
    want0, _ = m.run(x0, want_classes=False)
    out = np.empty(m.output_shape(0), np.float32)
    ticket = m.submit_raw(x0.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), out.size)
    got = spin_write_segment_read(frames[0], torch.cuda.Stream())
    m.wait(ticket)
    assert np.array_equal(out, want0)
    assert np.array_equal(host(got), want[0])


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")  # the refused call leaves the caller's capture empty, as it should
def test_refusals_launch_nothing_write_nothing_and_leave_the_model_usable(ctx, model_dir):
    m = conv_model(ctx, model_dir, 3, 21, fuse=True, use_cuda_graph=True)
    y, u, v = random_yuv(m.batch, 90, 120, seed=3)
    keep, f = laid_out("nv12", y, u, v)
    set_params(f)
    keep_before = host(keep)
    buf, good = labels_out(m.batch, 45, 61, pitch=64, gap=5)
    segment(m, f, good)
    want, _ = read_labels(buf, good, m.batch)
    buf.fill_(FILL)
    torch.cuda.synchronize()

    def refused(fn, text, model=m):
        before = ctx.launches
        with pytest.raises(SnnbError) as e:
            fn()
        assert text in str(e.value), str(e.value)
        assert ctx.launches == before, "a refused call launched kernels"
        assert (host(buf) == FILL).all(), "a refused call wrote to the label plane"
        assert np.array_equal(host(keep), keep_before), "a refused call wrote to the frames"
        segment(m, f, good)
        assert_labels(read_labels(buf, good, m.batch)[0], want, "after a refusal")
        buf.fill_(FILL)
        torch.cuda.synchronize()

    def bad(**kw):
        o = _lib.LabelsOut.from_buffer_copy(good)  # `buf` holds the plane
        for k, val in kw.items():
            setattr(o, k, val)
        return o

    def bad_in(**kw):
        g = _lib.Frames.from_buffer_copy(f)
        for k, val in kw.items():
            if k in ("plane", "pitch"):
                getattr(g, k)[val[0]] = val[1]
            else:
                setattr(g, k, val)
        return g

    lib = _lib.lib()
    refused(lambda: _lib.check(lib.snnb_model_segment_frames(m.h, None, 0, C.byref(good), None), "s"), "snnb_model_segment_frames: null frames")
    refused(lambda: _lib.check(lib.snnb_model_segment_frames(m.h, C.byref(f), 0, None, None), "s"), "snnb_model_segment_frames: null out")
    # run_frames' own checks
    refused(lambda: segment(m, bad_in(format=7), good), "unknown frame format 7")
    refused(lambda: segment(m, bad_in(matrix=5), good), "unknown YUV matrix 5")
    refused(lambda: segment(m, bad_in(pitch=(0, 7)), good), "plane 0: pitch 7 is less than its row's 120 bytes")
    # the label plane
    refused(lambda: segment(m, f, bad(width=0)), "label plane size 0 x 45; width and height must be >= 1")
    refused(lambda: segment(m, f, bad(height=-1)), "width and height must be >= 1")
    refused(lambda: segment(m, f, bad(pitch=60)), "label plane pitch 60 is less than its width 61")
    host_plane = np.zeros(100000, np.uint8)
    refused(lambda: segment(m, f, bad(plane=host_plane.ctypes.data)), "unregistered host memory")
    pinned = torch.zeros(100000, dtype=torch.uint8).pin_memory()
    refused(lambda: segment(m, f, bad(plane=pinned.data_ptr())), "pinned host memory")
    refused(lambda: segment(m, f, bad(plane=None)), "label plane 0: null data pointer")
    g = torch.cuda.CUDAGraph()

    def capture():
        with torch.cuda.graph(g, capture_error_mode="relaxed"):
            segment(m, f, good)
    refused(capture, "being captured")
    # luma input from RGBA8 frames or into a 3-channel model
    rgba = expected_rgba("nv12", y, u, v, "bt601")
    keep_rgba, f_rgba = laid_out("rgba8", None, None, None, rgba=rgba)
    one = conv_model(ctx, model_dir, 1, 21)
    refused(lambda: segment(one, set_params(f_rgba), good, luma=True), "RGBA8 frames have no Y plane")
    refused(lambda: segment(m, f, good, luma=True), "the model input has 3 channels; the Y plane feeds exactly 1")
    # outputs no label plane is written from
    wide = conv_model(ctx, model_dir, 3, 257)
    yolo = load(ctx, model_dir, "yolov3tiny", (416, 416), m.batch)
    refused(lambda: segment(wide, f, good), "output 0 has 257 channels; an 8-bit label plane is written from 1 to 256")
    refused(lambda: segment(yolo, f, good), "output 0 is a YOLO detection list")
    for other in (one, wide, yolo):
        other.close()
    # the Python wrapper's own checks
    frames = packed("nv12", y, u, v)
    with pytest.raises(ValueError):
        m.segment_frames(frames, format="yuyv")
    with pytest.raises(ValueError):
        m.segment_frames(frames, out=torch.empty((m.batch, 90, 120), dtype=torch.int32, device="cuda"))
    with pytest.raises(ValueError):
        m.segment_frames(frames, out_hw=(45, 61), out=torch.empty((m.batch, 90, 120), dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        m.segment_frames(frames, out=torch.empty((m.batch + 1, 90, 120), dtype=torch.uint8, device="cuda"))


@pytest.mark.parametrize("fuse", [False, True])
def test_unet_256_batch_8_every_layer_and_1080p_labels(ctx, model_dir, fuse):
    # the reference's U-Net (modelzoo/U-Net/unet.param, grey 256 x 256 input) at batch 8: every layer of a 2-image sample against the
    # oracle at the fp32x3 bar; then 1920 x 1080 NV12 frames in, 1080p label planes out, every byte held to the restatement
    m, x, want, worst = baseline_size_check(ctx, "unet", (256, 256), 8, 2, model_dir + "/unet_full", fuse, eps=LIMIT["fp32x3"],
                                            min_layers=30 if fuse else 37)
    out, _ = m.run(x, want_classes=False)
    assert out.shape == (8, 256, 256, 1)
    np.testing.assert_allclose(out[:2], want[-1], rtol=0, atol=LIMIT["fp32x3"] * float(np.abs(want[-1]).max()))
    y, u, v = random_yuv(8, 1080, 1920, seed=1080)
    frames = packed("nv12", y, u, v)
    got = host(m.segment_frames(frames, luma=True, mean4=[0.0] * 4, norm4=[1.0 / 255.0] * 4))
    assert got.shape == (8, 1080, 1920)
    t = y_scores(m, y, True, 0.0, 1.0 / 255.0)
    assert_labels(got, seg.segment(t, (1080, 1920), True, 0.5), ("unet 1080p", fuse))
    assert 0 < int(got.sum()) < got.size, "every pixel got the same label: the comparison would be vacuous"
    m.close()
