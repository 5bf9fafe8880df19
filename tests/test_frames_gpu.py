"""snnb_model_run_frames / snnb_model_detect_frames (MixedInferenceCore.run_frames / detect_frames): device-resident 8-bit video frames
of any size converted, resized and normalised in one kernel.

The model input must be bit-identical to what snnb_model_submit_image computes from libyuv's RGBA8 image of the same frames (its first
C components), so every output is compared bit for bit with submit_image on the same model handle. libyuv's image comes from the numpy
restatement in oracle/yuv.py, which tests/test_frames_cpu.py holds to libyuv itself."""
import ctypes as C

import numpy as np
import pytest

from oracle import yuv
from shadernn_b200 import _lib, core, modelzoo
from shadernn_b200._lib import SnnbError
from test_detect_gpu import assert_rows_agree

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

_paths = {}
NORM = {"resnet18": ([127.5] * 4, [1.0 / 127.5] * 4), "mobilenetv2": ([0.0] * 4, [1.0 / 255.0] * 4), "candy": ([0.0] * 4, [1.0] * 4),
        "espcn": ([0.0] * 4, [1.0 / 255.0] * 4), "yolov3tiny": ([127.5] * 4, [1.0 / 127.5] * 4)}
FORMAT_IDS = {"nv12": _lib.FRAME_NV12, "nv21": _lib.FRAME_NV21, "i420": _lib.FRAME_I420, "rgba8": _lib.FRAME_RGBA8}


def load(ctx, model_dir, name, hw, batch, **kw):
    key = (name, tuple(hw))
    if key not in _paths:
        _paths[key], _ = modelzoo.build(name, "%s/frames_%s_%dx%d" % (model_dir, name, hw[0], hw[1]), input_hw=hw)
    return core.MixedInferenceCore(ctx, _paths[key], batch=batch, input_hw=hw, **kw)


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def random_yuv(n, h, w, seed):
    """Smooth-ish frames (so that the resize has something to interpolate) with noise: Y [n, h, w], U and V [n, ceil(h/2), ceil(w/2)]."""
    rng = np.random.default_rng(seed)
    ch, cw = yuv.chroma_shape(h, w)
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    base = (yy * 200 // max(h, 1) + xx * 50 // max(w, 1))[None]
    y = np.clip(base + rng.integers(-20, 21, (n, h, w)), 0, 255).astype(np.uint8)
    u = rng.integers(0, 256, (n, ch, cw), dtype=np.uint8)
    v = rng.integers(0, 256, (n, ch, cw), dtype=np.uint8)
    return y, u, v


def packed(fmt, y, u, v):
    """The [N, H * 3 // 2, W] packed 4:2:0 tensor of even-sized frames (run_frames' layout)."""
    n, h, w = y.shape
    py, c1, c2 = yuv.planes_from_yuv(fmt, y, u, v)
    if fmt == "i420":
        chroma = np.concatenate([c1.reshape(n, -1), c2.reshape(n, -1)], axis=1).reshape(n, h // 2, w)
    else:
        chroma = c1
    return torch.from_numpy(np.ascontiguousarray(np.concatenate([py, chroma], axis=1))).cuda()


def laid_out(fmt, y, u, v, pitch_align=1, uv_row_align=1, pad_image=0, rgba=None):
    """Frames in ONE device buffer at any layout, as a decoder surface holds them: every plane's rows padded to `pitch_align` bytes,
    the chroma planes starting at pitch * align(H, uv_row_align), and `pad_image` spare bytes after each image. Returns (the buffer,
    which must stay alive, and its snnb_frames)."""
    n, h, w = (rgba.shape[:3] if fmt == "rgba8" else y.shape)
    al = lambda x, a: (x + a - 1) // a * a  # noqa: E731
    planes = [rgba.reshape(n, h, 4 * w)] if fmt == "rgba8" else [p for p in yuv.planes_from_yuv(fmt, y, u, v) if p is not None]
    pitches = [al(p.shape[2], pitch_align) for p in planes]
    offs, cur = [], 0
    for i, p in enumerate(planes):
        offs.append(cur)
        cur += pitches[i] * (al(p.shape[1], uv_row_align) if i == 0 else p.shape[1])
    stride = cur + pad_image
    buf = np.full((n, stride), 0xA5, np.uint8)  # filler: a read outside the planes would show
    for i, p in enumerate(planes):
        view = buf[:, offs[i]:offs[i] + pitches[i] * p.shape[1]].reshape(n, p.shape[1], pitches[i])
        view[:, :, :p.shape[2]] = p
    d = torch.from_numpy(buf).cuda()
    f = _lib.Frames()
    f.format, f.width, f.height = FORMAT_IDS[fmt], w, h
    for i in range(len(planes)):
        f.plane[i], f.pitch[i], f.image_stride[i] = d.data_ptr() + offs[i], pitches[i], stride
    return d, f


def set_params(f, matrix="bt601", linear=True, mean4=(0.0,) * 4, norm4=(1.0,) * 4):
    f.matrix, f.linear_filter = {"bt601": 0, "bt709": 1}[matrix], int(bool(linear))
    f.mean4 = (C.c_float * 4)(*mean4)
    f.norm4 = (C.c_float * 4)(*norm4)
    return f


def raw_run(m, f, out_dtype=None, stream=None):
    outs, obufs, _ = m._device_outputs("test", out_dtype, "nhwc", 1.0, 0.0, False)
    _lib.check(_lib.lib().snnb_model_run_frames(m.h, C.byref(f), obufs, len(outs), None, stream if stream is not None else m._torch_stream()),
               "snnb_model_run_frames")
    return outs[0]


def expected_rgba(fmt, y, u, v, matrix):
    return np.stack([yuv.frames_to_rgba(fmt, *yuv.planes_from_yuv(fmt, y[i], u[i], v[i]), matrix=matrix) for i in range(y.shape[0])])


def want_image(m, rgba, mean4, norm4, linear, out_u8=False):
    """submit_image + wait on libyuv's image (its first C components)."""
    c = m.input_shape(0)[3]
    out, _ = m.run_image(np.ascontiguousarray(rgba[..., :c]), mean4, norm4, linear=linear, out_u8=out_u8)
    return out


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("matrix", ["bt601", "bt709"])
@pytest.mark.parametrize("fmt", ["nv12", "nv21", "i420", "rgba8"])
def test_formats_matrices_filters_bit_identical_to_submit_image(ctx, model_dir, fmt, matrix, linear):
    m = load(ctx, model_dir, "resnet18", (64, 64), 2, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["resnet18"]
    y, u, v = random_yuv(2, 96, 80, seed=1)
    rgba = expected_rgba("nv12", y, u, v, matrix)
    if fmt == "rgba8":
        got = m.run_frames(torch.from_numpy(rgba).cuda(), format="rgba8", linear=linear, mean4=mean4, norm4=norm4)
    else:
        got = m.run_frames(packed(fmt, y, u, v), format=fmt, matrix=matrix, linear=linear, mean4=mean4, norm4=norm4)
    assert np.array_equal(host(got), want_image(m, rgba, mean4, norm4, linear))


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("fmt", ["nv12", "i420", "rgba8"])
@pytest.mark.parametrize("hw", [(64, 64), (100, 90), (40, 36), (33, 17), (1, 1), (63, 65)])  # equal, above, below, odd
def test_frame_sizes(ctx, model_dir, hw, fmt, linear):
    m = load(ctx, model_dir, "mobilenetv2", (64, 64), 2, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["mobilenetv2"]
    y, u, v = random_yuv(2, hw[0], hw[1], seed=hw[0] * 1000 + hw[1])
    rgba = expected_rgba("nv12", y, u, v, "bt601")
    keep, f = laid_out(fmt, y, u, v, rgba=rgba)
    got = raw_run(m, set_params(f, linear=linear, mean4=mean4, norm4=norm4))
    assert np.array_equal(host(got), want_image(m, rgba, mean4, norm4, linear))


@pytest.mark.parametrize("fmt", ["nv12", "nv21", "i420", "rgba8"])
def test_pitched_planes_and_image_strides(ctx, model_dir, fmt):
    # NVDEC's surface: 256-byte row pitch, the chroma plane at pitch * align(H, 16); and spare bytes between the images
    m = load(ctx, model_dir, "resnet18", (64, 64), 3, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["resnet18"]
    y, u, v = random_yuv(3, 90, 120, seed=9)
    rgba = expected_rgba("nv12", y, u, v, "bt709")
    keep, f = laid_out(fmt, y, u, v, pitch_align=256, uv_row_align=16, pad_image=4096 + 3, rgba=rgba)
    assert f.pitch[0] == (256 if fmt != "rgba8" else 512) and f.image_stride[0] % 256 == 3
    got = raw_run(m, set_params(f, matrix="bt709", mean4=mean4, norm4=norm4))
    want = want_image(m, rgba, mean4, norm4, True)
    assert np.array_equal(host(got), want)
    if fmt == "nv12":  # the same pitched surface through run_frames: a strided [N, H * 3 // 2, W] view with the UV rows right below Y
        p = packed("nv12", y, u, v)
        surf = torch.zeros((3, 135 + 7, 256), dtype=torch.uint8, device="cuda")
        surf[:, :135, :120] = p
        assert np.array_equal(host(m.run_frames(surf[:, :135, :120], matrix="bt709", mean4=mean4, norm4=norm4)), want)
    if fmt == "rgba8":
        surf = torch.zeros((3, 90, 130, 4), dtype=torch.uint8, device="cuda")
        surf[:, :, :120] = torch.from_numpy(rgba).cuda()
        assert np.array_equal(host(m.run_frames(surf[:, :, :120], format="rgba8", mean4=mean4, norm4=norm4)), want)


CONFIGS = [("resnet18", (64, 64), 3),  # stem reads the feed copy only (feed_only input)
           ("mobilenetv2", (64, 64), 2),
           ("candy", (48, 64), 2),  # U8 output below
           ("espcn", (32, 32), 1)]  # one channel: RGBA component R


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("fuse", [False, True])
@pytest.mark.parametrize("name,hw,batch", CONFIGS)
def test_models_bit_identical_and_nv12_equals_rgba8(ctx, model_dir, name, hw, batch, fuse, graph):
    m = load(ctx, model_dir, name, hw, batch, fuse=fuse, use_cuda_graph=graph)
    mean4, norm4 = NORM[name]
    y, u, v = random_yuv(batch, hw[0] * 3 // 2, hw[1] + 10, seed=len(name))
    rgba = expected_rgba("nv12", y, u, v, "bt601")
    out_u8 = name == "candy"
    dt = torch.uint8 if out_u8 else None
    got = host(m.run_frames(packed("nv12", y, u, v), mean4=mean4, norm4=norm4, out_dtype=dt))
    assert np.array_equal(got, want_image(m, rgba, mean4, norm4, True, out_u8=out_u8))
    assert np.array_equal(got, host(m.run_frames(torch.from_numpy(rgba).cuda(), format="rgba8", mean4=mean4, norm4=norm4, out_dtype=dt)))


def test_resnet18_fp16_and_classes(ctx, model_dir):
    m = load(ctx, model_dir, "resnet18", (64, 64), 3, fuse=True, use_cuda_graph=True, precision="fp16")
    mean4, norm4 = NORM["resnet18"]
    y, u, v = random_yuv(3, 120, 100, seed=16)
    rgba = expected_rgba("i420", y, u, v, "bt601")
    out, cls = m.run_frames(packed("i420", y, u, v), format="i420", mean4=mean4, norm4=norm4, want_classes=True)
    want, want_cls = m.run_image(np.ascontiguousarray(rgba[..., :3]), mean4, norm4, want_classes=True)
    assert np.array_equal(host(out), want) and np.array_equal(host(cls), want_cls)


def _submit_image_boxes(m, img, mean4, norm4, linear=True):
    io = _lib.ImageIO()
    n, sh, sw, _ = img.shape
    io.input_u8, io.src_height, io.src_width, io.linear_filter = img.ctypes.data, sh, sw, int(linear)
    io.mean4 = (C.c_float * 4)(*mean4)
    io.norm4 = (C.c_float * 4)(*norm4)
    t = C.c_int()
    _lib.check(_lib.lib().snnb_model_submit_image(m.h, C.byref(io), C.byref(t)), "snnb_model_submit_image")
    m.wait(t.value)
    return [m.boxes(i) for i in range(m.batch)]


def test_yolov3tiny_416_batch16_from_1080p_nv12(ctx, model_dir):
    m = load(ctx, model_dir, "yolov3tiny", (416, 416), 16, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["yolov3tiny"]
    y, u, v = random_yuv(16, 1080, 1920, seed=1080)
    rgba = expected_rgba("nv12", y, u, v, "bt601")
    img = np.ascontiguousarray(rgba[..., :3])
    rows, counts = m.detect_frames(packed("nv12", y, u, v), mean4=mean4, norm4=norm4)
    want = _submit_image_boxes(m, img, mean4, norm4)
    assert_rows_agree(rows, counts, want, "detect_frames 1080p NV12")
    # at the model's size the frames feed the network exactly as detect_torch's U8 input of libyuv's RGB does: bit-identical rows
    y, u, v = random_yuv(16, 416, 416, seed=416)
    rgb = np.ascontiguousarray(expected_rgba("nv12", y, u, v, "bt601")[..., :3])
    r1, c1 = m.detect_frames(packed("nv12", y, u, v), mean4=mean4, norm4=norm4)
    r2, c2 = m.detect_torch(torch.from_numpy(rgb).cuda(), mean4=mean4, norm4=norm4)
    assert np.array_equal(host(c1), host(c2)) and np.array_equal(host(r1), host(r2))


def test_ordering_on_the_callers_stream(ctx, model_dir):
    m = load(ctx, model_dir, "resnet18", (64, 64), 3, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["resnet18"]
    frames = [random_yuv(3, 90, 120, seed=s) for s in (1, 2)]
    want = [want_image(m, expected_rgba("nv12", *fr, "bt601"), mean4, norm4, True) for fr in frames]
    src = [packed("nv12", *fr) for fr in frames]
    torch.cuda.synchronize()

    def spin_write_run_read(s, stream):
        with torch.cuda.stream(stream):
            torch.cuda._sleep(100_000_000)
            x = torch.empty_like(s)
            x.copy_(s)
            return m.run_frames(x, mean4=mean4, norm4=norm4).clone()

    m.run_frames(src[0], mean4=mean4, norm4=norm4)
    s1 = torch.cuda.Stream()
    assert np.array_equal(host(spin_write_run_read(src[1], s1)), want[1])
    # run_frames between submit and wait of the same model: both results correct
    x0 = np.ascontiguousarray(modelzoo.synthetic_input("resnet18", 3, (64, 64)))
    want0, _ = m.run(x0, want_classes=False)
    out = np.empty(m.output_shape(0), np.float32)
    ticket = m.submit_raw(x0.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), out.size)
    got = spin_write_run_read(src[0], torch.cuda.Stream())
    m.wait(ticket)
    assert np.array_equal(out, want0)
    assert np.array_equal(host(got), want[0])


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")  # the refused call leaves the caller's capture empty, as it should
def test_refusals_launch_nothing_and_leave_the_model_usable(ctx, model_dir, tmp_path):
    m = load(ctx, model_dir, "resnet18", (64, 64), 3, fuse=True, use_cuda_graph=True)
    y, u, v = random_yuv(3, 90, 120, seed=3)
    keep, good = laid_out("nv12", y, u, v)
    want = host(raw_run(m, set_params(good)))

    def refused(fn, text):
        before = ctx.launches
        with pytest.raises(SnnbError) as e:
            fn()
        assert text in str(e.value), str(e.value)
        assert ctx.launches == before, "a refused call launched kernels"
        assert np.array_equal(host(raw_run(m, set_params(good))), want)

    def bad(**kw):
        f = _lib.Frames.from_buffer_copy(good)  # `keep` holds the planes
        for k, val in kw.items():
            if k in ("plane", "pitch"):
                getattr(f, k)[val[0]] = val[1]
            else:
                setattr(f, k, val)
        return f

    refused(lambda: raw_run(m, bad(format=4)), "unknown frame format 4")
    refused(lambda: raw_run(m, bad(matrix=2)), "unknown YUV matrix 2")
    refused(lambda: raw_run(m, bad(width=0)), "width and height must be >= 1")
    refused(lambda: raw_run(m, bad(height=-3)), "width and height must be >= 1")
    refused(lambda: raw_run(m, bad(pitch=(0, 119))), "pitch 119 is less than its row's 120 bytes")
    refused(lambda: raw_run(m, bad(pitch=(1, 118))), "pitch 118 is less than its row's 120 bytes")
    host_frames = np.zeros(1000, np.uint8)
    refused(lambda: raw_run(m, bad(plane=(1, host_frames.ctypes.data))), "unregistered host memory")
    pinned = torch.zeros(1000, dtype=torch.uint8).pin_memory()
    refused(lambda: raw_run(m, bad(plane=(0, pinned.data_ptr()))), "pinned host memory")
    refused(lambda: raw_run(m, bad(plane=(1, None))), "null data pointer")
    # the caller's stream is being captured
    g = torch.cuda.CUDAGraph()

    def capture():
        with torch.cuda.graph(g, capture_error_mode="relaxed"):
            raw_run(m, set_params(good))
    refused(capture, "being captured")
    # models the frames cannot feed: more than 4 input channels, two inputs; detect_frames on a classifier; run_frames on a detector
    b = modelzoo.Builder(seed=5)
    b.batchnorm(b.input(20, 13, 5), "relu")
    wide = core.MixedInferenceCore(ctx, modelzoo.write_model(b.layers, str(tmp_path / "wide.json")), batch=3)
    b = modelzoo.Builder(seed=3)
    b.add(b.input(20, 16, 3, index=0), b.input(20, 16, 3, index=1))
    two = core.MixedInferenceCore(ctx, modelzoo.write_model(b.layers, str(tmp_path / "two.json")), batch=3)
    yolo = load(ctx, model_dir, "yolov3tiny", (416, 416), 3)
    refused(lambda: raw_run(wide, set_params(good)), "frames feed 1 to 4")
    refused(lambda: raw_run(two, set_params(good)), "the model has 2 inputs")
    refused(lambda: m.detect_frames(packed("nv12", y, u, v)), "no YOLO output; use snnb_model_run_frames")
    refused(lambda: yolo.run_frames(packed("nv12", y, u, v)), "use snnb_model_detect_frames")
    refused(lambda: yolo.detect_frames(packed("nv12", y, u, v), max_rows=0), "max_rows 0")
    # the Python wrapper's own checks
    with pytest.raises(ValueError):
        m.run_frames(packed("nv12", y, u, v)[:2])  # 2 frames, batch 3
    with pytest.raises(ValueError):
        m.run_frames(packed("nv12", y, u, v), format="yuyv")
