"""10-bit device video frames (P010) on every frame path, and the BT.2020 and full-range BT.601 (JPEG) matrices.

The model input of a P010 frame is defined so that numpy float32 restates it bit for bit (oracle/yuv10.py, held to libyuv's rows by
tests/test_p010_cpu.py). So every result is held to the same entry point, or run_torch / detect_torch, on the same handle fed the
restated input: equal inputs give equal outputs. P010 output is held word for word to the restatement of the float32 output the same
handle computes. The new matrices on the 8-bit formats are held to submit_image of libyuv's RGBA8 image, as tests/test_frames_gpu.py
does for BT.601 and BT.709."""
import ctypes as C

import numpy as np
import pytest

from oracle import seg, yuv, yuv10
from shadernn_b200 import _lib
from shadernn_b200._lib import SnnbError
from test_frames_gpu import NORM, host, load, packed, random_yuv, want_image
from test_frames_out_gpu import model as out_model
from test_frames_out_gpu import params as out_params
from test_frames_out_gpu import expected as expected_8bit
from test_frames_out_gpu import spread
from test_segment_gpu import assert_labels, conv_model

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

MATRICES = ["bt601", "bt709", "bt2020", "jpeg"]
MATRIX_IDS = {"bt601": 0, "bt709": 1, "bt2020": 9, "jpeg": 0x100}
FILL16 = 0xA5A5


def random_yuv10(n, h, w, seed):
    """Smooth-ish 10-bit frames with noise: Y [n, h, w], U and V [n, ceil(h/2), ceil(w/2)] (int64)."""
    rng = np.random.default_rng(seed)
    ch, cw = yuv.chroma_shape(h, w)
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    base = (yy * 800 // max(h, 1) + xx * 200 // max(w, 1))[None]
    y = np.clip(base + rng.integers(-80, 81, (n, h, w)), 0, 1023)
    return y, rng.integers(0, 1024, (n, ch, cw)), rng.integers(0, 1024, (n, ch, cw))


def p010(y, u, v, low=0):
    """The [N, H * 3 // 2, W] uint16 CUDA tensor of even-sized frames (the Python wrapper's P010 layout)."""
    return torch.from_numpy(yuv10.p010_pack(y, u, v, low)).cuda()


def laid_out10(y, u, v, pitch_align=1, uv_row_align=1, pad_image=0, low=0):
    """P010 frames of any size in ONE device buffer filled with 0xA5A5: rows padded to `pitch_align` samples, the UV plane at
    pitch * align(H, uv_row_align), `pad_image` spare samples after each image. Returns (the buffer, its snnb_frames)."""
    n, h, w = y.shape
    ch, cw = yuv.chroma_shape(h, w)
    al = lambda x, a: (x + a - 1) // a * a  # noqa: E731
    c = np.empty((n, ch, 2 * cw), np.int64)
    c[..., 0::2], c[..., 1::2] = u, v
    planes = [y, c]
    pitches = [al(p.shape[2], pitch_align) for p in planes]
    offs = [0, pitches[0] * al(h, uv_row_align)]
    stride = offs[1] + pitches[1] * ch + pad_image
    buf = np.full((n, stride), FILL16, np.uint16)
    for i, p in enumerate(planes):
        view = buf[:, offs[i]:offs[i] + pitches[i] * p.shape[1]].reshape(n, p.shape[1], pitches[i])
        view[:, :, :p.shape[2]] = (p.astype(np.uint16) << 6) | (np.uint16(low) & 0x3F)
    d = torch.from_numpy(buf).cuda()
    f = _lib.Frames()
    f.format, f.width, f.height = _lib.FRAME_P010, w, h
    for i in range(2):
        f.plane[i], f.pitch[i], f.image_stride[i] = d.data_ptr() + 2 * offs[i], 2 * pitches[i], 2 * stride
    return d, f


def set_params(f, matrix="bt601", linear=True, mean4=(0.0,) * 4, norm4=(1.0,) * 4):
    f.matrix, f.linear_filter = MATRIX_IDS[matrix], int(bool(linear))
    f.mean4 = (C.c_float * 4)(*mean4)
    f.norm4 = (C.c_float * 4)(*norm4)
    return f


def raw_run(m, f, out_dtype=None):
    outs, obufs, _ = m._device_outputs("test", out_dtype, "nhwc", 1.0, 0.0, False)
    _lib.check(_lib.lib().snnb_model_run_frames(m.h, C.byref(f), obufs, len(outs), None, m._torch_stream()), "snnb_model_run_frames")
    return outs[0]


def model_input(m, y, u, v, matrix, linear, mean4, norm4, luma=False):
    """The restated model input [N, H, W, C] of 10-bit frames."""
    _, h, w, c = m.input_shape(0)
    tex = yuv10.luma_texels(y) if luma else yuv10.texels(y, u, v, matrix)
    return yuv10.model_input(tex, (h, w), c, linear, mean4, norm4)


def torch_out(m, x, out_dtype=None):
    return host(m.run_torch(torch.from_numpy(np.ascontiguousarray(x)).cuda(), out_dtype=out_dtype))


def split_out(words, h):
    """(Y10, U10, V10, low bits all zero) of P010 words [N, H * 3 // 2, W] read back from the device."""
    w = np.asarray(words).view(np.uint16)
    y, u, v = yuv10.p010_split(w)
    return y, u, v, not (w & 0x3F).any()


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("matrix", MATRICES)
def test_run_frames_matrices_filters(ctx, model_dir, matrix, linear):
    m = load(ctx, model_dir, "resnet18", (64, 64), 2, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["resnet18"]
    y, u, v = random_yuv10(2, 96, 80, seed=1)
    got = host(m.run_frames(p010(y, u, v), format="p010", matrix=matrix, linear=linear, mean4=mean4, norm4=norm4))
    assert np.array_equal(got, torch_out(m, model_input(m, y, u, v, matrix, linear, mean4, norm4)))
    # the low 6 bits of every word are ignored
    low = np.random.default_rng(2).integers(1, 64, (2, 144, 80))
    assert np.array_equal(host(m.run_frames(p010(y, u, v, low), format="p010", matrix=matrix, linear=linear, mean4=mean4, norm4=norm4)), got)


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("hw", [(64, 64), (100, 90), (40, 36), (33, 17), (1, 1), (63, 65)])  # equal, above, below, odd
def test_run_frames_sizes(ctx, model_dir, hw, linear):
    m = load(ctx, model_dir, "mobilenetv2", (64, 64), 2, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["mobilenetv2"]
    y, u, v = random_yuv10(2, hw[0], hw[1], seed=hw[0] * 1000 + hw[1])
    keep, f = laid_out10(y, u, v)
    got = host(raw_run(m, set_params(f, "bt2020", linear, mean4, norm4)))
    assert np.array_equal(got, torch_out(m, model_input(m, y, u, v, "bt2020", linear, mean4, norm4)))


def test_pitched_planes_gaps_and_image_strides(ctx, model_dir):
    # NVDEC's surface: 256-byte row pitch, the UV plane at pitch * align(H, 16); spare bytes between the images; P016 low bits set
    m = load(ctx, model_dir, "resnet18", (64, 64), 3, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["resnet18"]
    y, u, v = random_yuv10(3, 90, 120, seed=9)
    keep, f = laid_out10(y, u, v, pitch_align=128, uv_row_align=16, pad_image=2048 + 3, low=0x15)
    assert f.pitch[0] == 256 and f.image_stride[0] % 256 == 6
    want = torch_out(m, model_input(m, y, u, v, "bt709", True, mean4, norm4))
    assert np.array_equal(host(raw_run(m, set_params(f, "bt709", True, mean4, norm4))), want)
    surf = torch.from_numpy(np.full((3, 135 + 7, 128), FILL16, np.uint16)).cuda()  # through the wrapper: a strided view
    surf[:, :135, :120] = p010(y, u, v)
    assert np.array_equal(host(m.run_frames(surf[:, :135, :120], format="p010", matrix="bt709", mean4=mean4, norm4=norm4)), want)
    assert np.array_equal(host(m.run_frames(surf[:, :135, :120].view(torch.int16), format="p010", matrix="bt709", mean4=mean4, norm4=norm4)), want)


@pytest.mark.parametrize("matrix", ["bt2020", "jpeg"])
@pytest.mark.parametrize("fmt", ["nv12", "nv21", "i420"])
def test_new_matrices_on_8bit_formats_equal_submit_image(ctx, model_dir, fmt, matrix):
    m = load(ctx, model_dir, "resnet18", (64, 64), 2, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["resnet18"]
    y, u, v = random_yuv(2, 96, 80, seed=4)
    rgba = np.stack([yuv10.yuv_pixel(y[i], np.repeat(np.repeat(u[i], 2, 0), 2, 1), np.repeat(np.repeat(v[i], 2, 0), 2, 1), matrix)
                     for i in range(2)])
    for linear in (True, False):
        got = m.run_frames(packed(fmt, y, u, v), format=fmt, matrix=matrix, linear=linear, mean4=mean4, norm4=norm4)
        assert np.array_equal(host(got), want_image(m, rgba, mean4, norm4, linear))


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("fuse", [False, True])
def test_fuse_graph_and_fp16(ctx, model_dir, fuse, graph):
    for precision in ("fp32x3", "fp16"):
        if precision == "fp16" and not (fuse and graph):
            continue
        m = load(ctx, model_dir, "mobilenetv2", (64, 64), 2, fuse=fuse, use_cuda_graph=graph, precision=precision)
        mean4, norm4 = NORM["mobilenetv2"]
        y, u, v = random_yuv10(2, 72, 100, seed=12)
        got, cls = m.run_frames(p010(y, u, v), format="p010", matrix="jpeg", mean4=mean4, norm4=norm4, want_classes=True)
        want, want_cls = m.run_torch(torch.from_numpy(model_input(m, y, u, v, "jpeg", True, mean4, norm4)).cuda(), want_classes=True)
        assert np.array_equal(host(got), host(want)) and np.array_equal(host(cls), host(want_cls))


def test_detect_frames(ctx, model_dir):
    m = load(ctx, model_dir, "yolov3tiny", (416, 416), 2, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["yolov3tiny"]
    y, u, v = random_yuv10(2, 480, 640, seed=21)
    r1, c1 = m.detect_frames(p010(y, u, v), format="p010", matrix="bt2020", mean4=mean4, norm4=norm4)
    r2, c2 = m.detect_torch(torch.from_numpy(model_input(m, y, u, v, "bt2020", True, mean4, norm4)).cuda())
    assert np.array_equal(host(c1), host(c2)) and np.array_equal(host(r1), host(r2))


def test_run_rois(ctx, model_dir):
    m = load(ctx, model_dir, "resnet18", (64, 64), 4, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["resnet18"]
    y, u, v = random_yuv10(2, 90, 121, seed=31)
    keep, f = laid_out10(y, u, v, pitch_align=64)
    set_params(f, "bt709", True, mean4, norm4)
    rois = np.array([[0, 0, 3, 5, 64, 64], [1, 1, 10, 7, 33, 51], [1, 2, 0, 0, 121, 90], [0, 3, 100, 80, 30, 30]], np.int32)  # last: outside
    outs, obufs, _ = m._device_outputs("test", None, "nhwc", 1.0, 0.0, False)
    rois_dev = torch.from_numpy(rois).cuda()
    _lib.check(_lib.lib().snnb_model_run_rois(m.h, C.byref(f), 2, rois_dev.data_ptr(), None, obufs, len(outs), None,
                                              m._torch_stream()), "snnb_model_run_rois")
    got = host(outs[0])
    tex = [yuv10.texels(y[i:i + 1], u[i:i + 1], v[i:i + 1], "bt709") for i in range(2)]
    crops = [yuv10.model_input(tex[r[0]][:, r[3]:r[3] + r[5], r[2]:r[2] + r[4]], (64, 64), 3, True, mean4, norm4) for r in rois[:3]]
    want = torch_out(m, np.concatenate(crops + [np.zeros((1, 64, 64, 3), np.float32)]))
    assert np.array_equal(got[:3], want[:3])
    assert not got[3].any()


@pytest.mark.parametrize("luma", [False, True])
def test_segment_frames(ctx, model_dir, luma):
    m = conv_model(ctx, model_dir, 1 if luma else 3, 5, batch=2, hw=(24, 40))
    mean4, norm4 = [16.0] * 4, [1.0 / 219.0] * 4
    y, u, v = random_yuv10(2, 60, 90, seed=41)
    t = torch_out(m, model_input(m, y, u, v, "bt2020", True, mean4, norm4, luma=luma))
    for out_hw, out_linear in [((60, 90), True), ((24, 40), False), ((31, 47), True)]:
        got = host(m.segment_frames(p010(y, u, v), format="p010", matrix="bt2020", mean4=mean4, norm4=norm4, luma=luma, out_hw=out_hw,
                                    out_linear=out_linear))
        assert_labels(got, seg.segment(t, out_hw, out_linear), (luma, out_hw, out_linear))


def read_p010(buf, h, w):
    """(Y10, U10, V10, low bits zero, filler intact) of a [N, H * 3 // 2 + extra, W + extra] uint16 surface holding frames at [:, :H*3//2, :W]."""
    b = host(buf).view(np.uint16)
    y, u, v, zero = split_out(b[:, :h * 3 // 2, :w], h)
    outside = np.ones(b.shape, bool)
    outside[:, :h * 3 // 2, :w] = False
    return y, u, v, zero, bool((b[outside] == FILL16).all())


def surface(n, h, w):
    return torch.from_numpy(np.full((n, h * 3 // 2 + 3, w + 6), FILL16, np.uint16)).cuda()


@pytest.mark.parametrize("name", ["candy", "espcn", "rgba4"])
def test_transform_frames_p010(ctx, model_dir, name):
    m = out_model(ctx, model_dir, name, fuse=True, use_cuda_graph=True)
    mean4, norm4 = out_params(name)
    ih, iw = 50, 66
    y, u, v = random_yuv10(m.batch, ih, iw, seed=51)
    y8, u8, v8 = random_yuv(m.batch, ih, iw, seed=52)
    src10, src8 = p010(y, u, v), packed("nv12", y8, u8, v8)
    t10 = host(m.run_frames(src10, format="p010", matrix="bt2020", mean4=mean4, norm4=norm4, out_dtype=torch.float32))
    t8 = host(m.run_frames(src8, format="nv12", mean4=mean4, norm4=norm4, out_dtype=torch.float32))
    scale, offset = spread(t10)
    for hw, lin in [((50, 66), True), ((80, 100), True), ((30, 42), False)]:
        for fmt_in, src, t in (("p010", src10, t10), ("nv12", src8, t8)):
            buf = surface(m.batch, *hw)
            m.transform_frames(src, format=fmt_in, matrix="bt2020" if fmt_in == "p010" else "bt601", mean4=mean4, norm4=norm4,
                               out_format="p010", out_hw=hw, out_linear=lin, out_scale=scale, out_offset=offset,
                               out=buf[:, :hw[0] * 3 // 2, :hw[1]])
            gy, gu, gv, zero, intact = read_p010(buf, *hw)
            wy, wu, wv = yuv10.frames_out(t, hw, lin, scale, offset)
            assert zero and intact, (name, fmt_in, hw)
            assert np.array_equal(gy, wy) and np.array_equal(gu, wu) and np.array_equal(gv, wv), (name, fmt_in, hw, lin)
        # P010 in, 8-bit NV12 out: the 8-bit output of the same 10-bit input
        mu8 = host(m.run_frames(src10, format="p010", matrix="bt2020", mean4=mean4, norm4=norm4, out_dtype=torch.uint8, out_scale=scale,
                                out_offset=offset))
        got = host(m.transform_frames(src10, format="p010", matrix="bt2020", mean4=mean4, norm4=norm4, out_format="nv12", out_hw=hw,
                                      out_linear=lin, out_scale=scale, out_offset=offset))
        want = expected_8bit("nv12", mu8, hw, lin)
        assert np.array_equal(got[:, :hw[0]], want[0]) and np.array_equal(got[:, hw[0]:], want[1])
    # in place over the input frames (the output is written after the forward pass)
    want = host(m.transform_frames(src10, format="p010", matrix="bt2020", mean4=mean4, norm4=norm4, out_scale=scale, out_offset=offset))
    inplace = src10.clone()
    m.transform_frames(inplace, format="p010", matrix="bt2020", mean4=mean4, norm4=norm4, out_scale=scale, out_offset=offset, out=inplace)
    assert np.array_equal(host(inplace).view(np.uint16), want.view(np.uint16))


def test_transform_luma_p010(ctx, model_dir):
    m = load(ctx, model_dir, "espcn", (32, 32), 2, fuse=True, use_cuda_graph=True)
    mean, norm = 64.0 * 0.25, 1.0 / 219.0
    y, u, v = random_yuv10(2, 40, 52, seed=61)
    src = p010(y, u, v)
    t = torch_out(m, model_input(m, y, u, v, "bt601", True, [mean] * 4, [norm] * 4, luma=True))
    scale, offset = 219.0, 16.0
    for hw, lin in [((40, 52), True), ((96, 96), True), ((64, 90), False)]:
        buf = surface(2, *hw)
        m.transform_luma(src, format="p010", mean=mean, norm=norm, out_hw=hw, out_linear=lin, out_scale=scale, out_offset=offset,
                         out=buf[:, :hw[0] * 3 // 2, :hw[1]])
        gy, gu, gv, zero, intact = read_p010(buf, *hw)
        wy, wu, wv = yuv10.luma_out(t, u, v, hw, lin, scale, offset)
        assert zero and intact, hw
        assert np.array_equal(gy, wy) and np.array_equal(gu, wu) and np.array_equal(gv, wv), (hw, lin)
    want = host(m.transform_luma(src, format="p010", mean=mean, norm=norm, out_scale=scale, out_offset=offset))
    inplace = src.clone()
    m.transform_luma(inplace, format="p010", mean=mean, norm=norm, out_scale=scale, out_offset=offset, out=inplace)
    assert np.array_equal(host(inplace).view(np.uint16), want.view(np.uint16))


def test_ordering_on_the_callers_stream(ctx, model_dir):
    m = load(ctx, model_dir, "resnet18", (64, 64), 3, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["resnet18"]
    y, u, v = random_yuv10(3, 90, 120, seed=71)
    want = torch_out(m, model_input(m, y, u, v, "bt601", True, mean4, norm4))
    src = p010(y, u, v)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(100_000_000)
        x = torch.empty_like(src)
        x.copy_(src)
        got = m.run_frames(x, format="p010", mean4=mean4, norm4=norm4).clone()
    assert np.array_equal(host(got), want)


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")
def test_refusals_launch_nothing_and_leave_the_model_usable(ctx, model_dir):
    m = load(ctx, model_dir, "espcn", (32, 32), 2, fuse=True, use_cuda_graph=True)
    y, u, v = random_yuv10(2, 40, 52, seed=81)
    keep, good = laid_out10(y, u, v, pitch_align=64)
    set_params(good)
    want = host(raw_run(m, good))
    y8, u8, v8 = random_yuv(2, 40, 52, seed=82)
    nv12 = packed("nv12", y8, u8, v8)

    def refused(fn, text):
        before = ctx.launches
        with pytest.raises(SnnbError) as e:
            fn()
        assert text in str(e.value), str(e.value)
        assert ctx.launches == before, "a refused call launched kernels"
        assert np.array_equal(host(raw_run(m, good)), want)

    def bad(**kw):
        f = _lib.Frames.from_buffer_copy(good)
        for k, val in kw.items():
            if k in ("plane", "pitch", "image_stride"):
                getattr(f, k)[val[0]] = val[1]
            else:
                setattr(f, k, val)
        return f

    refused(lambda: raw_run(m, bad(pitch=(0, good.pitch[0] - 1))), "must be even")
    refused(lambda: raw_run(m, bad(image_stride=(1, good.image_stride[1] + 1))), "must be even")
    refused(lambda: raw_run(m, bad(plane=(1, good.plane[1] + 1))), "is not aligned to its 2-byte elements")
    refused(lambda: raw_run(m, bad(pitch=(1, 100))), "pitch 100 is less than its row's 104 bytes")
    refused(lambda: raw_run(m, bad(matrix=_lib.YUV_BT709 | _lib.YUV_FULL_RANGE)), "full range is defined for BT.601 only")
    refused(lambda: raw_run(m, bad(matrix=_lib.YUV_BT2020 | _lib.YUV_FULL_RANGE)), "full range is defined for BT.601 only")
    refused(lambda: raw_run(m, bad(matrix=2 | _lib.YUV_FULL_RANGE)), "unknown YUV matrix 258")
    refused(lambda: raw_run(m, bad(matrix=0x200)), "unknown YUV matrix 512")
    # transform_luma: P010 pairs with P010 only
    refused(lambda: m.transform_luma(p010(y, u, v), format="p010", out_format="nv12"), "the bit depths differ")
    refused(lambda: m.transform_luma(nv12, format="nv12", out_format="p010"), "the bit depths differ")
    # transform_frames: P010 out with an odd pitch
    o = _lib.FramesOut()
    out = torch.from_numpy(np.zeros((2, 60, 53), np.uint16)).cuda()
    o.format, o.width, o.height, o.scale, o.offset, o.linear_filter = _lib.FRAME_P010, 52, 40, 1.0, 0.0, 1
    o.plane[0], o.pitch[0], o.image_stride[0] = out.data_ptr(), 105, 60 * 106
    o.plane[1], o.pitch[1], o.image_stride[1] = out.data_ptr() + 40 * 106, 106, 60 * 106
    refused(lambda: _lib.check(_lib.lib().snnb_model_transform_frames(m.h, C.byref(good), C.byref(o), None), "t"), "must be even")
    # the wrapper's own dtype check
    with pytest.raises(ValueError):
        m.run_frames(nv12, format="p010")


def test_yolov3tiny_416_batch16_from_1080p_p010(ctx, model_dir):
    m = load(ctx, model_dir, "yolov3tiny", (416, 416), 16, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["yolov3tiny"]
    y, u, v = random_yuv10(16, 1080, 1920, seed=1080)
    x = np.concatenate([model_input(m, y[i:i + 1], u[i:i + 1], v[i:i + 1], "bt2020", True, mean4, norm4) for i in range(16)])
    r1, c1 = m.detect_frames(p010(y, u, v), format="p010", matrix="bt2020", mean4=mean4, norm4=norm4)
    r2, c2 = m.detect_torch(torch.from_numpy(x).cuda())
    assert np.array_equal(host(c1), host(c2)) and np.array_equal(host(r1), host(r2))
    assert int(host(c1).sum()) > 0


def test_candy_720_batch8_1080p_p010_to_1080p_p010(ctx, model_dir):
    m = load(ctx, model_dir, "candy", (720, 720), 8, fuse=True, use_cuda_graph=True)
    y, u, v = random_yuv10(8, 1080, 1920, seed=720)
    src = p010(y, u, v)
    t = host(m.run_frames(src, format="p010", out_dtype=torch.float32))
    x = np.concatenate([model_input(m, y[i:i + 1], u[i:i + 1], v[i:i + 1], "bt601", True, [0.0] * 4, [1.0] * 4) for i in range(8)])
    assert np.array_equal(t, torch_out(m, x, out_dtype=torch.float32))
    scale, offset = spread(t)
    got = host(m.transform_frames(src, format="p010", out_scale=scale, out_offset=offset)).view(np.uint16)
    for i in range(8):
        wy, wu, wv = yuv10.frames_out(t[i:i + 1], (1080, 1920), True, scale, offset)
        gy, gu, gv, zero = split_out(got[i:i + 1], 1080)
        assert zero and np.array_equal(gy, wy) and np.array_equal(gu, wu) and np.array_equal(gv, wv), i
