"""snnb_model_transform_frames (MixedInferenceCore.transform_frames): device frames in, model output 0 written as device frames of any
size, every byte exact.

The expected frames compose paths that are tested elsewhere: run_frames(out_dtype=uint8) on the same handle and the same frames gives M,
the model-size 8-bit output (tests/test_frames_gpu.py, tests/test_device_io_gpu.py); oracle/yuv_out.py then resizes it and converts it
as libyuv does on the host (held to libyuv by tests/test_frames_out_cpu.py)."""
import ctypes as C

import numpy as np
import pytest

from oracle import yuv, yuv_out
from shadernn_b200 import _lib, core, modelzoo
from shadernn_b200._lib import SnnbError
from test_frames_gpu import FORMAT_IDS, host, laid_out, load, packed, random_yuv, set_params

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

OUT_FORMATS = ["nv12", "nv21", "i420", "rgba8"]
# name -> (input hw, batch, input mean4, norm4); "rgba4" is a small Builder model with 4 output channels
MODELS = {"candy": ((48, 64), 2, [0.0] * 4, [1.0] * 4),
          "espcn": ((32, 32), 1, [0.0] * 4, [1.0 / 255.0] * 4),
          "rgba4": ((24, 40), 2, [0.0] * 4, [1.0 / 255.0] * 4)}
_rgba4 = {}


def model(ctx, model_dir, name, **kw):
    hw, batch = MODELS[name][:2]
    if name != "rgba4":
        return load(ctx, model_dir, name, hw, batch, **kw)
    if "path" not in _rgba4:
        b = modelzoo.Builder(seed=44)
        b.conv(b.input(hw[1], hw[0], 4), 4, 3)
        _rgba4["path"] = modelzoo.write_model(b.layers, "%s/rgba4.json" % model_dir)
    return core.MixedInferenceCore(ctx, _rgba4["path"], batch=batch, **kw)


def params(name):
    return MODELS[name][2:]


def spread(out):
    """out_scale, out_offset that map the float output's range onto a little more than 0..255, so that the 8-bit values span the
    range and both ends clamp."""
    lo, hi = float(out.min()), float(out.max())
    scale = 300.0 / (hi - lo)
    return scale, -20.0 - lo * scale


def run_f32(m, f):
    outs, obufs, _ = m._device_outputs("test", torch.float32, "nhwc", 1.0, 0.0, False)
    _lib.check(_lib.lib().snnb_model_run_frames(m.h, C.byref(f), obufs, len(outs), None, m._torch_stream()), "snnb_model_run_frames")
    return host(outs[0])


def run_u8(m, f, scale, offset):
    """M: output 0 of snnb_model_run_frames as uint8 NHWC, clamp(round(v * scale + offset), 0, 255)."""
    outs, obufs, _ = m._device_outputs("test", torch.uint8, "nhwc", scale, offset, False)
    _lib.check(_lib.lib().snnb_model_run_frames(m.h, C.byref(f), obufs, len(outs), None, m._torch_stream()), "snnb_model_run_frames")
    return host(outs[0])


def as_rgba(mu8):
    """M as RGBA8: 1 channel grey (R = G = B), 3 channels alpha 255."""
    n, h, w, c = mu8.shape
    if c == 4:
        return mu8
    rgb = np.repeat(mu8, 3, axis=3) if c == 1 else mu8
    return np.concatenate([rgb, np.full((n, h, w, 1), 255, np.uint8)], axis=3)


def expected(fmt, mu8, out_hw, linear):
    """The planes the device must write: [F] for RGBA8, else (y, c1[, c2]) of libyuv's conversion of F."""
    f = yuv_out.resize_rgba8(as_rgba(mu8), out_hw, linear)
    if fmt == "rgba8":
        return [f]
    return [p for p in yuv_out.rgba_to_frames(fmt, f) if p is not None]


def al(x, a):
    return (x + a - 1) // a * a


def out_frames(fmt, n, h, w, pitch_align=1, uv_row_align=1, pad_image=0, linear=True, scale=1.0, offset=0.0):
    """An snnb_frames_out over ONE device buffer of filler bytes, laid out as laid_out() lays out the input: returns (buffer, descriptor,
    layout)."""
    ch, cw = yuv.chroma_shape(h, w)
    shapes = {"rgba8": [(h, 4 * w)], "i420": [(h, w), (ch, cw), (ch, cw)]}.get(fmt, [(h, w), (ch, 2 * cw)])
    pitches = [al(s[1], pitch_align) for s in shapes]
    offs, cur = [], 0
    for i, s in enumerate(shapes):
        offs.append(cur)
        cur += pitches[i] * (al(s[0], uv_row_align) if i == 0 else s[0])
    stride = cur + pad_image
    buf = torch.full((n, stride), 0xA5, dtype=torch.uint8, device="cuda")
    o = _lib.FramesOut()
    o.format, o.width, o.height, o.linear_filter, o.scale, o.offset = FORMAT_IDS[fmt], w, h, int(bool(linear)), scale, offset
    for i in range(len(shapes)):
        o.plane[i], o.pitch[i], o.image_stride[i] = buf.data_ptr() + offs[i], pitches[i], stride
    return buf, o, (fmt, shapes, pitches, offs)


def read_planes(buf, layout):
    """The planes written into an out_frames() buffer; every byte outside them must still be filler."""
    fmt, shapes, pitches, offs = layout
    b = host(buf)
    untouched = np.ones(b.shape, bool)
    planes = []
    for (rows, cols), pitch, off in zip(shapes, pitches, offs):
        view = b[:, off:off + rows * pitch].reshape(b.shape[0], rows, pitch)
        planes.append(view[:, :, :cols].copy())
        untouched[:, off:off + rows * pitch].reshape(b.shape[0], rows, pitch)[:, :, :cols] = False
    assert (b[untouched] == 0xA5).all(), "bytes outside the planes were written"
    if fmt == "rgba8":
        planes[0] = planes[0].reshape(b.shape[0], shapes[0][0], -1, 4)
    return planes


def transform(m, f, o, stream=None):
    _lib.check(_lib.lib().snnb_model_transform_frames(m.h, C.byref(f), C.byref(o), stream if stream is not None else m._torch_stream()),
               "snnb_model_transform_frames")


def assert_planes(got, want, what):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape, (what, i, g.shape, w.shape)
        bad = np.argwhere(g != w)
        assert len(bad) == 0, "%s: plane %d: %d bytes differ, first at %s (%d, want %d)" % (what, i, len(bad), bad[0], g[tuple(bad[0])], w[tuple(bad[0])])


@pytest.mark.parametrize("out_fmt", OUT_FORMATS)
@pytest.mark.parametrize("name", list(MODELS))
def test_formats_filters_and_sizes(ctx, model_dir, name, out_fmt):
    m = model(ctx, model_dir, name, fuse=True, use_cuda_graph=True)
    mean4, norm4 = params(name)
    n, _, _, c = m.input_shape(0)
    _, oh, ow, oc = m.output_shape(0)
    assert oc == {"candy": 3, "espcn": 1, "rgba4": 4}[name]
    y, u, v = random_yuv(n, 50, 70, seed=len(name))
    keep, f = laid_out("nv12", y, u, v)
    set_params(f, mean4=mean4, norm4=norm4)
    scale, offset = spread(run_f32(m, f))
    mu8 = run_u8(m, f, scale, offset)
    assert len(np.unique(mu8)) > 100 and (mu8 == 0).any() and (mu8 == 255).any()
    for hw in [(oh, ow), (oh * 3 // 2 + 1, ow * 2 - 1), (oh // 2 + 1, ow // 3), (33, 17), (1, 1), (2, 3)]:
        for linear in (True, False):
            buf, o, lay = out_frames(out_fmt, n, hw[0], hw[1], linear=linear, scale=scale, offset=offset)
            transform(m, f, o)
            assert_planes(read_planes(buf, lay), expected(out_fmt, mu8, hw, linear), (name, out_fmt, hw, linear))


def test_rgba8_at_the_output_size_equals_run_frames_u8(ctx, model_dir):
    m = model(ctx, model_dir, "rgba4", fuse=True, use_cuda_graph=True)
    mean4, norm4 = params("rgba4")
    _, oh, ow, _ = m.output_shape(0)
    y, u, v = random_yuv(m.batch, 60, 90, seed=4)
    frames = packed("nv12", y, u, v)
    scale, offset = spread(host(m.run_frames(frames, mean4=mean4, norm4=norm4)))
    want = m.run_frames(frames, mean4=mean4, norm4=norm4, out_dtype=torch.uint8, out_scale=scale, out_offset=offset)
    got = m.transform_frames(frames, mean4=mean4, norm4=norm4, out_format="rgba8", out_hw=(oh, ow), out_scale=scale, out_offset=offset)
    assert got.shape == want.shape and torch.equal(got, want)
    assert len(np.unique(host(got)[..., 3])) > 100, "alpha should come from the model"


@pytest.mark.parametrize("out_fmt", OUT_FORMATS)
def test_pitched_planes_and_image_strides(ctx, model_dir, out_fmt):
    # an NVENC input surface: 256-byte row pitch, the chroma plane at pitch * align(H, 16), spare bytes between the images
    m = model(ctx, model_dir, "candy", fuse=True, use_cuda_graph=True)
    mean4, norm4 = params("candy")
    y, u, v = random_yuv(m.batch, 90, 120, seed=9)
    keep, f = laid_out("i420", y, u, v, pitch_align=256, uv_row_align=16, pad_image=4096 + 3)
    set_params(f, mean4=mean4, norm4=norm4)
    scale, offset = spread(run_f32(m, f))
    mu8 = run_u8(m, f, scale, offset)
    for hw in [(90, 120), (45, 61)]:
        buf, o, lay = out_frames(out_fmt, m.batch, hw[0], hw[1], pitch_align=256, uv_row_align=16, pad_image=4096 + 3, scale=scale, offset=offset)
        assert o.pitch[0] % 256 == 0 and o.image_stride[0] % 256 == 3
        transform(m, f, o)
        assert_planes(read_planes(buf, lay), expected(out_fmt, mu8, hw, True), (out_fmt, hw))


@pytest.mark.parametrize("fmt", ["nv12", "i420", "rgba8"])
def test_in_place_over_the_input_frames(ctx, model_dir, fmt):
    m = model(ctx, model_dir, "candy", fuse=True, use_cuda_graph=True)
    mean4, norm4 = params("candy")
    y, u, v = random_yuv(m.batch, 96, 128, seed=12)
    if fmt == "rgba8":
        frames = torch.from_numpy(np.stack([yuv.frames_to_rgba("nv12", *yuv.planes_from_yuv("nv12", y[i], u[i], v[i])) for i in range(m.batch)])).cuda()
    else:
        frames = packed(fmt, y, u, v)
    scale, offset = spread(host(m.run_frames(frames, format=fmt, mean4=mean4, norm4=norm4)))
    mu8 = host(m.run_frames(frames, format=fmt, mean4=mean4, norm4=norm4, out_dtype=torch.uint8, out_scale=scale, out_offset=offset))
    want = expected(fmt, mu8, (96, 128), True)
    got = m.transform_frames(frames, format=fmt, mean4=mean4, norm4=norm4, out_scale=scale, out_offset=offset, out=frames)
    assert got is frames
    g = host(frames)
    if fmt == "rgba8":
        assert_planes([g], want, fmt)
    elif fmt == "nv12":
        assert_planes([g[:, :96], g[:, 96:]], want, fmt)
    else:
        chroma = g[:, 96:].reshape(m.batch, -1)
        assert_planes([g[:, :96], chroma[:, :48 * 64].reshape(-1, 48, 64), chroma[:, 48 * 64:].reshape(-1, 48, 64)], want, fmt)


@pytest.mark.parametrize("fuse,graph,precision", [(False, False, None), (True, False, None), (False, True, None), (True, True, "fp16")])
def test_fuse_graph_and_fp16(ctx, model_dir, fuse, graph, precision):
    kw = {"precision": precision} if precision else {}
    for name in ("candy", "espcn"):
        m = model(ctx, model_dir, name, fuse=fuse, use_cuda_graph=graph, **kw)
        mean4, norm4 = params(name)
        y, u, v = random_yuv(m.batch, 64, 96, seed=21)
        frames = packed("nv12", y, u, v)
        scale, offset = spread(host(m.run_frames(frames, mean4=mean4, norm4=norm4)))
        mu8 = host(m.run_frames(frames, mean4=mean4, norm4=norm4, out_dtype=torch.uint8, out_scale=scale, out_offset=offset))
        for out_fmt, hw in (("nv12", (64, 96)), ("nv21", (100, 150)), ("rgba8", (31, 47))):
            got = host(m.transform_frames(frames, mean4=mean4, norm4=norm4, out_format=out_fmt, out_hw=hw, out_scale=scale, out_offset=offset))
            want = expected(out_fmt, mu8, hw, True)
            if out_fmt == "rgba8":
                assert_planes([got], want, (name, out_fmt))
            else:
                assert_planes([got[:, :hw[0]], got[:, hw[0]:]], want, (name, out_fmt))
        m.close()


def test_candy_720_batch8_1080p_nv12_to_1080p_nv12(ctx, model_dir):
    m = load(ctx, model_dir, "candy", (720, 720), 8, fuse=True, use_cuda_graph=True)
    y, u, v = random_yuv(8, 1080, 1920, seed=1920)
    frames = packed("nv12", y, u, v)
    scale, offset = spread(host(m.run_frames(frames)))
    mu8 = host(m.run_frames(frames, out_dtype=torch.uint8, out_scale=scale, out_offset=offset))
    got = host(m.transform_frames(frames, out_scale=scale, out_offset=offset))
    assert got.shape == (8, 1620, 1920)
    for i in range(8):  # one image at a time: the float32 resize of 1080p on the host is large
        assert_planes([got[i:i + 1, :1080], got[i:i + 1, 1080:]], expected("nv12", mu8[i:i + 1], (1080, 1920), True), i)
    m.close()


def test_ordering_on_the_callers_stream(ctx, model_dir):
    m = model(ctx, model_dir, "candy", fuse=True, use_cuda_graph=True)
    mean4, norm4 = params("candy")
    frames = [packed("nv12", *random_yuv(m.batch, 90, 120, seed=s)) for s in (1, 2)]
    scale, offset = spread(host(m.run_frames(frames[0], mean4=mean4, norm4=norm4)))
    kw = dict(mean4=mean4, norm4=norm4, out_scale=scale, out_offset=offset)
    want = [host(m.transform_frames(fr, **kw)) for fr in frames]
    assert not np.array_equal(want[0], want[1])
    torch.cuda.synchronize()

    def spin_write_transform_read(src, stream):
        with torch.cuda.stream(stream):
            torch.cuda._sleep(100_000_000)
            x = torch.empty_like(src)
            x.copy_(src)
            return m.transform_frames(x, **kw).clone()

    m.transform_frames(frames[0], **kw)
    assert np.array_equal(host(spin_write_transform_read(frames[1], torch.cuda.Stream())), want[1])
    # transform_frames between submit and wait of the same model: both results correct
    x0 = np.ascontiguousarray(modelzoo.synthetic_input("candy", m.batch, MODELS["candy"][0]))
    want0, _ = m.run(x0, want_classes=False)
    out = np.empty(m.output_shape(0), np.float32)
    ticket = m.submit_raw(x0.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), out.size)
    got = spin_write_transform_read(frames[0], torch.cuda.Stream())
    m.wait(ticket)
    assert np.array_equal(out, want0)
    assert np.array_equal(host(got), want[0])


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")  # the refused call leaves the caller's capture empty, as it should
def test_refusals_launch_nothing_write_nothing_and_leave_the_model_usable(ctx, model_dir, tmp_path):
    m = model(ctx, model_dir, "candy", fuse=True, use_cuda_graph=True)
    mean4, norm4 = params("candy")
    y, u, v = random_yuv(m.batch, 90, 120, seed=3)
    keep, f = laid_out("nv12", y, u, v)
    set_params(f, mean4=mean4, norm4=norm4)
    buf, good, lay = out_frames("nv12", m.batch, 90, 120)
    transform(m, f, good)
    want = read_planes(buf, lay)
    buf.fill_(0xA5)
    torch.cuda.synchronize()

    def refused(fn, text):
        before = ctx.launches
        with pytest.raises(SnnbError) as e:
            fn()
        assert text in str(e.value), str(e.value)
        assert ctx.launches == before, "a refused call launched kernels"
        assert (host(buf) == 0xA5).all(), "a refused call wrote to out"
        transform(m, f, good)
        assert_planes(read_planes(buf, lay), want, "after a refusal")
        buf.fill_(0xA5)
        torch.cuda.synchronize()

    def bad(**kw):
        o = _lib.FramesOut.from_buffer_copy(good)  # `buf` holds the planes
        for k, val in kw.items():
            if k in ("plane", "pitch"):
                getattr(o, k)[val[0]] = val[1]
            else:
                setattr(o, k, val)
        return o

    lib = _lib.lib()
    refused(lambda: _lib.check(lib.snnb_model_transform_frames(m.h, None, C.byref(good), None), "t"), "snnb_model_transform_frames: null frames")
    refused(lambda: _lib.check(lib.snnb_model_transform_frames(m.h, C.byref(f), None, None), "t"), "snnb_model_transform_frames: null out")
    refused(lambda: transform(m, f, bad(format=4)), "unknown out frame format 4")
    refused(lambda: transform(m, f, bad(width=0)), "width and height must be >= 1")
    refused(lambda: transform(m, f, bad(height=-2)), "width and height must be >= 1")
    refused(lambda: transform(m, f, bad(pitch=(0, 119))), "out plane 0: pitch 119 is less than its row's 120 bytes")
    refused(lambda: transform(m, f, bad(pitch=(1, 100))), "out plane 1: pitch 100 is less than its row's 120 bytes")
    host_frames = np.zeros(100000, np.uint8)
    refused(lambda: transform(m, f, bad(plane=(1, host_frames.ctypes.data))), "unregistered host memory")
    pinned = torch.zeros(100000, dtype=torch.uint8).pin_memory()
    refused(lambda: transform(m, f, bad(plane=(0, pinned.data_ptr()))), "pinned host memory")
    refused(lambda: transform(m, f, bad(plane=(1, None))), "out plane 1: null data pointer")
    bad_in = _lib.Frames.from_buffer_copy(f)
    bad_in.pitch[0] = 7
    refused(lambda: transform(m, bad_in, good), "plane 0: pitch 7 is less than its row's 120 bytes")
    g = torch.cuda.CUDAGraph()

    def capture():
        with torch.cuda.graph(g, capture_error_mode="relaxed"):
            transform(m, f, good)
    refused(capture, "being captured")
    # models whose output 0 cannot be written as frames, and models the frames cannot feed
    b = modelzoo.Builder(seed=5)
    b.batchnorm(b.input(20, 16, 2), "relu")
    two_ch = core.MixedInferenceCore(ctx, modelzoo.write_model(b.layers, str(tmp_path / "two_ch.json")), batch=m.batch)
    b = modelzoo.Builder(seed=3)
    b.add(b.input(20, 16, 3, index=0), b.input(20, 16, 3, index=1))
    two_in = core.MixedInferenceCore(ctx, modelzoo.write_model(b.layers, str(tmp_path / "two_in.json")), batch=m.batch)
    yolo = load(ctx, model_dir, "yolov3tiny", (416, 416), m.batch)
    refused(lambda: transform(two_ch, f, good), "output 0 has 2 channels")
    refused(lambda: transform(two_in, f, good), "the model has 2 inputs")
    refused(lambda: transform(yolo, f, good), "output 0 is a YOLO detection list")
    # the Python wrapper's own checks
    frames = packed("nv12", y, u, v)
    with pytest.raises(ValueError):
        m.transform_frames(frames, out_format="yuyv")
    with pytest.raises(ValueError):
        m.transform_frames(frames, out_hw=(45, 61))  # odd: the packed layout cannot hold it
    with pytest.raises(ValueError):
        m.transform_frames(frames, out_hw=(90, 120), out=torch.empty((m.batch, 60, 64), dtype=torch.uint8, device="cuda"))
