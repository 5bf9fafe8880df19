"""snnb_model_transform_luma (MixedInferenceCore.transform_luma): the Y plane of device frames into a 1-channel model, output 0 written
back as the Y plane of device frames of any size, the source chroma resized beside it; every byte exact.

The expected values compose paths that are tested elsewhere: run_image of the host Y planes on the same handle gives the model input
(compared through the last layer's output) and M, the model-size 8-bit output (tests/test_frames_gpu.py, tests/test_device_io_gpu.py);
oracle/yuv_out.py resizes M, and oracle/luma.py resizes the chroma planes (tests/test_luma_cpu.py)."""
import ctypes as C

import numpy as np
import pytest

from oracle import luma, oracle, yuv, yuv_out
from shadernn_b200 import _lib, core, modelzoo
from shadernn_b200._lib import SnnbError
from test_frames_gpu import FORMAT_IDS, host, laid_out, load, packed, random_yuv, set_params
from test_frames_out_gpu import assert_planes, out_frames, read_planes, spread

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

YUV = ["nv12", "nv21", "i420"]
MEAN, NORM = 16.0, 1.0 / 219.0  # limited-range Y into a model trained on Y / 255
_paths = {}


def espcn(ctx, model_dir, hw=(24, 40), batch=2, **kw):
    return load(ctx, model_dir, "espcn", hw, batch, **kw)


def builder_model(ctx, model_dir, name, hw, in_c, out_c, batch, **kw):
    """A small Builder model: one 3x3 convolution from in_c to out_c channels at the input's size."""
    if name not in _paths:
        b = modelzoo.Builder(seed=61)
        b.conv(b.input(hw[1], hw[0], in_c), out_c, 3)
        _paths[name] = modelzoo.write_model(b.layers, "%s/%s.json" % (model_dir, name))
    return core.MixedInferenceCore(ctx, _paths[name], batch=batch, **kw)


def last_layer(m):
    torch.cuda.synchronize()
    return m.layer_output(m.num_layers - 1)


def want_input(m, y, linear):
    """The last layer's output after run_image of the Y planes [N, H, W] (submit_image + wait on the same handle)."""
    m.run_image(np.ascontiguousarray(y[..., None]), [MEAN] * 4, [NORM] * 4, linear=linear)
    return last_layer(m)


def want_m(m, y, linear, scale, offset):
    """M: run_image's U8 output [N, h, w, 1] for the Y planes."""
    out, _ = m.run_image(np.ascontiguousarray(y[..., None]), [MEAN] * 4, [NORM] * 4, linear=linear, out_u8=True, out_scale=scale, out_offset=offset)
    return out


def expected(fmt, mu8, u, v, out_hw, linear):
    """The planes the device must write: Y = M resized as transform_frames resizes R, chroma by oracle/luma.py."""
    y = yuv_out.resize_rgba8(mu8, out_hw, linear)[..., 0]
    assert np.array_equal(luma.resize_plane(mu8[..., 0], out_hw, linear), y)
    uo, vo = luma.resize_chroma(u, v, out_hw, linear)
    return [p for p in yuv.planes_from_yuv(fmt, y, uo, vo) if p is not None]


def luma_frames(f, linear):
    set_params(f, linear=linear, mean4=(MEAN,) * 4, norm4=(NORM,) * 4)
    return f


def transform(m, f, o, stream=None):
    _lib.check(_lib.lib().snnb_model_transform_luma(m.h, C.byref(f), C.byref(o), stream if stream is not None else m._torch_stream()),
               "snnb_model_transform_luma")


def scale_for(m, y):
    """out_scale, out_offset that spread the float output over a little more than 0..255, so that both ends clamp."""
    out, _ = m.run_image(np.ascontiguousarray(y[..., None]), [MEAN] * 4, [NORM] * 4)
    return spread(out)


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("fmt", YUV)
def test_model_input_bit_identical_to_submit_image_of_the_y_planes(ctx, model_dir, fmt, linear):
    m = espcn(ctx, model_dir, fuse=True, use_cuda_graph=True)
    mh, mw = m.input_shape(0)[1:3]
    assert m.input_shape(0)[3] == 1
    _, oh, ow, _ = m.output_shape(0)
    for hw in [(mh, mw), (mh * 2 + 3, mw * 3 // 2), (mh // 2, mw // 3), (33, 17), (1, 1), (mh + 1, mw - 1)]:  # equal, above, below, odd
        y, u, v = random_yuv(m.batch, hw[0], hw[1], seed=hw[0] * 100 + hw[1])
        keep, f = laid_out(fmt, y, u, v)
        buf, o, _ = out_frames("nv12", m.batch, oh, ow)
        transform(m, luma_frames(f, linear), o)
        got = last_layer(m)
        assert np.array_equal(got, want_input(m, y, linear)), (fmt, hw, linear)


@pytest.mark.parametrize("fmt", YUV)
def test_model_input_from_pitched_planes_and_image_strides(ctx, model_dir, fmt):
    m = espcn(ctx, model_dir, fuse=True, use_cuda_graph=True)
    _, oh, ow, _ = m.output_shape(0)
    y, u, v = random_yuv(m.batch, 45, 61, seed=8)
    keep, f = laid_out(fmt, y, u, v, pitch_align=256, uv_row_align=16, pad_image=4096 + 3)
    assert f.pitch[0] == 256 and f.image_stride[0] % 256 == 3
    buf, o, _ = out_frames("nv12", m.batch, oh, ow)
    transform(m, luma_frames(f, True), o)
    assert np.array_equal(last_layer(m), want_input(m, y, True))


@pytest.mark.parametrize("out_fmt", YUV)
@pytest.mark.parametrize("fmt", YUV)
def test_y_plane_and_chroma_for_every_format_pair_filter_and_size(ctx, model_dir, fmt, out_fmt):
    m = espcn(ctx, model_dir, fuse=True, use_cuda_graph=True)
    mh, mw = m.input_shape(0)[1:3]
    _, oh, ow, _ = m.output_shape(0)
    fh, fw = 30, 44
    y, u, v = random_yuv(m.batch, fh, fw, seed=len(fmt) * 10 + len(out_fmt))
    keep, f = laid_out(fmt, y, u, v)
    scale, offset = scale_for(m, y)
    for linear in (True, False):
        mu8 = want_m(m, y, linear, scale, offset)
        assert len(np.unique(mu8)) > 100 and (mu8 == 0).any() and (mu8 == 255).any()
        # equal to the frames, 2x the frames (= the output's size), smaller, odd on both sides, and 1 x 1
        for hw in [(fh, fw), (2 * fh, 2 * fw), (oh, ow), (fh // 2 + 1, fw // 3), (33, 17), (61, 89), (1, 1)]:
            for out_linear in (True, False):
                buf, o, lay = out_frames(out_fmt, m.batch, hw[0], hw[1], linear=out_linear, scale=scale, offset=offset)
                transform(m, luma_frames(f, linear), o)
                assert_planes(read_planes(buf, lay), expected(out_fmt, mu8, u, v, hw, out_linear), (fmt, out_fmt, hw, linear, out_linear))


@pytest.mark.parametrize("out_fmt", YUV)
def test_pitched_out_planes_leave_every_filler_byte(ctx, model_dir, out_fmt):
    # an NVENC input surface: 256-byte row pitch, the chroma plane at pitch * align(H, 16), spare bytes between the images
    m = espcn(ctx, model_dir, fuse=True, use_cuda_graph=True)
    y, u, v = random_yuv(m.batch, 45, 61, seed=19)
    keep, f = laid_out("i420", y, u, v, pitch_align=256, uv_row_align=16, pad_image=4096 + 3)
    scale, offset = scale_for(m, y)
    mu8 = want_m(m, y, True, scale, offset)
    for hw in [(90, 122), (45, 61), (23, 31)]:
        buf, o, lay = out_frames(out_fmt, m.batch, hw[0], hw[1], pitch_align=256, uv_row_align=16, pad_image=4096 + 3, scale=scale, offset=offset)
        assert o.pitch[0] % 256 == 0 and o.image_stride[0] % 256 == 3
        transform(m, luma_frames(f, True), o)
        assert_planes(read_planes(buf, lay), expected(out_fmt, mu8, u, v, hw, True), (out_fmt, hw))


@pytest.mark.parametrize("fmt", ["nv12", "i420"])
def test_in_place_equals_out_of_place(ctx, model_dir, fmt):
    m = builder_model(ctx, model_dir, "luma_1to1", (48, 64), 1, 1, 2, fuse=True, use_cuda_graph=True)
    y, u, v = random_yuv(m.batch, 48, 64, seed=31)
    frames = packed(fmt, y, u, v)
    scale, offset = scale_for(m, y)
    kw = dict(format=fmt, mean=MEAN, norm=NORM, out_scale=scale, out_offset=offset)
    want = host(m.transform_luma(frames, **kw))
    assert not np.array_equal(want[:, :48], y), "the filter should change Y"
    got = m.transform_luma(frames, out=frames, **kw)
    assert got is frames
    assert np.array_equal(host(frames), want)
    mu8 = want_m(m, y, True, scale, offset)
    g = host(frames)
    if fmt == "nv12":
        assert_planes([g[:, :48], g[:, 48:]], expected(fmt, mu8, u, v, (48, 64), True), fmt)
    else:
        chroma = g[:, 48:].reshape(m.batch, -1)
        assert_planes([g[:, :48], chroma[:, :24 * 32].reshape(-1, 24, 32), chroma[:, 24 * 32:].reshape(-1, 24, 32)],
                      expected(fmt, mu8, u, v, (48, 64), True), fmt)


@pytest.mark.parametrize("fuse,graph,precision", [(False, False, None), (True, False, None), (False, True, None), (True, True, "fp16")])
def test_espcn_fuse_graph_and_fp16(ctx, model_dir, fuse, graph, precision):
    kw = {"precision": precision} if precision else {}
    m = espcn(ctx, model_dir, (32, 48), 2, fuse=fuse, use_cuda_graph=graph, **kw)
    y, u, v = random_yuv(m.batch, 64, 96, seed=41)
    frames = packed("nv12", y, u, v)
    scale, offset = scale_for(m, y)
    mu8 = want_m(m, y, True, scale, offset)
    for out_fmt, hw in (("nv12", (64, 96)), ("i420", (128, 192)), ("nv21", (30, 46))):
        got = host(m.transform_luma(frames, mean=MEAN, norm=NORM, out_format=out_fmt, out_hw=hw, out_scale=scale, out_offset=offset))
        want = expected(out_fmt, mu8, u, v, hw, True)
        if out_fmt == "i420":
            ch, cw = hw[0] // 2, hw[1] // 2
            chroma = got[:, hw[0]:].reshape(m.batch, -1)
            planes = [got[:, :hw[0]], chroma[:, :ch * cw].reshape(-1, ch, cw), chroma[:, ch * cw:].reshape(-1, ch, cw)]
        else:
            planes = [got[:, :hw[0]], got[:, hw[0]:]]
        assert_planes(planes, want, (fuse, graph, precision, out_fmt))
    m.close()


def test_espcn_1080p_nv12_to_2160p_nv12(ctx, model_dir):
    # the reference's runESPCN input is a 1920 x 1080 single-channel image: a 1080p decoder frame's Y plane, upscaled 2x
    hw = (1080, 1920)
    path, layers = modelzoo.build("espcn", model_dir + "/espcn_1080p", input_hw=hw)
    m = core.MixedInferenceCore(ctx, path, batch=1, input_hw=hw, fuse=False)
    y, u, v = random_yuv(1, hw[0], hw[1], seed=1080)
    frames = packed("nv12", y, u, v)
    yin = np.ascontiguousarray(y[..., None])
    scale, offset = spread(m.run_image(yin, [0.0] * 4, [1.0 / 255.0] * 4)[0])
    got = host(m.transform_luma(frames, mean=0.0, norm=1.0 / 255.0, out_hw=(2160, 3840), out_scale=scale, out_offset=offset))
    assert got.shape == (1, 3240, 3840)
    # every layer against the oracle, fed the model input (Y - 0) * (1 / 255) in float32
    x = ((y[..., None].astype(np.float32) - np.float32(0.0)) * np.float32(1.0 / 255.0)).astype(np.float32)
    want_layers = oracle.Model(path).run(x, return_all=True)
    torch.cuda.synchronize()
    assert m.num_layers == len(want_layers) == len(layers)
    for i in range(m.num_layers):
        lname, _, shape = m.layer_info(i)
        out = m.layer_output(i)
        assert out.shape == want_layers[i].shape, (lname, out.shape, want_layers[i].shape)
        top = float(np.abs(want_layers[i]).max())
        err = float(np.abs(out.astype(np.float64) - want_layers[i].astype(np.float64)).max())
        assert err <= 1e-3 * top, "%s: max |err| %.3g of the range %.3g" % (lname, err, top)
    # the model input is submit_image's of the Y plane, compared through the last layer
    m.run_image(yin, [0.0] * 4, [1.0 / 255.0] * 4)
    assert np.array_equal(out, last_layer(m))
    mu8, _ = m.run_image(yin, [0.0] * 4, [1.0 / 255.0] * 4, out_u8=True, out_scale=scale, out_offset=offset)
    assert mu8.shape == (1, 2160, 3840, 1) and len(np.unique(mu8)) > 100 and (mu8 == 0).any() and (mu8 == 255).any()
    uo, vo = luma.resize_chroma(u, v, (2160, 3840), True)
    assert_planes([got[:, :2160], got[:, 2160:]], [mu8[..., 0], yuv.planes_from_yuv("nv12", mu8[..., 0], uo, vo)[1]], "espcn 1080p")
    m.close()


def test_ordering_on_the_callers_stream(ctx, model_dir):
    m = espcn(ctx, model_dir, fuse=True, use_cuda_graph=True)
    frames = [packed("nv12", *random_yuv(m.batch, 60, 80, seed=s)) for s in (1, 2)]
    kw = dict(mean=MEAN, norm=NORM, out_hw=(120, 160), out_scale=219.0, out_offset=16.0)
    want = [host(m.transform_luma(fr, **kw)) for fr in frames]
    assert not np.array_equal(want[0], want[1])
    torch.cuda.synchronize()

    def spin_write_transform_read(src, stream):
        with torch.cuda.stream(stream):
            torch.cuda._sleep(100_000_000)
            x = torch.empty_like(src)
            x.copy_(src)
            return m.transform_luma(x, **kw).clone()

    m.transform_luma(frames[0], **kw)
    assert np.array_equal(host(spin_write_transform_read(frames[1], torch.cuda.Stream())), want[1])
    # transform_luma between submit and wait of the same model: both results correct
    x0 = np.ascontiguousarray(modelzoo.synthetic_input("espcn", m.batch, m.input_shape(0)[1:3]))
    want0, _ = m.run(x0, want_classes=False)
    out = np.empty(m.output_shape(0), np.float32)
    ticket = m.submit_raw(x0.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), out.size)
    got = spin_write_transform_read(frames[0], torch.cuda.Stream())
    m.wait(ticket)
    assert np.array_equal(out, want0)
    assert np.array_equal(host(got), want[0])


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")  # the refused call leaves the caller's capture empty, as it should
def test_refusals_launch_nothing_write_nothing_and_leave_the_model_usable(ctx, model_dir, tmp_path):
    m = espcn(ctx, model_dir, fuse=True, use_cuda_graph=True)
    y, u, v = random_yuv(m.batch, 90, 120, seed=3)
    keep, f = laid_out("nv12", y, u, v)
    luma_frames(f, True)
    keep_before = host(keep)
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
        assert np.array_equal(host(keep), keep_before), "a refused call wrote to the frames"
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

    def bad_in(**kw):
        g = _lib.Frames.from_buffer_copy(f)
        for k, val in kw.items():
            if k in ("plane", "pitch"):
                getattr(g, k)[val[0]] = val[1]
            else:
                setattr(g, k, val)
        return g

    lib = _lib.lib()
    refused(lambda: _lib.check(lib.snnb_model_transform_luma(m.h, None, C.byref(good), None), "t"), "snnb_model_transform_luma: null frames")
    refused(lambda: _lib.check(lib.snnb_model_transform_luma(m.h, C.byref(f), None, None), "t"), "snnb_model_transform_luma: null out")
    # RGBA8 on either side, unknown formats and matrices
    rgba = np.stack([yuv.frames_to_rgba("nv12", *yuv.planes_from_yuv("nv12", y[i], u[i], v[i])) for i in range(m.batch)])
    keep_rgba, f_rgba = laid_out("rgba8", None, None, None, rgba=rgba)
    refused(lambda: transform(m, luma_frames(f_rgba, True), good), "RGBA8 frames have no Y plane")
    refused(lambda: transform(m, f, bad(format=_lib.FRAME_RGBA8, pitch=(0, 4 * 120))), "out format RGBA8 has no Y plane")
    refused(lambda: transform(m, bad_in(format=7), good), "unknown frame format 7")
    refused(lambda: transform(m, bad_in(matrix=5), good), "unknown YUV matrix 5")
    refused(lambda: transform(m, f, bad(format=4)), "unknown out frame format 4")
    refused(lambda: transform(m, f, bad(width=0)), "width and height must be >= 1")
    # short pitches, host memory, null planes
    refused(lambda: transform(m, bad_in(pitch=(0, 7)), good), "plane 0: pitch 7 is less than its row's 120 bytes")
    refused(lambda: transform(m, f, bad(pitch=(0, 119))), "out plane 0: pitch 119 is less than its row's 120 bytes")
    refused(lambda: transform(m, f, bad(pitch=(1, 100))), "out plane 1: pitch 100 is less than its row's 120 bytes")
    host_frames = np.zeros(100000, np.uint8)
    refused(lambda: transform(m, f, bad(plane=(1, host_frames.ctypes.data))), "unregistered host memory")
    refused(lambda: transform(m, bad_in(plane=(1, host_frames.ctypes.data)), good), "unregistered host memory")
    pinned = torch.zeros(100000, dtype=torch.uint8).pin_memory()
    refused(lambda: transform(m, f, bad(plane=(0, pinned.data_ptr()))), "pinned host memory")
    refused(lambda: transform(m, f, bad(plane=(1, None))), "out plane 1: null data pointer")
    g = torch.cuda.CUDAGraph()

    def capture():
        with torch.cuda.graph(g, capture_error_mode="relaxed"):
            transform(m, f, good)
    refused(capture, "being captured")
    # out chroma over the source chroma at another size, or shifted at the same size; out's Y over the source chroma
    c0 = f.plane[1]
    small = bad(width=60, height=45, plane=(1, c0))
    small.pitch[0], small.pitch[1] = 60, 60
    refused(lambda: transform(m, f, small), "out plane 1 overlaps source chroma plane 1")
    refused(lambda: transform(m, f, bad(plane=(1, c0 + 2))), "out plane 1 overlaps source chroma plane 1")
    refused(lambda: transform(m, f, bad(plane=(0, c0 + 5))), "out plane 0 overlaps source chroma plane 1")
    # models the Y plane cannot feed, and outputs it cannot be written from
    resnet = load(ctx, model_dir, "resnet18", (64, 64), m.batch)
    candy = load(ctx, model_dir, "candy", (48, 64), m.batch)
    yolo = load(ctx, model_dir, "yolov3tiny", (416, 416), m.batch)
    one_to_three = builder_model(ctx, model_dir, "luma_1to3", (24, 40), 1, 3, m.batch)
    refused(lambda: transform(resnet, f, good), "the model input has 3 channels; the Y plane feeds exactly 1")
    refused(lambda: transform(candy, f, good), "the model input has 3 channels; the Y plane feeds exactly 1")
    refused(lambda: transform(yolo, f, good), "the model input has 3 channels; the Y plane feeds exactly 1")
    refused(lambda: transform(one_to_three, f, good), "output 0 has 3 channels; the Y plane is written from exactly 1")
    for other in (resnet, candy, yolo, one_to_three):
        other.close()
    # the Python wrapper's own checks
    frames = packed("nv12", y, u, v)
    with pytest.raises(ValueError):
        m.transform_luma(frames, out_format="yuyv")
    with pytest.raises(ValueError):
        m.transform_luma(frames, out_format="rgba8")
    with pytest.raises(ValueError):
        m.transform_luma(frames, out_hw=(45, 61))  # odd: the packed layout cannot hold it
    with pytest.raises(ValueError):
        m.transform_luma(frames, out_hw=(90, 120), out=torch.empty((m.batch, 60, 64), dtype=torch.uint8, device="cuda"))
