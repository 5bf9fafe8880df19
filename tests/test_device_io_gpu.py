"""snnb_model_run_device / MixedInferenceCore.run_torch: device-resident inputs and outputs, ordered on the caller's stream.

The device path must compute exactly what the host paths compute for the same values (same conversion arithmetic, same stores,
same forward pass), order itself correctly on torch streams without host synchronisation, and refuse bad arguments on the host
with nothing launched."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle
from shadernn_b200 import _lib, core, modelzoo
from shadernn_b200._lib import SnnbError

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

_paths = {}


def model_path(model_dir, name, hw):
    key = (name, tuple(hw))
    if key not in _paths:
        _paths[key], _ = modelzoo.build(name, "%s/devio_%s_%dx%d" % (model_dir, name, hw[0], hw[1]), input_hw=hw)
    return _paths[key]


def load(ctx, model_dir, name, hw, batch, **kw):
    return core.MixedInferenceCore(ctx, model_path(model_dir, name, hw), batch=batch, input_hw=hw, **kw)


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


CONFIGS = [("resnet18", (64, 64), 3),  # stem reads the feed copy only (feed_only input)
           ("mobilenetv2", (64, 64), 2),
           ("candy", (48, 64), 2),  # reflect pre-pad of a 3-channel input with regular planes
           ("espcn", (32, 32), 1)]  # one channel


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("fuse", [False, True])
@pytest.mark.parametrize("name,hw,batch", CONFIGS)
def test_f32_nhwc_bit_identical_to_host_run(ctx, model_dir, name, hw, batch, fuse, graph):
    m = load(ctx, model_dir, name, hw, batch, fuse=fuse, use_cuda_graph=graph)
    x = modelzoo.synthetic_input(name, batch, hw)
    want, _ = m.run(x, want_classes=False)
    got = m.run_torch(cuda(x))
    assert got.dtype == torch.float32 and got.is_cuda and tuple(got.shape) == want.shape
    assert np.array_equal(host(got), want)


@pytest.mark.parametrize("precision", ["fp16w", "fp16"])
def test_f32_nhwc_bit_identical_reduced_precision(ctx, model_dir, precision):
    m = load(ctx, model_dir, "resnet18", (64, 64), 3, fuse=True, use_cuda_graph=True, precision=precision)
    x = modelzoo.synthetic_input("resnet18", 3, (64, 64))
    want, _ = m.run(x, want_classes=False)
    assert np.array_equal(host(m.run_torch(cuda(x))), want)


def test_input_layouts_and_dtypes_match_host_paths(ctx, model_dir):
    m = load(ctx, model_dir, "resnet18", (64, 64), 3, fuse=True, use_cuda_graph=True)
    x = modelzoo.synthetic_input("resnet18", 3, (64, 64))
    want, _ = m.run(x, want_classes=False)
    # NCHW input == the NHWC run of the same values
    assert np.array_equal(host(m.run_torch(cuda(x.transpose(0, 3, 1, 2)), layout="nchw")), want)
    # F16 input == run() fed the same values widened to fp32
    x16 = x.astype(np.float16)
    want16, _ = m.run(x16.astype(np.float32), want_classes=False)
    assert np.array_equal(host(m.run_torch(cuda(x16))), want16)
    assert np.array_equal(host(m.run_torch(cuda(x16.transpose(0, 3, 1, 2)), layout="nchw")), want16)
    # U8 with per-channel constants == snnb_model_submit_u8
    img = np.random.default_rng(4).integers(0, 256, (3, 64, 64, 3), dtype=np.uint8)
    mean4, norm4 = [10.0, 20.0, 30.0, 0.0], [0.01, 0.02, 0.03, 1.0]
    want_u8, _ = m.run_u8(img, mean4, norm4, want_classes=False)
    assert np.array_equal(host(m.run_torch(cuda(img), mean4=mean4, norm4=norm4)), want_u8)
    assert np.array_equal(host(m.run_torch(cuda(img.transpose(0, 3, 1, 2)), layout="nchw", mean4=mean4, norm4=norm4)), want_u8)


def test_output_dtypes_and_layouts(ctx, model_dir):
    m = load(ctx, model_dir, "candy", (48, 64), 2, fuse=True, use_cuda_graph=True)
    img = np.random.default_rng(6).integers(0, 256, (2, 48, 64, 3), dtype=np.uint8)
    mean4, norm4 = [0.0] * 4, [1.0] * 4
    x = cuda(img)
    ref = host(m.run_torch(x, mean4=mean4, norm4=norm4))
    assert np.array_equal(ref, m.run(img.astype(np.float32), want_classes=False)[0])
    assert float(np.abs(ref).max()) > 1.0  # a u8 output below would not be all zeros
    # F16 output == fp16 rounding of the F32 output; NCHW output == the permuted NHWC output
    f16 = host(m.run_torch(x, mean4=mean4, norm4=norm4, out_dtype=torch.float16))
    assert f16.dtype == np.float16 and np.array_equal(f16, ref.astype(np.float16))
    nchw = host(m.run_torch(x, mean4=mean4, norm4=norm4, out_layout="nchw"))
    assert np.array_equal(nchw, ref.transpose(0, 3, 1, 2))
    # U8 output == the submit_image u8 output, and == clamp(round(v * scale + offset)) of the F32 output (scale 2: v * scale is exact)
    for scale, offset in ((2.0, 12.0), (0.7, 3.0)):
        u8 = host(m.run_torch(x, mean4=mean4, norm4=norm4, out_dtype=torch.uint8, out_scale=scale, out_offset=offset))
        want_img, _ = m.run_image(img, mean4, norm4, out_u8=True, out_scale=scale, out_offset=offset)
        assert u8.dtype == np.uint8 and np.array_equal(u8, want_img)
        if scale == 2.0:
            assert np.array_equal(u8, np.clip(np.rint(ref * np.float32(scale) + np.float32(offset)), 0, 255).astype(np.uint8))
        u8_nchw = host(m.run_torch(x, mean4=mean4, norm4=norm4, out_dtype=torch.uint8, out_layout="nchw", out_scale=scale, out_offset=offset))
        assert np.array_equal(u8_nchw, u8.transpose(0, 3, 1, 2))


def test_wide_nchw_input_through_shared_memory(ctx, tmp_path):
    # more than 8 channels in NCHW take the shared-memory transpose: 70 channels = one full 64-channel tile + a partial one with
    # the zero channels [70, 72); 13 x 20 pixels = a partial 32-pixel tile
    b = modelzoo.Builder(seed=5)
    b.batchnorm(b.input(20, 13, 70), "relu")
    m = core.MixedInferenceCore(ctx, modelzoo.write_model(b.layers, str(tmp_path / "wide.json")), batch=3)
    rng = np.random.default_rng(2)
    x = rng.uniform(-2, 2, (3, 13, 20, 70)).astype(np.float32)
    want, _ = m.run(x, want_classes=False)
    assert np.array_equal(host(m.run_torch(cuda(x.transpose(0, 3, 1, 2)), layout="nchw")), want)
    x16 = x.astype(np.float16)
    assert np.array_equal(host(m.run_torch(cuda(x16.transpose(0, 3, 1, 2)), layout="nchw")), m.run(x16.astype(np.float32), want_classes=False)[0])
    img = rng.integers(0, 256, (3, 13, 20, 70), dtype=np.uint8)
    mean4, norm4 = [1.0, 2.0, 3.0, 4.0], [0.01, 0.02, 0.03, 0.04]
    want_u8, _ = m.run_u8(img, mean4, norm4, want_classes=False)
    got_u8 = host(m.run_torch(cuda(img.transpose(0, 3, 1, 2)), layout="nchw", mean4=mean4, norm4=norm4))
    assert np.array_equal(got_u8, want_u8)
    assert np.array_equal(host(m.run_torch(cuda(x), out_layout="nchw")), want.transpose(0, 3, 1, 2))


@pytest.mark.parametrize("name,hw,batch", [("resnet18", (64, 64), 3), ("mobilenetv2", (64, 64), 2)])
def test_device_classes_equal_host_classes(ctx, model_dir, name, hw, batch):
    m = load(ctx, model_dir, name, hw, batch, fuse=True, use_cuda_graph=True)
    x = modelzoo.synthetic_input(name, batch, hw)
    want, cls = m.run(x)
    out, dev_cls = m.run_torch(cuda(x), want_classes=True)
    assert dev_cls.dtype == torch.int32 and dev_cls.is_cuda
    assert np.array_equal(host(dev_cls), cls)
    assert np.array_equal(host(out), want)


def _spin_write_run_read(m, src, stream, **kw):
    """On `stream`: a long spin, then a torch op writes the input, then run_torch, then a torch op reads the output."""
    with torch.cuda.stream(stream):
        torch.cuda._sleep(100_000_000)
        x = torch.empty_like(src)
        x.copy_(src)
        out = m.run_torch(x, **kw)
        return out.clone()


def test_ordering_on_the_callers_stream(ctx, model_dir):
    r = load(ctx, model_dir, "resnet18", (64, 64), 3, fuse=True, use_cuda_graph=True)
    c = load(ctx, model_dir, "candy", (48, 64), 2, fuse=True)
    xr = [modelzoo.synthetic_input("resnet18", 3, (64, 64), seed=s) for s in (1, 2)]
    xc = [modelzoo.synthetic_input("candy", 2, (48, 64), seed=s) for s in (1, 2)]
    want_r = [r.run(x, want_classes=False)[0] for x in xr]
    want_c = [c.run(x, want_classes=False)[0] for x in xc]
    src_r, src_c = [cuda(x) for x in xr], [cuda(x) for x in xc]
    torch.cuda.synchronize()
    # one model: the tensors hold the results of xr[0]; the spin delays the write of xr[1] on the new stream
    r.run_torch(src_r[0])
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    got = _spin_write_run_read(r, src_r[1], s1)
    assert np.array_equal(host(got), want_r[1])
    # two models on two streams in flight at once
    got_r = _spin_write_run_read(r, src_r[0], s1)
    got_c = _spin_write_run_read(c, src_c[1], s2)
    assert np.array_equal(host(got_r), want_r[0])
    assert np.array_equal(host(got_c), want_c[1])
    # run_torch between submit and wait of the same model: both results correct
    out = np.empty(r.output_shape(0), np.float32)
    x0 = np.ascontiguousarray(xr[0])  # read by the copy engine until wait()
    ticket = r.submit_raw(x0.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), out.size)
    got = _spin_write_run_read(r, src_r[1], s2)
    r.wait(ticket)
    assert np.array_equal(out, want_r[0])
    assert np.array_equal(host(got), want_r[1])


def test_two_input_model(ctx, tmp_path):
    b = modelzoo.Builder(seed=3)
    a0, a1 = b.input(20, 16, 5, index=0), b.input(20, 16, 5, index=1)
    b.conv(b.add(a0, a1), 8, 3, 1, "same", "relu", bias=True)
    path = modelzoo.write_model(b.layers, str(tmp_path / "two_inputs.json"))
    m = core.MixedInferenceCore(ctx, path, batch=2)
    assert m.num_inputs == 2
    rng = np.random.default_rng(8)
    x0, x1 = rng.uniform(-1, 1, (2, 16, 20, 5)).astype(np.float32), rng.uniform(-1, 1, (2, 16, 20, 5)).astype(np.float32)
    got = host(m.run_torch([cuda(x0), cuda(x1)]))
    m.set_input(x0, 0)
    m.set_input(x1, 1)
    m.forward()
    assert np.array_equal(got, m.get_output(0))
    w = b.layers[-1]["_w"]
    want = oracle.conv2d(oracle.add(x0, x1), w["kernel"], w["bias"], stride=1, pad_x=1, pad_y=1, activation="relu", out_hw=(16, 20))
    assert float(np.abs(got - want).max()) <= 1e-4 * max(1.0, float(np.abs(want).max()))
    assert np.array_equal(host(m.run_torch([cuda(x0.transpose(0, 3, 1, 2)), cuda(x1.transpose(0, 3, 1, 2))], layout="nchw")), got)


def _raw_run(m, bufs, n_in, out=None, classes=None, stream=None):
    outs = (_lib.DeviceBuffer * 1)()
    if out is not None:
        outs[0].data, outs[0].dtype, outs[0].layout = out.data_ptr(), _lib.DTYPE_F32, _lib.LAYOUT_NHWC
    return _lib.lib().snnb_model_run_device(m.h, bufs, n_in, outs, 1 if out is not None else 0, classes, stream)


def _f32_buf(t, offset=0, dtype=_lib.DTYPE_F32, layout=_lib.LAYOUT_NHWC):
    bufs = (_lib.DeviceBuffer * 1)()
    bufs[0].data, bufs[0].dtype, bufs[0].layout = t.data_ptr() + offset, dtype, layout
    return bufs


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")  # the refused call leaves the caller's capture empty, as it should
def test_refusals_launch_nothing_and_leave_the_model_usable(ctx, model_dir):
    m = load(ctx, model_dir, "resnet18", (64, 64), 3, fuse=True, use_cuda_graph=True)
    x = modelzoo.synthetic_input("resnet18", 3, (64, 64))
    want, _ = m.run(x, want_classes=False)
    xd = cuda(x)
    out = torch.empty(m.output_shape(0), device="cuda")
    torch.cuda.synchronize()

    def refused(fn, text):
        before = ctx.launches
        with pytest.raises(SnnbError) as e:
            fn()
        assert text in str(e.value), str(e.value)
        assert ctx.launches == before, "a refused call launched kernels"
        assert np.array_equal(host(m.run_torch(xd)), want)

    def raw(*a, **kw):
        _lib.check(_raw_run(m, *a, **kw), "snnb_model_run_device")

    refused(lambda: m.run_torch(torch.from_numpy(x)), "unregistered host memory")  # a host pointer
    pinned = torch.from_numpy(x).pin_memory()
    refused(lambda: m.run_torch(pinned), "pinned host memory")
    refused(lambda: raw(_f32_buf(xd, offset=2), 1, out), "not aligned")  # F32 buffer at a 2-byte offset
    refused(lambda: m.run_torch([xd, xd]), "2 inputs given, the model has 1")
    refused(lambda: raw(_f32_buf(xd, dtype=7), 1, out), "unknown dtype 7")
    refused(lambda: raw(_f32_buf(xd, layout=5), 1, out), "unknown layout 5")
    refused(lambda: raw(None, 1, out), "null inputs")
    refused(lambda: raw(_f32_buf(xd), 1, out, classes=out.data_ptr() + 1), "not aligned")
    # the caller's stream is being captured
    g = torch.cuda.CUDAGraph()

    def capture():
        with torch.cuda.graph(g, capture_error_mode="relaxed"):
            m.run_torch(xd)
    refused(capture, "being captured")
    # classes from a model that is not a classifier
    c = load(ctx, model_dir, "candy", (48, 64), 2)
    before = ctx.launches
    with pytest.raises(SnnbError) as e:
        c.run_torch(cuda(modelzoo.synthetic_input("candy", 2, (48, 64))), want_classes=True)
    assert "not a classifier" in str(e.value) and ctx.launches == before
    # a detection model
    y = load(ctx, model_dir, "yolov3tiny", (416, 416), 1)
    before = ctx.launches
    with pytest.raises(SnnbError) as e:
        y.run_torch(cuda(modelzoo.synthetic_input("yolov3tiny", 1, (416, 416))))
    assert "snnb_model_get_boxes" in str(e.value) and ctx.launches == before
    assert np.array_equal(host(m.run_torch(xd)), want)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_buffer_on_another_gpu_is_refused(ctx, model_dir):
    m = load(ctx, model_dir, "resnet18", (64, 64), 3)
    x = modelzoo.synthetic_input("resnet18", 3, (64, 64))
    before = ctx.launches
    with pytest.raises(SnnbError) as e:
        m.run_torch(torch.from_numpy(x).to("cuda:1"))
    assert "of device 1" in str(e.value) and ctx.launches == before
