"""Partial batches (snnb_model_set_batch, MixedInferenceCore.set_batch): a model loaded for B images runs any batch n <= B on every entry
point. The oracle is a second model on the same context, loaded from the same file with the same options at batch n: every result of the
batch-B model after set_batch(n) must be bit-identical to that model's, because the same kernels run with the same plans on the same
extents. Also: switching back and forth reproduces the first results, only n images of a caller's buffer are touched, submitted tickets
keep their batch, the n-image plan is the one launched, and refused calls launch and write nothing."""
import ctypes as C

import numpy as np
import pytest

from shadernn_b200 import _lib, core
from shadernn_b200._lib import SnnbError
from test_detect_gpu import yolo_path
from test_frame_list_out_gpu import candy
from test_frames_gpu import load
from test_luma_gpu import espcn
from test_rois_gpu import cuda_i32
from test_segment_gpu import unet

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

MEAN4, NORM4 = (127.5,) * 4, (1 / 127.5,) * 4
SIZES = [(72, 96), (90, 120), (64, 64), (40, 36), (120, 160), (32, 18), (64, 64), (62, 66)]  # frame sizes of the lists


def batches(b):
    return sorted({1, 3, b - 1, b})


def np_of(v):
    if isinstance(v, torch.Tensor):
        torch.cuda.synchronize()
        return v.cpu().numpy()
    if isinstance(v, (list, tuple)):
        return [np_of(x) for x in v]
    return v


def assert_identical(got, want, what):
    if isinstance(want, (list, tuple)):
        assert isinstance(got, (list, tuple)) and len(got) == len(want), what
        for i, (g, w) in enumerate(zip(got, want)):
            assert_identical(g, w, "%s[%d]" % (what, i))
        return
    if want is None:
        assert got is None, what
        return
    g, w = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert g.shape == w.shape and g.dtype == w.dtype, (what, g.shape, w.shape)
    assert g.tobytes() == w.tobytes(), "%s: %d of %d bytes differ" % (what, int((g.view(np.uint8) != w.view(np.uint8)).sum()), g.nbytes)


def nv12(h, w, seed, n=None):
    g = torch.Generator().manual_seed(seed)
    shape = (h * 3 // 2, w) if n is None else (n, h * 3 // 2, w)
    return torch.randint(0, 256, shape, dtype=torch.uint8, generator=g).cuda()


def compare(make, b, results, **kw):
    """results(m, n) on the batch-b model after set_batch(n) against a model loaded at n, for every n of batches(b); returns the first."""
    big = make(b, **kw)
    first = None
    for n in batches(b):
        big.set_batch(n)
        assert big.batch == n and big.max_batch == b and big.input_shape(0)[0] == n and big.layer_info(0)[2][0] == n
        got = results(big, n)
        small = make(n, **kw)
        want = results(small, n)
        assert_identical(got, want, "n=%d" % n)
        assert big.launches_per_forward == small.launches_per_forward, n
        small.close()
        first = first or got
    big.close()
    return first


# ---- ResNet-18 (B = 8): every classifier entry point, fused or not, graph or not, in each product form --------------------------------
R_HW, R_B = (64, 64), 8
R_X = np.random.default_rng(5).uniform(-1, 1, (R_B,) + R_HW + (3,)).astype(np.float32)
R_U8 = np.random.default_rng(6).integers(0, 256, (R_B,) + R_HW + (3,), dtype=np.uint8)


def resnet_results(m, n):
    frames = nv12(90, 120, 1, n=R_B)
    flist = [nv12(h, w, 10 + i) for i, (h, w) in enumerate(SIZES)]
    rois = cuda_i32([(i % R_B, i, i, 2 * i, 40 + i, 30 + 2 * i) for i in range(n)])
    r = {}
    r["run"] = m.run(R_X[:n])
    r["submit_u8"] = m.run_u8(R_U8[:n], MEAN4, NORM4)
    xt = torch.from_numpy(R_X[:n]).cuda()
    r["torch_f32"] = np_of(m.run_torch(xt, want_classes=True))
    r["torch_u8"] = np_of(m.run_torch(torch.from_numpy(R_U8[:n]).cuda(), mean4=MEAN4, norm4=NORM4, out_dtype=torch.uint8, out_scale=50.0,
                                      out_offset=128.0, want_classes=True))
    r["frames"] = np_of(m.run_frames(frames[:n], mean4=MEAN4, norm4=NORM4, want_classes=True))
    r["frame_list"] = np_of(m.run_frame_list(flist[:n], mean4=MEAN4, norm4=NORM4, want_classes=True))
    for k in (n + 2, n // 2):
        r["rois%d" % k] = np_of(m.run_rois(frames, rois, cuda_i32([k]), mean4=MEAN4, norm4=NORM4, want_classes=True))
        r["rois_list%d" % k] = np_of(m.run_rois_list(flist, rois, cuda_i32([k]), mean4=MEAN4, norm4=NORM4, want_classes=True))
    return [r[k] for k in sorted(r)]


@pytest.mark.parametrize("precision", ["fp32x3", "fp16w", "fp16"])
@pytest.mark.parametrize("fuse,graph", [(False, False), (False, True), (True, False), (True, True)])
def test_resnet18_every_entry_point_equals_a_model_loaded_at_n(ctx, model_dir, fuse, graph, precision):
    compare(lambda b, **kw: load(ctx, model_dir, "resnet18", R_HW, b, **kw), R_B, resnet_results, fuse=fuse, use_cuda_graph=graph,
            precision=precision)


# ---- YOLOv3-tiny (B = 4): host boxes, device detections, frames and frame lists ---------------------------------------------------
def test_yolov3tiny_detections_equal_a_model_loaded_at_n(ctx, model_dir):
    x = np.random.default_rng(7).uniform(-1, 1, (4, 416, 416, 3)).astype(np.float32)
    frames = nv12(540, 960, 2, n=4)
    flist = [nv12(h, w, 20 + i) for i, (h, w) in enumerate([(540, 960), (720, 1280), (416, 416), (300, 500)])]

    def results(m, n):
        m.run(x[:n], want_classes=False)
        boxes = [m.boxes(i) for i in range(n)]
        with pytest.raises(SnnbError):
            m.boxes(n)
        return [boxes, np_of(m.detect_torch(torch.from_numpy(x[:n]).cuda())), np_of(m.detect_frames(frames[:n], mean4=MEAN4, norm4=NORM4)),
                np_of(m.detect_frame_list(flist[:n], mean4=MEAN4, norm4=NORM4))]
    path = yolo_path(model_dir, "planted", (416, 416))
    first = compare(lambda b, **kw: core.MixedInferenceCore(ctx, path, batch=b, input_hw=(416, 416), **kw), 4, results, fuse=True,
                    use_cuda_graph=True)
    assert sum(len(b) for b in first[0]) > 0  # the planted scores give detections to compare


# ---- image models: Candy (InstanceNorm, whose chunking depends on n), ESPCN (luma), U-Net (labels) -------------------------------
def test_candy_transforms_equal_a_model_loaded_at_n(ctx, model_dir):
    frames = nv12(90, 120, 3, n=4)
    flist = [nv12(h, w, 30 + i) for i, (h, w) in enumerate(SIZES[:4])]
    compare(lambda b, **kw: candy(ctx, model_dir, b, **kw), 4,
            lambda m, n: [np_of(m.transform_frames(frames[:n], out_format="nv12", out_hw=(50, 70))),
                          np_of(m.transform_frame_list(flist[:n], out_format="nv12"))], fuse=True, use_cuda_graph=True)


def test_espcn_luma_equals_a_model_loaded_at_n(ctx, model_dir):
    frames = nv12(48, 80, 4, n=4)
    flist = [nv12(h, w, 40 + i) for i, (h, w) in enumerate(SIZES[:4])]
    compare(lambda b, **kw: espcn(ctx, model_dir, hw=(24, 40), batch=b, **kw), 4,
            lambda m, n: [np_of(m.transform_luma(frames[:n].clone())), np_of(m.transform_luma_list([f.clone() for f in flist[:n]]))])


@pytest.mark.parametrize("classes", [1, 21])
def test_unet_labels_equal_a_model_loaded_at_n(ctx, model_dir, classes):
    frames = nv12(90, 120, 5, n=4)
    flist = [nv12(h, w, 50 + i) for i, (h, w) in enumerate(SIZES[:4])]
    compare(lambda b, **kw: unet(ctx, model_dir, (64, 64), classes, b, **kw), 4,
            lambda m, n: [np_of(m.segment_frames(frames[:n], luma=True, out_hw=(91, 121))), np_of(m.segment_frame_list(flist[:n], luma=True))],
            fuse=True, use_cuda_graph=True)


# ---- switching, tickets, the launched plan, untouched bytes, refusals -----------------------------------------------------------
def test_switching_back_and_forth_reproduces_the_first_results(ctx, model_dir):
    m = load(ctx, model_dir, "resnet18", R_HW, R_B, fuse=True, use_cuda_graph=True)
    seen, launches = {}, {}
    for n in (R_B, 1, R_B, 3, 1, 3, R_B):
        m.set_batch(n)
        got = resnet_results(m, n)
        if n in seen:
            assert_identical(got, seen[n], "n=%d again" % n)
            assert m.launches_per_forward == launches[n]
        seen[n], launches[n] = got, m.launches_per_forward
    m.close()


def test_tickets_keep_the_batch_they_were_submitted_with(ctx, model_dir):
    m = load(ctx, model_dir, "resnet18", R_HW, R_B, fuse=True, use_cuda_graph=True)
    two = load(ctx, model_dir, "resnet18", R_HW, 2, fuse=True, use_cuda_graph=True)
    want_b, want_2 = m.run_u8(R_U8, MEAN4, NORM4), two.run_u8(R_U8[:2], MEAN4, NORM4)
    oshape = (R_B,) + m.output_shape(0)[1:]
    out_b, out_2 = np.full(oshape, -7.0, np.float32), np.full(oshape, -7.0, np.float32)
    cls_b, cls_2 = (C.c_int * R_B)(*[-5] * R_B), (C.c_int * R_B)(*[-5] * R_B)
    u8 = np.ascontiguousarray(R_U8)
    t0 = m.submit_u8_raw(u8.ctypes.data, MEAN4, NORM4, out_b.ctypes.data, out_b.size, cls_b)
    m.set_batch(2)
    t1 = m.submit_u8_raw(u8.ctypes.data, MEAN4, NORM4, out_2.ctypes.data, out_b.size, cls_2)
    m.wait(t0)
    m.wait(t1)
    assert_identical(out_b, want_b[0], "ticket at B")
    assert list(cls_b) == list(want_b[1])
    assert_identical(out_2[:2], want_2[0], "ticket at 2")
    assert list(cls_2)[:2] == list(want_2[1]) and list(cls_2)[2:] == [-5] * (R_B - 2)
    assert (out_2[2:] == -7.0).all()
    m.close(), two.close()


def test_one_image_runs_its_own_plan(ctx, model_dir):
    # ResNet-18 224 x 224 at B = 32: the last 7 x 7 x 512 convolution takes 64-channel tiles unsplit at 32 images and 32-channel tiles in
    # four K pieces at one (tests/test_partial_batch_cpu.py). Fused, the classifier head is one pool + Dense kernel, so the last
    # convolution a time_layers pass launches is that layer.
    import test_conv_plan as cp
    m = load(ctx, model_dir, "resnet18", (224, 224), 32, fuse=True)
    last = max(i for i in range(m.num_layers) if m.layer_info(i)[1] == "Conv2D")
    assert m.layer_info(last)[2][1:] == (7, 7, 512)
    for n in (32, 1, 32):
        m.set_batch(n)
        m.time_layers()
        want = cp.plan((7, 7, 512), (7, 7, 512), 3, 1, 1, 1, pad_mode=cp.PAD_NONE, n=n, sms=torch.cuda.get_device_properties(0).multi_processor_count)
        # the record of the most recent convolution launch: the model's last convolution
        assert ctx.last_conv_variant()["n_blk"] == want["n_blk"] and ctx.last_conv_variant()["ksplit"] == want["ksplit"], n
    m.close()


def test_only_n_images_of_a_caller_buffer_are_touched(ctx, model_dir):
    m = load(ctx, model_dir, "resnet18", R_HW, R_B, fuse=True, use_cuda_graph=True)
    lib, n = _lib.lib(), 3
    m.set_batch(n)
    x = torch.from_numpy(R_X).cuda()  # B images: only the first n may be read
    out = torch.full((R_B,) + m.output_shape(0)[1:], -7.0, device="cuda")
    cls = torch.full((R_B,), -5, dtype=torch.int32, device="cuda")
    ins, outs = (_lib.DeviceBuffer * 1)(), (_lib.DeviceBuffer * 1)()
    ins[0].data, ins[0].dtype, ins[0].layout = x.data_ptr(), _lib.DTYPE_F32, _lib.LAYOUT_NHWC
    outs[0].data, outs[0].dtype, outs[0].layout = out.data_ptr(), _lib.DTYPE_F32, _lib.LAYOUT_NHWC
    _lib.check(lib.snnb_model_run_device(m.h, ins, 1, outs, 1, cls.data_ptr(), None), "run_device")
    want, wcls = m.run_torch(x[:n], want_classes=True)
    assert_identical(np_of(out[:n]), np_of(want), "outputs")
    assert_identical(np_of(cls[:n]), np_of(wcls), "classes")
    assert (np_of(out[n:]) == -7.0).all() and (np_of(cls[n:]) == -5).all()
    # frames out and labels: B-image destinations, sentinels past image n - 1
    c = candy(ctx, model_dir, 4, fuse=True, use_cuda_graph=True)
    c.set_batch(2)
    frames = nv12(48, 64, 8, n=4)
    dst = torch.full((4, 72, 64), 0xA5, dtype=torch.uint8, device="cuda")
    c.transform_frames(frames[:2], out_format="nv12", out=dst[:2])
    assert (np_of(dst[2:]) == 0xA5).all() and not (np_of(dst[:2]) == 0xA5).all()
    u = unet(ctx, model_dir, (64, 64), 21, 4, fuse=True)
    u.set_batch(1)
    labels = torch.full((4, 48, 64), 0xA5, dtype=torch.uint8, device="cuda")
    u.segment_frames(frames[:1], luma=True, out=labels[:1])
    assert (np_of(labels[1:]) == 0xA5).all()
    # detections: rows and counts of B images
    y = core.MixedInferenceCore(ctx, yolo_path(model_dir, "planted", (416, 416)), batch=4, input_hw=(416, 416), fuse=True, use_cuda_graph=True)
    y.set_batch(2)
    rows = torch.full((4, 100, 6), -3.0, device="cuda")
    counts = torch.full((4,), -9, dtype=torch.int32, device="cuda")
    yin = torch.from_numpy(np.random.default_rng(9).uniform(-1, 1, (4, 416, 416, 3)).astype(np.float32)).cuda()
    ins[0].data = yin.data_ptr()
    _lib.check(lib.snnb_model_detect_device(y.h, ins, 1, rows.data_ptr(), 100, counts.data_ptr(), None), "detect_device")
    assert (np_of(rows[2:]) == -3.0).all() and (np_of(counts[2:]) == -9).all()
    for mm in (m, c, u, y):
        mm.close()


def test_refusals_launch_and_write_nothing(ctx, model_dir):
    m = load(ctx, model_dir, "resnet18", R_HW, R_B, fuse=True, use_cuda_graph=True)
    m.set_batch(3)
    before = ctx.launches
    for bad in (0, R_B + 1, -1):
        with pytest.raises(SnnbError) as e:
            m.set_batch(bad)
        assert "snnb_model_set_batch: batch %d; the model was loaded for 1 to %d images" % (bad, R_B) in str(e.value)
        assert m.batch == 3 and m.input_shape(0)[0] == 3
    fl, images = m._frame_list("t", [nv12(64, 64, i) for i in range(4)], "nv12", "bt601", True, None, None)
    out = torch.full((R_B,) + m.output_shape(0)[1:], -7.0, device="cuda")
    outs = (_lib.DeviceBuffer * 1)()
    outs[0].data, outs[0].dtype, outs[0].layout = out.data_ptr(), _lib.DTYPE_F32, _lib.LAYOUT_NHWC
    assert _lib.lib().snnb_model_run_frame_list(m.h, C.byref(fl), outs, 1, None, None) != 0
    assert b"count 4; the list must hold the model's batch of 3 images" in _lib.lib().snnb_last_error()
    with pytest.raises(ValueError, match="the model takes"):
        m.run_torch(torch.from_numpy(R_X[:4]).cuda())
    assert ctx.launches == before
    assert (np_of(out) == -7.0).all()
    m.close()
