"""snnb_model_detect_device / MixedInferenceCore.detect_torch: YOLO decode, stable score sort and NMS on the device.

The device rows must be the host path's rows (run() + boxes(n) on the same model handle and input): the same count per image, the
same class column and row order, scores and x, y within 1e-6, w and h within 5e-7 relative. They are not held to bit-identity: the
device takes the correctly rounded exponential where the host calls glibc's expf (snnb.h). The fixtures reach the sort and the NMS:
planted heads with scores around the threshold, all-pass heads where every cell passes and neighbours suppress each other (up to the
1024 x 1024 grid), and constant images where many scores are exactly equal, so the stable order decides."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle
from shadernn_b200 import _lib, core, modelzoo
from shadernn_b200._lib import SnnbError
from test_models_gpu import assert_same_boxes

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

_paths = {}


def yolo_path(model_dir, kind, hw):
    """YOLOv3-tiny at hw: "synthetic" (BASELINE weights), "planted" (scores scattered around 0.35) or "allpass" (objectness and class
    bias +8 for every anchor: every cell passes)."""
    key = (kind, tuple(hw))
    if key not in _paths:
        kw = {"seed": 21} if kind == "planted" else {}
        path, layers = modelzoo.build("yolov3tiny", "%s/detect_%s_%dx%d" % (model_dir, kind, hw[0], hw[1]), input_hw=hw, **kw)
        if kind != "synthetic":
            for head in [l for l in layers if l["type"] == "Conv2D" and l["outputPlanes"] == 18]:
                head["_w"]["bias"][:] = 0
                if kind == "planted":
                    head["_w"]["bias"][[4, 5, 10, 11]] = [-1.0, 0.0, -1.0, 0.0]
                else:
                    head["_w"]["bias"][[4, 5, 10, 11, 16, 17]] = 8.0
            modelzoo.write_model(layers, path, split=True)
        _paths[key] = path
    return _paths[key]


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def host_rows(m, max_rows=100):
    return [m.boxes(n, max_rows) for n in range(m.batch)]


def assert_rows_agree(rows, counts, want, what):
    """Device (rows, counts) against the host path's rows per image. Returns (bit-identical rows, rows)."""
    rows, counts = host(rows), host(counts)
    same = total = 0
    for n, ref in enumerate(want):
        k = int(counts[n])
        assert k == len(ref), "%s: image %d: %d device rows, %d host rows" % (what, n, k, len(ref))
        got = rows[n, :k]
        assert np.array_equal(got[:, 0], ref[:, 0]), (what, n)
        d = np.abs(got.astype(np.float64) - ref.astype(np.float64))
        assert float(d[:, 1:4].max(initial=0)) <= 1e-6, (what, n, float(d[:, 1:4].max()))
        assert np.all(d[:, 4:6] <= 5e-7 * np.abs(ref[:, 4:6].astype(np.float64))), (what, n, got, ref)
        assert not rows[n, k:].any(), "%s: image %d: rows past the count are not zero" % (what, n)
        same += int(np.all(got.view(np.uint32) == ref.view(np.uint32), axis=1).sum())
        total += k
    print("%s: %d of %d rows bit-identical to the host path" % (what, same, total))
    return same, total


def test_baseline_yolov3tiny_416_batch16_and_oracle(ctx, model_dir):
    # BASELINE configs[3] with its synthetic input; the first two images also against the oracle's all-CPU decode
    hw = (416, 416)
    path = yolo_path(model_dir, "synthetic", hw)
    m = core.MixedInferenceCore(ctx, path, batch=16, input_hw=hw, fuse=True, use_cuda_graph=True)
    x = modelzoo.synthetic_input("yolov3tiny", 16, hw)
    m.run(x, want_classes=False)
    want = host_rows(m)
    before = ctx.launches
    rows, counts = m.detect_torch(cuda(x))
    assert ctx.launches - before == m.launches_per_forward + 1 + 3  # input conversion, forward pass, three decode kernels
    assert rows.dtype == torch.float32 and rows.is_cuda and tuple(rows.shape) == (16, 100, 6)
    assert counts.dtype == torch.int32 and counts.is_cuda and tuple(counts.shape) == (16,)
    assert_rows_agree(rows, counts, want, "yolov3tiny 416 batch 16")
    om = oracle.Model(path)
    om.run(x[:2])
    got = host(rows)
    for n in range(2):
        assert_same_boxes(got[n, :int(host(counts)[n])], om.boxes[n][:100])


@pytest.mark.parametrize("fuse,precision", [(False, "fp32x3"), (True, "fp32x3"), (False, "fp16"), (True, "fp16")])
def test_planted_heads_match_host_path(ctx, model_dir, fuse, precision):
    hw = (416, 416)
    path = yolo_path(model_dir, "planted", hw)
    m = core.MixedInferenceCore(ctx, path, batch=4, input_hw=hw, fuse=fuse, use_cuda_graph=fuse, precision=precision)
    om = oracle.Model(path) if precision == "fp32x3" else None
    total = 0
    for seed in (1, 2, 3):
        x = modelzoo.synthetic_input("yolov3tiny", 4, hw, seed=seed)
        m.run(x, want_classes=False)
        want = host_rows(m)
        rows, counts = m.detect_torch(cuda(x))
        total += assert_rows_agree(rows, counts, want, "planted seed %d fuse=%d %s" % (seed, fuse, precision))[1]
        if om is not None:
            om.run(x)
            got, cnt = host(rows), host(counts)
            for n in range(4):
                assert_same_boxes(got[n, :int(cnt[n])], om.boxes[n][:100])
    assert total > 20, "the planted heads should produce detections"


@pytest.mark.parametrize("hw,batch", [((416, 416), 2), ((608, 608), 2), ((1024, 1024), 1)])
def test_all_pass_heads_match_host_path(ctx, model_dir, hw, batch):
    # every one of the 2535 / 5415 / 15360 cells per image passes: the longest lists, the deepest NMS
    m = core.MixedInferenceCore(ctx, yolo_path(model_dir, "allpass", hw), batch=batch, input_hw=hw, fuse=True, use_cuda_graph=True)
    x = modelzoo.synthetic_input("yolov3tiny", batch, hw)
    m.run(x, want_classes=False)
    want = host_rows(m)
    rows, counts = m.detect_torch(cuda(x))
    assert_rows_agree(rows, counts, want, "all-pass %dx%d" % hw)
    assert int(host(counts).min()) == 100  # more than 100 boxes survive NMS: the count is capped as snnb_model_get_boxes caps it


def test_constant_image_ties_keep_scan_order(ctx, model_dir):
    # a constant image gives every interior cell of a head the same six values: runs of exactly equal scores, ordered by the stable sort
    hw = (416, 416)
    m = core.MixedInferenceCore(ctx, yolo_path(model_dir, "allpass", hw), batch=2, input_hw=hw, fuse=True, use_cuda_graph=True)
    x = np.empty((2, 416, 416, 3), np.float32)
    x[0], x[1] = 0.25, 0.75
    m.run(x, want_classes=False)
    want = host_rows(m)
    for ref in want:
        assert len(np.unique(ref[:, 1])) < len(ref), "the constant image should produce equal scores"
    rows, counts = m.detect_torch(cuda(x))
    assert_rows_agree(rows, counts, want, "constant image")


def test_max_rows_truncates_in_host_order_and_zero_pads(ctx, model_dir):
    hw = (416, 416)
    m = core.MixedInferenceCore(ctx, yolo_path(model_dir, "planted", hw), batch=4, input_hw=hw, fuse=True, use_cuda_graph=True)
    x = modelzoo.synthetic_input("yolov3tiny", 4, hw, seed=2)
    m.run(x, want_classes=False)
    full = host_rows(m)
    assert max(len(r) for r in full) > 3, [len(r) for r in full]
    for max_rows in (1, 3, 100):
        rows, counts = m.detect_torch(cuda(x), max_rows=max_rows)
        assert tuple(rows.shape) == (4, max_rows, 6)
        assert_rows_agree(rows, counts, [r[:max_rows] for r in full], "max_rows %d" % max_rows)
        assert np.array_equal(host(counts), [min(len(r), max_rows) for r in full])


def _spin_write_detect(m, src, stream, **kw):
    """On `stream`: a long spin, then a torch op writes the input, then detect_torch, then torch ops read the results."""
    with torch.cuda.stream(stream):
        torch.cuda._sleep(100_000_000)
        x = torch.empty_like(src)
        x.copy_(src)
        rows, counts = m.detect_torch(x, **kw)
        return rows.clone(), counts.clone()


def test_ordering_on_the_callers_stream(ctx, model_dir):
    hw = (416, 416)
    m = core.MixedInferenceCore(ctx, yolo_path(model_dir, "planted", hw), batch=4, input_hw=hw, fuse=True, use_cuda_graph=True)
    xs = [modelzoo.synthetic_input("yolov3tiny", 4, hw, seed=s) for s in (1, 2)]
    refs = []
    for x in xs:
        m.run(x, want_classes=False)
        refs.append(host_rows(m))
    src = [cuda(x) for x in xs]
    torch.cuda.synchronize()
    m.detect_torch(src[0])  # the heads hold xs[0]; the spin delays the write of xs[1] on the new stream
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    rows, counts = _spin_write_detect(m, src[1], s1)
    assert_rows_agree(rows, counts, refs[1], "behind a spin")
    # detect_torch between submit and wait: the submission's host boxes and the device rows are both right
    x0 = np.ascontiguousarray(xs[0])  # read by the copy engine until wait()
    ticket = m.submit_raw(x0.ctypes.data_as(C.c_void_p), None, 0, None)
    rows, counts = _spin_write_detect(m, src[1], s2)
    m.wait(ticket)
    for n in range(4):
        assert np.array_equal(m.boxes(n), refs[0][n])
    assert_rows_agree(rows, counts, refs[1], "between submit and wait")


def _raw(m, bufs, n_in, rows_ptr, max_rows, counts_ptr, stream=None):
    _lib.check(_lib.lib().snnb_model_detect_device(m.h, bufs, n_in, rows_ptr, max_rows, counts_ptr, stream), "snnb_model_detect_device")


def _buf(t, offset=0):
    bufs = (_lib.DeviceBuffer * 1)()
    bufs[0].data, bufs[0].dtype, bufs[0].layout = t.data_ptr() + offset, _lib.DTYPE_F32, _lib.LAYOUT_NHWC
    return bufs


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")  # the refused call leaves the caller's capture empty, as it should
def test_refusals_launch_nothing_and_leave_the_model_usable(ctx, model_dir):
    hw = (416, 416)
    m = core.MixedInferenceCore(ctx, yolo_path(model_dir, "planted", hw), batch=4, input_hw=hw, fuse=True, use_cuda_graph=True)
    x = modelzoo.synthetic_input("yolov3tiny", 4, hw, seed=1)
    m.run(x, want_classes=False)
    want = host_rows(m)
    xd = cuda(x)
    rows = torch.empty((4, 100, 6), device="cuda")
    counts = torch.empty(4, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()

    def refused(fn, text):
        before = ctx.launches
        with pytest.raises(SnnbError) as e:
            fn()
        assert text in str(e.value), str(e.value)
        assert ctx.launches == before, "a refused call launched kernels"
        assert_rows_agree(*m.detect_torch(xd), want, "after a refusal")

    refused(lambda: m.detect_torch(torch.from_numpy(x)), "unregistered host memory")  # a host input
    refused(lambda: m.detect_torch([xd, xd]), "2 inputs given, the model has 1")
    refused(lambda: m.detect_torch(xd, max_rows=0), "max_rows 0 is outside 1..100")
    refused(lambda: m.detect_torch(xd, max_rows=101), "max_rows 101 is outside 1..100")
    refused(lambda: _raw(m, None, 1, rows.data_ptr(), 100, counts.data_ptr()), "null inputs")
    refused(lambda: _raw(m, _buf(xd), 1, None, 100, counts.data_ptr()), "rows 0: null data pointer")
    refused(lambda: _raw(m, _buf(xd), 1, rows.data_ptr(), 100, None), "counts 0: null data pointer")
    refused(lambda: _raw(m, _buf(xd), 1, rows.data_ptr() + 2, 100, counts.data_ptr()), "not aligned")
    refused(lambda: _raw(m, _buf(xd), 1, rows.data_ptr(), 100, counts.data_ptr() + 1), "not aligned")
    pinned = torch.empty((4, 100, 6)).pin_memory()
    refused(lambda: _raw(m, _buf(xd), 1, pinned.data_ptr(), 100, counts.data_ptr()), "pinned host memory")
    g = torch.cuda.CUDAGraph()

    def capture():
        with torch.cuda.graph(g, capture_error_mode="relaxed"):
            m.detect_torch(xd)
    refused(capture, "being captured")
    # a model without a YOLO output
    r_path, _ = modelzoo.build("resnet18", model_dir + "/detect_resnet18", input_hw=(64, 64))
    r = core.MixedInferenceCore(ctx, r_path, batch=2, input_hw=(64, 64))
    before = ctx.launches
    with pytest.raises(SnnbError) as e:
        r.detect_torch(cuda(modelzoo.synthetic_input("resnet18", 2, (64, 64))))
    assert "no YOLO output" in str(e.value) and ctx.launches == before
    # the host detections are not touched by any of the calls above
    for n in range(4):
        assert np.array_equal(m.boxes(n), want[n])
    # the ExceptionInfo tracebacks above keep this frame, and with it the models, alive until a garbage collection that may come
    # after the session's context is gone: release them while it exists
    m.close()
    r.close()
