"""snnb_model_run_rois / snnb_rois_from_detections (MixedInferenceCore.run_rois, GpuContext.rois_from_detections): regions of device
frames as the batch, and regions cut from detector rows on the device.

Slot i of run_rois must be bit-identical to run_frames(format="rgba8") on the same model handle fed S_i, the region cut out of libyuv's
RGBA8 image of the whole frame (oracle/yuv.py, held to libyuv by tests/test_frames_cpu.py), in every slot. The slots without a valid
region must be all-zero bytes with class 0. rois_from_detections must equal the float32 restatement in oracle/rois.py bit for bit."""
import ctypes as C

import numpy as np
import pytest

from oracle import rois as oracle_rois
from shadernn_b200 import _lib, modelzoo
from shadernn_b200._lib import SnnbError
from test_detect_gpu import yolo_path
from test_frames_gpu import NORM, expected_rgba, host, laid_out, load, packed, random_yuv, set_params

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

FH, FW = 91, 121  # odd frames: chroma sited in frame coordinates matters at odd region origins
# {frame, row, x, y, width, height} for a 64 x 64 model, batch 8
REGIONS = [(0, 0, 1, 1, 33, 17),  # odd origin, odd size, smaller than the model
           (1, 1, 0, 0, 64, 64),  # the model's size: sampled directly
           (0, 2, FW - 80, FH - 70, 80, 70),  # larger than the model, touching the right and bottom edges
           (1, 3, 0, 0, FW, FH),  # the whole frame: touching every edge
           (0, 4, 57, 44, 1, 1),  # 1 x 1
           (1, 5, 7, 11, 64, 64),  # the model's size at an odd origin
           (0, 6, 1, 1, 33, 17),  # the same region as slot 0
           (1, 7, FW - 1, 0, 1, FH)]  # the last column


def cuda_i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda()


def frames(fmt, n=2, hw=(FH, FW), seed=7, matrix="bt601", **layout):
    """(keep-alive buffer, snnb_frames, libyuv's RGBA8 of the frames) for n frames of `fmt`."""
    y, u, v = random_yuv(n, hw[0], hw[1], seed=seed)
    rgba = expected_rgba("nv12", y, u, v, matrix)
    keep, f = laid_out(fmt, y, u, v, rgba=rgba, **layout)
    return keep, f, rgba


def outputs(m, out_dtype=None, out_layout="nhwc", want_classes=False, fill=0x5A):
    """run_torch's outputs, pre-filled with a byte pattern so that an unwritten byte shows."""
    outs, obufs, classes = m._device_outputs("test", out_dtype, out_layout, 1.0, 0.0, want_classes)
    for o in outs + ([classes] if want_classes else []):
        o.view(torch.uint8).fill_(fill)
    return outs, obufs, classes


def raw_rois(m, f, num_frames, rois, count=None, out_dtype=None, out_layout="nhwc", want_classes=False, stream=None, out=None):
    outs, obufs, classes = out if out is not None else outputs(m, out_dtype, out_layout, want_classes)
    ptr = lambda t: None if t is None else (t if isinstance(t, int) else t.data_ptr())  # noqa: E731
    _lib.check(_lib.lib().snnb_model_run_rois(m.h, C.byref(f), num_frames, ptr(rois), ptr(count), obufs, len(outs),
                                              classes.data_ptr() if want_classes else None, stream if stream is not None else m._torch_stream()),
               "snnb_model_run_rois")
    return outs, classes


def want_slots(m, rgba, regions, linear, mean4, norm4, out_dtype=None, want_classes=False):
    """Per slot i: slot i of run_frames(format="rgba8") on the same handle fed S_i (crop_rgba of libyuv's RGBA8 frames) in every slot
    that has a region of S_i's size, one call per region size. Returns (outputs [batch, ...] per model output, classes)."""
    outs, cls = None, None
    sizes = sorted({(r[5], r[4]) for r in regions})
    for hw in sizes:
        crops = [oracle_rois.crop_rgba(rgba, r) for r in regions]
        fill = next(c for c in crops if c.shape[:2] == hw)
        batch = np.stack([c if c.shape[:2] == hw else fill for c in crops] + [fill] * (m.batch - len(crops)))
        got = m.run_frames(torch.from_numpy(batch).cuda(), format="rgba8", linear=linear, mean4=mean4, norm4=norm4, out_dtype=out_dtype,
                           want_classes=want_classes)
        res, c = got if want_classes else (got, None)
        res = [host(t) for t in (res if isinstance(res, list) else [res])]
        if outs is None:
            outs, cls = [np.zeros_like(r) for r in res], (np.zeros(m.batch, np.int32) if want_classes else None)
        for i, crop in enumerate(crops):
            if crop.shape[:2] == hw:
                for o, r in zip(outs, res):
                    o[i] = r[i]
                if want_classes:
                    cls[i] = host(c)[i]
    return outs, cls


def assert_slots_equal(got, want, slots):
    for g, w in zip(got, want):
        g = host(g)
        for i in slots:
            assert np.array_equal(g[i].view(np.uint8), w[i].view(np.uint8)), "slot %d differs" % i


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("matrix", ["bt601", "bt709"])
@pytest.mark.parametrize("fmt", ["nv12", "nv21", "i420", "rgba8"])
def test_every_slot_bit_identical_to_run_frames_of_its_crop(ctx, model_dir, fmt, matrix, linear):
    m = load(ctx, model_dir, "resnet18", (64, 64), 8, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["resnet18"]
    keep, f, rgba = frames(fmt, matrix=matrix)
    got, _ = raw_rois(m, set_params(f, matrix=matrix, linear=linear, mean4=mean4, norm4=norm4), 2, cuda_i32(REGIONS))
    want, _ = want_slots(m, rgba, REGIONS, linear, mean4, norm4)
    assert_slots_equal(got, want, range(8))
    g = host(got[0])
    assert np.array_equal(g[0], g[6]) and not np.array_equal(g[0], g[2])  # two slots on one region; different regions differ


@pytest.mark.parametrize("fmt", ["nv12", "i420", "rgba8"])
def test_pitched_nvdec_planes(ctx, model_dir, fmt):
    m = load(ctx, model_dir, "resnet18", (64, 64), 8, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["resnet18"]
    keep, f, rgba = frames(fmt, n=3, seed=11, matrix="bt709", pitch_align=256, uv_row_align=16, pad_image=4096 + 3)
    regions = [(r[0] + 1,) + r[1:] for r in REGIONS]  # frames 1 and 2 of three
    got, _ = raw_rois(m, set_params(f, matrix="bt709", mean4=mean4, norm4=norm4), 3, cuda_i32(regions))
    want, _ = want_slots(m, rgba, regions, True, mean4, norm4)
    assert_slots_equal(got, want, range(8))


CONFIGS = [(name, hw, "fp32x3", fuse, graph) for name, hw in (("resnet18", (64, 64)),  # the stem reads the feed copy only
                                                                 ("mobilenetv2", (64, 64)),
                                                                 ("candy", (48, 64)))  # an image model: U8 output as well
           for fuse in (False, True) for graph in (False, True)] + [("resnet18", (64, 64), "fp16", True, True)]


@pytest.mark.parametrize("name,hw,precision,fuse,graph", CONFIGS)
def test_models_and_classes(ctx, model_dir, name, hw, precision, fuse, graph):
    batch = 8
    m = load(ctx, model_dir, name, hw, batch, fuse=fuse, use_cuda_graph=graph, precision=precision)
    mean4, norm4 = NORM[name]
    keep, f, rgba = frames("nv12", seed=len(name))
    regions = [(r[0], r[1], r[2], r[3], hw[1] if r[4] == 64 else r[4], hw[0] if r[5] == 64 else r[5]) for r in REGIONS]
    set_params(f, mean4=mean4, norm4=norm4)
    image = name == "candy"
    for dt in ([None, torch.uint8] if image else [None]):
        got, cls = raw_rois(m, f, 2, cuda_i32(regions), out_dtype=dt, want_classes=not image)
        want, want_cls = want_slots(m, rgba, regions, True, mean4, norm4, out_dtype=dt, want_classes=not image)
        assert_slots_equal(got, want, range(8))
        if not image:
            assert np.array_equal(host(cls), want_cls) and (want_cls >= 1).all()


@pytest.mark.parametrize("layout", ["nhwc", "nchw"])
def test_count_and_invalid_regions_clear_only_their_slots(ctx, model_dir, layout):
    B = 8
    m = load(ctx, model_dir, "mobilenetv2", (64, 64), B, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["mobilenetv2"]
    keep, f, rgba = frames("nv12", seed=5)
    set_params(f, mean4=mean4, norm4=norm4)
    r = cuda_i32(REGIONS)
    for dt in (torch.float32, torch.float16, torch.uint8):
        full, full_cls = raw_rois(m, f, 2, r, out_dtype=dt, out_layout=layout, want_classes=True)
        full, full_cls = host(full[0]), host(full_cls)
        assert (full_cls >= 1).all()
        for k in (None, 0, 1, B - 1, B, B + 5, -1):
            got, cls = raw_rois(m, f, 2, r, cuda_i32([k]) if k is not None else None, out_dtype=dt, out_layout=layout, want_classes=True)
            got, cls = host(got[0]), host(cls)
            used = B if k is None else min(max(k, 0), B)
            assert np.array_equal(got[:used].view(np.uint8), full[:used].view(np.uint8)), (dt, k)
            assert not got[used:].view(np.uint8).any() and not cls[used:].any(), (dt, k)
            assert np.array_equal(cls[:used], full_cls[:used])
    # invalid regions clear their own slot only
    bad = list(REGIONS)
    bad[1] = (2, 1, 0, 0, 64, 64)  # frame out of range (two frames)
    bad[2] = (-1, 2, 0, 0, 64, 64)
    bad[3] = (0, 3, -1, 0, 10, 10)  # x < 0
    bad[4] = (0, 4, FW - 9, 0, 10, 10)  # x + width > W
    bad[5] = (0, 5, 3, 3, 0, 10)  # zero width
    bad[6] = (0, 6, 3, FH - 5, 10, 6)  # y + height > H
    ok = [0, 7]
    full, full_cls = raw_rois(m, f, 2, r, out_layout=layout, want_classes=True)
    got, cls = raw_rois(m, f, 2, cuda_i32(bad), out_layout=layout, want_classes=True)
    got, cls, full, full_cls = host(got[0]), host(cls), host(full[0]), host(full_cls)
    assert np.array_equal(got[ok], full[ok]) and np.array_equal(cls[ok], full_cls[ok])
    assert not got[1:7].view(np.uint8).any() and not cls[1:7].any()


def test_rois_from_detections_of_detector_rows_equal_the_restatement(ctx, model_dir):
    for kind, seed in (("planted", 1), ("allpass", 2)):
        m = load_yolo(ctx, model_dir, kind)
        y, u, v = random_yuv(2, 240, 320, seed=seed)
        rows, counts = m.detect_frames(packed("nv12", y, u, v), mean4=NORM["yolov3tiny"][0], norm4=NORM["yolov3tiny"][1])
        hrows, hcounts = host(rows), host(counts)
        if kind == "allpass":
            assert (hcounts == 100).all()  # many rows pass
        for cap, sel in ((256, {}), (7, {}), (64, {"min_score": 0.5}), (256, {"class_id": int(hrows[0, 0, 0])}), (256, {"expand": 0.1}),
                         (256, {"expand": 0.75, "min_score": 0.4})):
            got, cnt = ctx.rois_from_detections(rows, counts, (240, 320), cap, **sel)
            want, wcnt = oracle_rois.rois_from_detections(hrows, hcounts, (240, 320), cap, **sel)
            assert int(host(cnt)[0]) == wcnt and np.array_equal(host(got), want), (kind, cap, sel)
        assert wcnt > 0


def load_yolo(ctx, model_dir, kind, batch=2):
    from shadernn_b200 import core
    return core.MixedInferenceCore(ctx, yolo_path(model_dir, kind, (416, 416)), batch=batch, input_hw=(416, 416), fuse=True, use_cuda_graph=True)


def test_rois_from_detections_of_hand_made_rows_equal_the_restatement(ctx):
    rows = [[0, 0.5, 0.25, 0.25, 0.5, 0.5], [0, 0.5, 0.875, 0.125, 0.25, 0.25], [0, 0.5, 0.75, 0.75, 0.5, 0.5], [0, 0.5, 1.25, 0.25, 0.25, 0.25],
            [0, 0.5, -0.25, 0.5, 0.5, 0.25], [0, 0.5, 0.5, 0.0, 1e30, 0.5], [0, 0.5, 0.5, 0.0, 3e38, 0.5], [0, 0.5, -3e38, 0.0, 3e38, 0.5],
            [0, 0.5, 0.5, 0.0, np.inf, 0.5], [0, 0.5, -np.inf, 0.0, np.inf, 0.5], [3, 0.5, 0.25, 0.25, 0.5, 0.5], [3, -1.0, 0.25, 0.25, 0.5, 0.5],
            [np.nan, 0.5, 0.25, 0.25, 0.5, 0.5], [0, np.nan, 0.25, 0.25, 0.5, 0.5], [0, 0.5, np.nan, 0.25, 0.5, 0.5], [0, 0.5, 0.25, 0.25, 0.5, np.nan],
            [1, 0.3, 0.1, 0.2, 0.3, 0.4], [2, 0.7, 0.33, 0.66, 0.17, 0.05], [1, 0.9, 0.999, 0.999, 0.01, 0.01], [0, 0.5, 0.25, 0.25, 0.0, 0.0]]
    rng = np.random.default_rng(3)
    rand = np.concatenate([rng.integers(0, 4, (64, 1)), rng.random((64, 1)), rng.random((64, 4)) * 1.4 - 0.2], axis=1)
    allrows = np.concatenate([np.asarray(rows, np.float64), rand]).astype(np.float32)
    hr = np.zeros((3, 40, 6), np.float32)
    hr.reshape(-1, 6)[:len(allrows)] = allrows
    for hc in (np.array([40, 40, 4], np.int32), np.array([0, 17, 100], np.int32), np.array([-3, 0, 0], np.int32)):
        for fhw in ((50, 100), (1080, 1920), (1, 1)):
            for cap, sel in ((128, {}), (5, {}), (128, {"class_id": 3}), (128, {"min_score": 0.5, "expand": 0.25}), (128, {"class_id": 1, "expand": 2.0})):
                got, cnt = ctx.rois_from_detections(torch.from_numpy(hr).cuda(), cuda_i32(hc), fhw, cap, **sel)
                want, wcnt = oracle_rois.rois_from_detections(hr, hc, fhw, cap, **sel)
                assert int(host(cnt)[0]) == wcnt and np.array_equal(host(got), want), (hc, fhw, cap, sel)


def test_chain_on_a_new_stream_equals_the_synchronised_chain(ctx, model_dir):
    det = load_yolo(ctx, model_dir, "allpass")
    cls = load(ctx, model_dir, "resnet18", (64, 64), 16, fuse=True, use_cuda_graph=True)
    dmean, dnorm = NORM["yolov3tiny"]
    mean4, norm4 = NORM["resnet18"]
    y, u, v = random_yuv(2, 240, 320, seed=17)
    src = packed("nv12", y, u, v)
    # synchronised, regions computed on the host
    rows, counts = det.detect_frames(src, mean4=dmean, norm4=dnorm)
    want_rois, want_count = oracle_rois.rois_from_detections(host(rows), host(counts), (240, 320), 16, expand=0.1)
    assert want_count == 16
    want = host(cls.run_rois(src, cuda_i32(want_rois), cuda_i32([want_count]), mean4=mean4, norm4=norm4))
    torch.cuda.synchronize()

    def chain(stream):
        with torch.cuda.stream(stream):
            torch.cuda._sleep(100_000_000)
            x = torch.empty_like(src)
            x.copy_(src)
            r, c = det.detect_frames(x, mean4=dmean, norm4=dnorm)
            rois, count = ctx.rois_from_detections(r, c, (240, 320), 16, expand=0.1)
            return cls.run_rois(x, rois, count, mean4=mean4, norm4=norm4).clone(), rois.clone()

    got, got_rois = chain(torch.cuda.Stream())
    assert np.array_equal(host(got_rois), want_rois) and np.array_equal(host(got), want)
    # run_rois between submit and wait of the same model: both results correct
    x0 = np.ascontiguousarray(modelzoo.synthetic_input("resnet18", 16, (64, 64)))
    want0, _ = cls.run(x0, want_classes=False)
    out = np.empty(cls.output_shape(0), np.float32)
    ticket = cls.submit_raw(x0.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), out.size)
    got, _ = chain(torch.cuda.Stream())
    cls.wait(ticket)
    assert np.array_equal(out, want0) and np.array_equal(host(got), want)


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")  # the refused call leaves the caller's capture empty, as it should
def test_refusals_launch_nothing_and_write_nothing(ctx, model_dir):
    m = load(ctx, model_dir, "resnet18", (64, 64), 8, fuse=True, use_cuda_graph=True)
    keep, good, rgba = frames("nv12")
    set_params(good)
    r = cuda_i32(REGIONS)
    want = host(raw_rois(m, good, 2, r)[0][0])
    out = outputs(m, want_classes=True)

    def refused(fn, text):
        before = ctx.launches
        with pytest.raises(SnnbError) as e:
            fn()
        assert text in str(e.value), str(e.value)
        assert ctx.launches == before, "a refused call launched kernels"
        assert (host(out[0][0]).view(np.uint8) == 0x5A).all() and (host(out[2]).view(np.uint8) == 0x5A).all(), "a refused call wrote"
        assert np.array_equal(host(raw_rois(m, good, 2, r)[0][0]), want)

    run = lambda f=good, n=2, rois=r, count=None, stream=None: raw_rois(m, f, n, rois, count, want_classes=True, stream=stream, out=out)  # noqa: E731
    bad = _lib.Frames.from_buffer_copy(good)
    bad.format = 4
    refused(lambda: run(f=bad), "unknown frame format 4")
    refused(lambda: run(n=0), "num_frames 0")
    refused(lambda: run(rois=None), "null rois")
    host_rois = np.asarray(REGIONS, np.int32)
    refused(lambda: run(rois=host_rois.ctypes.data), "unregistered host memory")
    pinned = torch.tensor(REGIONS, dtype=torch.int32).pin_memory()
    refused(lambda: run(rois=pinned), "pinned host memory")
    big = torch.zeros(64, dtype=torch.int32, device="cuda")
    refused(lambda: run(rois=big.data_ptr() + 2), "is not aligned to its 4-byte elements")
    refused(lambda: run(count=big.data_ptr() + 1), "count 0")
    refused(lambda: run(count=np.zeros(1, np.int32).ctypes.data), "unregistered host memory")
    g = torch.cuda.CUDAGraph()

    def capture():
        with torch.cuda.graph(g, capture_error_mode="relaxed"):
            run()
    refused(capture, "being captured")
    yolo = load_yolo(ctx, model_dir, "planted")
    yr = cuda_i32(REGIONS[:2])
    refused(lambda: raw_rois(yolo, good, 2, yr), "detection on regions is not supported")
    with pytest.raises(ValueError):
        m.run_rois(packed("nv12", *random_yuv(2, 90, 120, seed=1)), r[:4])  # rois of 4 slots, batch 8

    # rois_from_detections: rows / counts / outputs pre-filled; a refused call writes nothing
    rows = torch.rand((2, 10, 6), device="cuda")
    counts = cuda_i32([10, 10])
    rois, count = cuda_i32(np.full((8, 6), 77)), cuda_i32([77])

    def rfd(rows_p=rows.data_ptr(), counts_p=counts.data_ptr(), n=2, max_rows=10, fw=320, fh=240, sel=(0.0, -1, 0.0), cap=8, rois_p=rois.data_ptr(),
            count_p=count.data_ptr(), stream=1):
        s = None if sel is None else C.byref(_lib.RoiSelect(*sel))
        _lib.check(_lib.lib().snnb_rois_from_detections(ctx.h, rows_p, counts_p, n, max_rows, fw, fh, s, rois_p, cap, count_p, stream),
                   "snnb_rois_from_detections")

    def refused_rfd(text, **kw):
        before = ctx.launches
        with pytest.raises(SnnbError) as e:
            rfd(**kw)
        assert text in str(e.value), str(e.value)
        assert ctx.launches == before and (host(rois) == 77).all() and int(host(count)[0]) == 77

    refused_rfd("null sel", sel=None)
    refused_rfd("num_frames 0", n=0)
    refused_rfd("max_rows 0 is outside 1..100", max_rows=0)
    refused_rfd("max_rows 101 is outside 1..100", max_rows=101)
    refused_rfd("frame size 0 x 240", fw=0)
    refused_rfd("frame size 320 x -1", fh=-1)
    refused_rfd("capacity 0", cap=0)
    refused_rfd("expand -0.5", sel=(0.0, -1, -0.5))
    refused_rfd("expand inf", sel=(0.0, -1, float("inf")))
    refused_rfd("expand nan", sel=(0.0, -1, float("nan")))
    refused_rfd("rows 0: null data pointer", rows_p=None)
    refused_rfd("unregistered host memory", counts_p=np.zeros(2, np.int32).ctypes.data)
    refused_rfd("rois 0: null data pointer", rois_p=None)
    refused_rfd("is not aligned to its 4-byte elements", count_p=count.data_ptr() + 2)
    refused_rfd("pinned host memory", rows_p=torch.zeros(120).pin_memory().data_ptr())
    g2 = torch.cuda.CUDAGraph()

    def capture_rfd():
        with torch.cuda.graph(g2, capture_error_mode="relaxed"):
            rfd(stream=torch.cuda.current_stream().cuda_stream)
    before = ctx.launches
    with pytest.raises(SnnbError) as e:
        capture_rfd()
    assert "being captured" in str(e.value) and ctx.launches == before and (host(rois) == 77).all()
    rfd()  # the same arguments, valid: it runs
    assert int(host(count)[0]) == 8
    with pytest.raises(ValueError):
        ctx.rois_from_detections(rows, counts[:1], (240, 320), 8)
