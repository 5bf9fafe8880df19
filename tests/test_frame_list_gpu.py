"""Frame lists (snnb_model_run_frame_list / detect_frame_list / run_rois_list, snnb_rois_from_detections_list; MixedInferenceCore.
run_frame_list / detect_frame_list / run_rois_list, GpuContext.rois_from_detections with per-frame sizes): a batch of separately
allocated device frames of mixed sizes, pitches and matrices, one descriptor per image.

Slot i of a list must be bit-identical to slot i of run_frames / detect_frames on the same handle fed a batch whose every frame is
image i: that batch is image i's own planes with an image stride of 0, so the reference path reads exactly the bytes the list names.
Regions must be bit-identical to run_frames(format="rgba8") fed the crop of their own frame (oracle/yuv.py's RGBA8, held to libyuv by
tests/test_frames_cpu.py), and rois_from_detections_list to the float32 restatement in tests/test_frame_list_cpu.py (oracle/rois.py's, with a size per frame)."""
import ctypes as C

import numpy as np
import pytest

from oracle import rois as oracle_rois
from shadernn_b200 import _lib, core, modelzoo
from shadernn_b200._lib import SnnbError
from test_frame_list_cpu import rois_from_detections_list
from test_frames_gpu import NORM, expected_rgba, host, laid_out, load, random_yuv
from test_p010_gpu import MATRIX_IDS, laid_out10, random_yuv10
from test_rois_gpu import CONFIGS, cuda_i32, load_yolo, outputs

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

MATRICES = ["bt601", "bt709", "bt2020", "jpeg"]
# (H, W, pitch alignment) of the 8 images of a 64 x 64 model's list: the model's size (sampled directly), odd, larger, smaller, 1 x 1
SIZES = [(64, 64, 1), (91, 121, 256), (100, 90, 64), (1, 1, 1), (40, 36, 128), (33, 17, 32), (64, 64, 512), (63, 65, 1)]


def image(fmt, h, w, seed, pitch_align=1):
    """One frame in its own device buffer at its own pitch: (the buffer, which must stay alive, its one-image snnb_frames)."""
    if fmt == "p010":
        return laid_out10(*random_yuv10(1, h, w, seed), pitch_align=pitch_align)
    y, u, v = random_yuv(1, h, w, seed)
    return laid_out(fmt, y, u, v, pitch_align=pitch_align, rgba=expected_rgba("nv12", y, u, v, "bt601"))


def frame_list(fmt, frames, matrices, linear=True, mean4=(0.0,) * 4, norm4=(1.0,) * 4):
    """The snnb_frame_list of one-image snnb_frames; returns (the list, its descriptor array, which must stay alive)."""
    images = (_lib.FrameImage * max(1, len(frames)))()
    for i, (f, m) in enumerate(zip(frames, matrices)):
        images[i].plane, images[i].pitch = f.plane, f.pitch
        images[i].width, images[i].height, images[i].matrix = f.width, f.height, MATRIX_IDS[m]
    fl = _lib.FrameList()
    fl.format, fl.count, fl.images, fl.linear_filter = (_lib.FRAME_P010 if fmt == "p010" else {"nv12": 0, "nv21": 1, "i420": 2, "rgba8": 3}[fmt]), len(frames), \
        images, int(bool(linear))
    fl.mean4 = (C.c_float * 4)(*mean4)
    fl.norm4 = (C.c_float * 4)(*norm4)
    return fl, images


def repeated(f, matrix, linear, mean4, norm4):
    """snnb_frames of a batch whose every image is the one image of f: its planes with an image stride of 0."""
    g = _lib.Frames.from_buffer_copy(f)
    for p in range(3):
        g.image_stride[p] = 0
    g.matrix, g.linear_filter = MATRIX_IDS[matrix], int(bool(linear))
    g.mean4 = (C.c_float * 4)(*mean4)
    g.norm4 = (C.c_float * 4)(*norm4)
    return g


def run_list(m, fl, out_dtype=None, out_layout="nhwc", want_classes=False, out=None, stream=None):
    outs, obufs, classes = out if out is not None else m._device_outputs("test", out_dtype, out_layout, 1.0, 0.0, want_classes)
    _lib.check(_lib.lib().snnb_model_run_frame_list(m.h, C.byref(fl), obufs, len(outs), classes.data_ptr() if want_classes else None,
                                                    stream if stream is not None else m._torch_stream()), "snnb_model_run_frame_list")
    return outs, classes


def run_frames(m, f, out_dtype=None, want_classes=False):
    outs, obufs, classes = m._device_outputs("test", out_dtype, "nhwc", 1.0, 0.0, want_classes)
    _lib.check(_lib.lib().snnb_model_run_frames(m.h, C.byref(f), obufs, len(outs), classes.data_ptr() if want_classes else None, m._torch_stream()),
               "snnb_model_run_frames")
    return outs, classes


def assert_slot_i_is_run_frames_of_image_i(m, fmt, frames, matrices, linear, mean4, norm4, out_dtype=None, want_classes=False):
    fl, keep = frame_list(fmt, frames, matrices, linear, mean4, norm4)
    got, cls = run_list(m, fl, out_dtype=out_dtype, want_classes=want_classes)
    got = [host(o) for o in got]
    for i, (f, mat) in enumerate(zip(frames, matrices)):
        want, wcls = run_frames(m, repeated(f, mat, linear, mean4, norm4), out_dtype=out_dtype, want_classes=want_classes)
        for g, w in zip(got, want):
            assert np.array_equal(g[i].view(np.uint8), host(w)[i].view(np.uint8)), "slot %d differs" % i
        if want_classes:
            assert host(cls)[i] == host(wcls)[i] >= 1
    return got


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("fmt", ["nv12", "nv21", "i420", "rgba8", "p010"])
def test_slot_i_equals_run_frames_of_image_i(ctx, model_dir, fmt, linear):
    m = load(ctx, model_dir, "resnet18", (64, 64), 8, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["resnet18"]
    made = [image(fmt, h, w, seed=10 + i, pitch_align=a) for i, (h, w, a) in enumerate(SIZES)]
    frames = [f for _, f in made]
    got = assert_slot_i_is_run_frames_of_image_i(m, fmt, frames, [MATRICES[i % 4] for i in range(8)], linear, mean4, norm4)
    assert not np.array_equal(got[0][0], got[0][6])  # the two 64 x 64 images differ, and so do their slots


@pytest.mark.parametrize("name,hw,precision,fuse,graph", CONFIGS)
def test_models_and_classes(ctx, model_dir, name, hw, precision, fuse, graph):
    m = load(ctx, model_dir, name, hw, 8, fuse=fuse, use_cuda_graph=graph, precision=precision)
    mean4, norm4 = NORM[name]
    sizes = [hw + (1,)] + SIZES[1:]
    made = [image("nv12", h, w, seed=len(name) + i, pitch_align=a) for i, (h, w, a) in enumerate(sizes)]
    image_model = name == "candy"
    for dt in ([None, torch.uint8] if image_model else [None]):
        assert_slot_i_is_run_frames_of_image_i(m, "nv12", [f for _, f in made], [MATRICES[(i + 1) % 4] for i in range(8)], True, mean4, norm4,
                                               out_dtype=dt, want_classes=not image_model)


def test_python_wrapper_takes_one_tensor_per_frame(ctx, model_dir):
    m = load(ctx, model_dir, "mobilenetv2", (64, 64), 3, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["mobilenetv2"]
    from test_frames_gpu import packed
    ts, want = [], []
    for i, (h, w) in enumerate([(64, 64), (90, 120), (36, 40)]):
        y, u, v = random_yuv(1, h, w, seed=40 + i)
        t = packed("i420", y, u, v)
        ts.append(t[0])
        want.append(host(m.run_frames(t.expand(3, -1, -1), format="i420", matrix=MATRICES[i], mean4=mean4, norm4=norm4))[i])
    got = host(m.run_frame_list(ts, format="i420", matrix=MATRICES[:3], mean4=mean4, norm4=norm4))
    for i in range(3):
        assert np.array_equal(got[i], want[i])
    with pytest.raises(ValueError):
        m.run_frame_list(ts[:2], format="i420")  # 2 frames, batch 3
    with pytest.raises(ValueError):
        m.run_frame_list(ts, format="i420", matrix=["bt601"] * 2)  # one matrix per frame, or one name


def test_detect_frame_list_equals_detect_frames_per_image(ctx, model_dir):
    det = load_yolo(ctx, model_dir, "allpass", batch=4)
    mean4, norm4 = NORM["yolov3tiny"]
    made = [image("nv12", h, w, seed=60 + i, pitch_align=a) for i, (h, w, a) in enumerate([(416, 416, 1), (240, 320, 256), (91, 121, 1), (480, 640, 64)])]
    mats = ["bt601", "bt709", "jpeg", "bt2020"]
    fl, keep = frame_list("nv12", [f for _, f in made], mats, True, mean4, norm4)
    rows = torch.empty((4, 100, 6), dtype=torch.float32, device="cuda")
    counts = torch.empty(4, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().snnb_model_detect_frame_list(det.h, C.byref(fl), rows.data_ptr(), 100, counts.data_ptr(), det._torch_stream()),
               "snnb_model_detect_frame_list")
    hr, hc = host(rows), host(counts)
    assert (hc == 100).all()
    for i, ((_, f), mat) in enumerate(zip(made, mats)):
        r2 = torch.empty_like(rows)
        c2 = torch.empty_like(counts)
        _lib.check(_lib.lib().snnb_model_detect_frames(det.h, C.byref(repeated(f, mat, True, mean4, norm4)), r2.data_ptr(), 100, c2.data_ptr(),
                                                       det._torch_stream()), "snnb_model_detect_frames")
        assert host(c2)[i] == hc[i] and np.array_equal(host(r2)[i].view(np.uint32), hr[i].view(np.uint32)), "image %d" % i


# three frames of different sizes (H, W) and matrices; regions on a 64 x 64 model, batch 8
RFRAMES = [(91, 121, "bt601"), (60, 200, "bt709"), (150, 80, "bt601")]
RREGIONS = [(0, 0, 1, 1, 33, 17),  # odd origin and size
            (1, 1, 130, 3, 64, 56),  # only inside frame 1 (200 wide)
            (2, 2, 5, 70, 75, 80),  # touching frame 2's bottom edge
            (1, 3, 0, 0, 200, 60),  # the whole of frame 1
            (2, 4, 7, 11, 64, 64),  # the model's size: sampled directly
            (0, 5, 120, 90, 1, 1),  # frame 0's last pixel
            (0, 6, 130, 3, 64, 56),  # region 1's rectangle on frame 0 (121 wide): valid only against the larger frame -> cleared
            (2, 7, 0, 0, 80, 150)]  # the whole of frame 2
INVALID = [6]


def region_frames(fmt="nv12", seed=80):
    made, rgba = [], []
    for i, (h, w, mat) in enumerate(RFRAMES):
        y, u, v = random_yuv(1, h, w, seed + i)
        rgba.append(expected_rgba(fmt if fmt != "rgba8" else "nv12", y, u, v, mat)[0])
        made.append(laid_out(fmt, y, u, v, pitch_align=64 * (i + 1), rgba=rgba[-1][None]))
    return made, rgba


def run_rois_list(m, fl, regions, count=None, out_dtype=None, out_layout="nhwc", want_classes=False, out=None, stream=None):
    outs, obufs, classes = out if out is not None else outputs(m, out_dtype, out_layout, want_classes)
    ptr = lambda t: None if t is None else (t if isinstance(t, int) else t.data_ptr())  # noqa: E731
    _lib.check(_lib.lib().snnb_model_run_rois_list(m.h, C.byref(fl), ptr(regions), ptr(count), obufs, len(outs), classes.data_ptr() if want_classes else None,
                                                   stream if stream is not None else m._torch_stream()), "snnb_model_run_rois_list")
    return outs, classes


def want_region_slots(m, rgba, regions, mean4, norm4, out_dtype=None, out_layout="nhwc"):
    """Per valid slot i: slot i of run_frames(format="rgba8") fed a batch of S_i, the crop of its own frame. Invalid slots: zero."""
    want, wcls = None, np.zeros(m.batch, np.int32)
    for i, r in enumerate(regions):
        if i in INVALID:
            continue
        crop = oracle_rois.crop_rgba(rgba[r[0]], r)
        got, cls = m.run_frames(torch.from_numpy(np.stack([crop] * m.batch)).cuda(), format="rgba8", mean4=mean4, norm4=norm4, out_dtype=out_dtype,
                                out_layout=out_layout, want_classes=True)
        got = host(got)
        if want is None:
            want = np.zeros_like(got)
        want[i], wcls[i] = got[i], host(cls)[i]
    return want, wcls


@pytest.mark.parametrize("layout", ["nhwc", "nchw"])
def test_regions_of_frames_of_mixed_sizes(ctx, model_dir, layout):
    B = 8
    m = load(ctx, model_dir, "mobilenetv2", (64, 64), B, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["mobilenetv2"]
    made, rgba = region_frames()
    fl, keep = frame_list("nv12", [f for _, f in made], [mat for _, _, mat in RFRAMES], True, mean4, norm4)
    r = cuda_i32(RREGIONS)
    want, wcls = want_region_slots(m, rgba, RREGIONS, mean4, norm4, out_layout=layout)
    got, cls = run_rois_list(m, fl, r, out_layout=layout, want_classes=True)
    got, cls = host(got[0]), host(cls)
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8)) and np.array_equal(cls, wcls)
    assert not got[INVALID].view(np.uint8).any() and (wcls[[i for i in range(B) if i not in INVALID]] >= 1).all()
    for k in (0, 3, B, -1):
        g, c = run_rois_list(m, fl, r, cuda_i32([k]), out_layout=layout, want_classes=True)
        g, c = host(g[0]), host(c)
        used = min(max(k, 0), B)
        assert np.array_equal(g[:used].view(np.uint8), got[:used].view(np.uint8)) and np.array_equal(c[:used], cls[:used]), k
        assert not g[used:].view(np.uint8).any() and not c[used:].any(), k


@pytest.mark.parametrize("fmt", ["nv12", "nv21", "i420", "rgba8", "p010"])
def test_rois_list_of_equal_frames_equals_run_rois(ctx, model_dir, fmt):
    # the images of one laid-out batch named one by one: every format through the list's region kernel and its clear kernel
    m = load(ctx, model_dir, "resnet18", (64, 64), 8, fuse=True, use_cuda_graph=True)
    mean4, norm4 = NORM["resnet18"]
    if fmt == "p010":
        keep, f = laid_out10(*random_yuv10(2, 91, 121, 5), pitch_align=128)
    else:
        y, u, v = random_yuv(2, 91, 121, 5)
        keep, f = laid_out(fmt, y, u, v, pitch_align=128, rgba=expected_rgba("nv12", y, u, v, "bt601"))
    frames = []
    for n in range(2):
        g = _lib.Frames.from_buffer_copy(f)
        for p in range(3):
            g.plane[p] = (f.plane[p] or 0) + n * f.image_stride[p] if f.plane[p] else None
        frames.append(g)
    regions = [(0, 0, 1, 1, 33, 17), (1, 1, 0, 0, 64, 64), (0, 2, 41, 21, 80, 70), (1, 3, 0, 0, 121, 91), (0, 4, 57, 44, 1, 1), (1, 5, 7, 11, 64, 64),
               (2, 6, 0, 0, 8, 8), (1, 7, 120, 0, 1, 91)]  # slot 6: frame 2 of two
    fl, keep2 = frame_list(fmt, frames, ["bt709"] * 2, True, mean4, norm4)
    got, cls = run_rois_list(m, fl, cuda_i32(regions), want_classes=True)
    outs, obufs, classes = outputs(m, want_classes=True)
    g = _lib.Frames.from_buffer_copy(f)
    g.matrix, g.linear_filter = MATRIX_IDS["bt709"], 1
    g.mean4, g.norm4 = (C.c_float * 4)(*mean4), (C.c_float * 4)(*norm4)
    _lib.check(_lib.lib().snnb_model_run_rois(m.h, C.byref(g), 2, cuda_i32(regions).data_ptr(), None, obufs, len(outs), classes.data_ptr(), m._torch_stream()),
               "snnb_model_run_rois")
    assert np.array_equal(host(got[0]).view(np.uint8), host(outs[0]).view(np.uint8)) and np.array_equal(host(cls), host(classes))
    assert host(cls)[6] == 0 and (np.delete(host(cls), 6) >= 1).all()


def test_rois_from_detections_list_equals_the_restatement(ctx):
    rng = np.random.default_rng(5)
    rows = np.concatenate([rng.integers(0, 4, (5, 30, 1)), rng.random((5, 30, 1)), rng.random((5, 30, 4)) * 1.4 - 0.2], axis=2).astype(np.float32)
    rows[1, 3, 2] = np.nan
    counts = np.array([30, 12, 0, 30, 7], np.int32)
    sizes = [(2160, 3840), (1080, 1920), (720, 1280), (91, 121), (1, 1)]
    rt, ct = torch.from_numpy(rows).cuda(), cuda_i32(counts)
    for cap, sel in ((256, {}), (9, {}), (256, {"class_id": 2}), (256, {"min_score": 0.5, "expand": 0.25})):
        got, cnt = ctx.rois_from_detections(rt, ct, sizes, cap, **sel)
        want, wcnt = rois_from_detections_list(rows, counts, sizes, cap, **sel)
        assert int(host(cnt)[0]) == wcnt and np.array_equal(host(got), want), (cap, sel)
        # every size equal: the same bytes as the single-size entry point
        same, c1 = ctx.rois_from_detections(rt, ct, [(1080, 1920)] * 5, cap, **sel)
        one, c2 = ctx.rois_from_detections(rt, ct, (1080, 1920), cap, **sel)
        assert int(host(c1)[0]) == int(host(c2)[0]) and np.array_equal(host(same), host(one)), (cap, sel)
    assert wcnt > 0
    with pytest.raises(ValueError):
        ctx.rois_from_detections(rt, ct, sizes[:4], 8)


def test_chain_on_a_new_stream_equals_the_synchronised_chain(ctx, model_dir):
    det = load_yolo(ctx, model_dir, "allpass", batch=3)
    cls = load(ctx, model_dir, "resnet18", (64, 64), 16, fuse=True, use_cuda_graph=True)
    dmean, dnorm = NORM["yolov3tiny"]
    mean4, norm4 = NORM["resnet18"]
    from test_frames_gpu import packed
    src = [packed("nv12", *random_yuv(1, h, w, seed=90 + h))[0] for h, w in ((240, 320), (180, 416), (120, 160))]
    hw = [tuple(int(v) for v in (t.shape[0] // 3 * 2, t.shape[1])) for t in src]
    rows, counts = det.detect_frame_list(src, mean4=dmean, norm4=dnorm)
    want_rois, want_count = rois_from_detections_list(host(rows), host(counts), hw, 16, expand=0.1)
    assert want_count == 16
    got_rois, got_count = ctx.rois_from_detections(rows, counts, hw, 16, expand=0.1)
    assert np.array_equal(host(got_rois), want_rois)
    want = host(cls.run_rois_list(src, cuda_i32(want_rois), cuda_i32([want_count]), mean4=mean4, norm4=norm4))
    torch.cuda.synchronize()

    def chain(stream):
        with torch.cuda.stream(stream):
            torch.cuda._sleep(100_000_000)
            xs = [torch.empty_like(s) for s in src]
            for x, s in zip(xs, src):
                x.copy_(s)
            r, c = det.detect_frame_list(xs, mean4=dmean, norm4=dnorm)
            regions, count = ctx.rois_from_detections(r, c, hw, 16, expand=0.1)
            return cls.run_rois_list(xs, regions, count, mean4=mean4, norm4=norm4).clone(), regions.clone()

    got, got_rois = chain(torch.cuda.Stream())
    assert np.array_equal(host(got_rois), want_rois) and np.array_equal(host(got), want)


def tiny(ctx, tmp_path, batch):
    b = modelzoo.Builder(seed=5)
    b.batchnorm(b.input(2, 2, 3))
    return core.MixedInferenceCore(ctx, modelzoo.write_model(b.layers, str(tmp_path / "tiny.json")), batch=batch)


def test_list_of_256_images_is_accepted_and_257_is_refused(ctx, model_dir, tmp_path):
    m = tiny(ctx, tmp_path, 256)
    made = [image("nv12", 1 + i % 7, 1 + i % 5, seed=i) for i in range(257)]
    frames = [f for _, f in made]
    mats = [MATRICES[i % 4] for i in range(257)]
    fl, keep = frame_list("nv12", frames[:256], mats[:256])
    got = host(run_list(m, fl)[0][0])
    for i in (0, 1, 6, 100, 255):
        assert np.array_equal(got[i], host(run_frames(m, repeated(frames[i], mats[i], True, (0.0,) * 4, (1.0,) * 4))[0][0])[i]), i
    big, keep2 = frame_list("nv12", frames, mats)
    with pytest.raises(SnnbError, match="count 257"):
        run_list(m, big)
    r = tiny(ctx, tmp_path, 4)
    regions = cuda_i32([(255, 0, 0, 0, 1, 1), (256, 1, 0, 0, 1, 1), (0, 2, 0, 0, 1, 1), (3, 3, 0, 0, 4, 4)])
    got, _ = run_rois_list(r, fl, regions)
    g = host(got[0])
    assert g[0].any() and not g[1].any() and g[2].any() and g[3].any()  # frame 256 does not exist in a list of 256
    with pytest.raises(SnnbError, match="count 257; a list holds 1 to 256 frames"):
        run_rois_list(r, big, regions)


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")  # the refused call leaves the caller's capture empty, as it should
def test_refusals_launch_nothing_and_write_nothing(ctx, model_dir, tmp_path):
    m = load(ctx, model_dir, "resnet18", (64, 64), 8, fuse=True, use_cuda_graph=True)
    made = [image("nv12", h, w, seed=i, pitch_align=a) for i, (h, w, a) in enumerate(SIZES)]
    frames = [f for _, f in made]
    made10 = [image("p010", 10, 12, seed=i) for i in range(8)]
    good, keep = frame_list("nv12", frames, MATRICES * 2)
    r = cuda_i32(RREGIONS)
    want = host(run_list(m, good)[0][0])
    out = outputs(m, want_classes=True)

    def refused(fn, text):
        before = ctx.launches
        with pytest.raises(SnnbError) as e:
            fn()
        assert text in str(e.value), str(e.value)
        assert ctx.launches == before, "a refused call launched kernels"
        assert (host(out[0][0]).view(np.uint8) == 0x5A).all() and (host(out[2]).view(np.uint8) == 0x5A).all(), "a refused call wrote"

    def bad(i=3, fmt="nv12", fr=None, **kw):
        fs = [_lib.Frames.from_buffer_copy(f) for f in (fr or frames)]
        for k, val in kw.items():
            if k in ("plane", "pitch"):
                getattr(fs[i], k)[val[0]] = val[1]
            else:
                setattr(fs[i], k, val)
        mats = MATRICES * 2
        fl, images = frame_list(fmt, fs, mats)
        if "matrix" in kw:
            images[i].matrix = kw["matrix"]
        bad.keep = images
        return fl

    run = lambda fl: run_list(m, fl, want_classes=True, out=out)  # noqa: E731
    rois = lambda fl, count=None, stream=None: run_rois_list(m, fl, r, count, want_classes=True, out=out, stream=stream)  # noqa: E731
    for call, name in ((run, "snnb_model_run_frame_list"), (rois, "snnb_model_run_rois_list")):
        f = bad()
        f.format = 4
        refused(lambda: call(f), "%s: unknown frame format 4" % name)
        f = bad()
        f.images = None
        refused(lambda: call(f), "%s: null images" % name)
        refused(lambda: call(bad(matrix=2)), "%s: image 3: unknown YUV matrix 2" % name)
        refused(lambda: call(bad(matrix=MATRIX_IDS["bt709"] | 0x100)), "image 3: YUV matrix 257: full range is defined for BT.601 only")
        refused(lambda: call(bad(i=5, width=0)), "%s: image 5: frame size 0 x 33; width and height must be >= 1" % name)
        refused(lambda: call(bad(i=2, height=-1)), "image 2: frame size 90 x -1")
        refused(lambda: call(bad(i=1, pitch=(0, 120))), "%s: image 1 plane 0: pitch 120 is less than its row's 121 bytes" % name)
        refused(lambda: call(bad(i=7, pitch=(1, 63))), "image 7 plane 1: pitch 63 is less than its row's 66 bytes")
        refused(lambda: call(bad(i=4, plane=(1, np.zeros(1000, np.uint8).ctypes.data))), "image 4 plane 1: ")
        pinned = torch.zeros(1000, dtype=torch.uint8).pin_memory()
        refused(lambda: call(bad(i=0, plane=(0, pinned.data_ptr()))), "pinned host memory")
        refused(lambda: call(bad(i=6, plane=(1, None))), "image 6 plane 1: null data pointer")
        p = [f for _, f in made10]
        refused(lambda: call(bad(i=2, fmt="p010", fr=p, pitch=(0, 25))), "image 2 plane 0: P010 pitch 25 and image stride 0 must be even")
        refused(lambda: call(bad(i=2, fmt="p010", fr=p, plane=(1, p[2].plane[1] + 1))), "image 2 plane 1: ")
        g = torch.cuda.CUDAGraph()

        def capture():
            with torch.cuda.graph(g, capture_error_mode="relaxed"):
                call(good)
        refused(capture, "being captured")
    # the count rules: the batch for run / detect, 1..256 for regions
    short, keep3 = frame_list("nv12", frames[:7], MATRICES * 2)
    refused(lambda: run(short), "count 7; the list must hold the model's batch of 8 images")
    none, keep4 = frame_list("nv12", [], [])
    refused(lambda: rois(none), "count 0; a list holds 1 to 256 frames")
    refused(lambda: run_rois_list(m, good, None, want_classes=True, out=out), "snnb_model_run_rois_list: null rois")
    refused(lambda: run_rois_list(m, good, r.data_ptr() + 2, want_classes=True, out=out), "is not aligned to its 4-byte elements")
    refused(lambda: _lib.check(_lib.lib().snnb_model_run_frame_list(m.h, None, out[1], 1, None, None), "x"), "snnb_model_run_frame_list: null frames")
    refused(lambda: _lib.check(_lib.lib().snnb_model_run_rois_list(m.h, None, r.data_ptr(), None, out[1], 1, None, None), "x"),
            "snnb_model_run_rois_list: null frames")
    # models the list cannot feed
    yolo = load_yolo(ctx, model_dir, "planted", batch=8)
    refused(lambda: run_list(yolo, good), "use snnb_model_detect_frame_list")
    refused(lambda: _lib.check(_lib.lib().snnb_model_detect_frame_list(m.h, C.byref(good), out[0][0].data_ptr(), 10, out[2].data_ptr(), None), "x"),
            "no YOLO output; use snnb_model_run_frame_list")
    refused(lambda: _lib.check(_lib.lib().snnb_model_detect_frame_list(m.h, None, out[0][0].data_ptr(), 10, out[2].data_ptr(), None), "x"),
            "snnb_model_detect_frame_list: null frames")
    b = modelzoo.Builder(seed=3)
    b.add(b.input(20, 16, 3, index=0), b.input(20, 16, 3, index=1))
    two = core.MixedInferenceCore(ctx, modelzoo.write_model(b.layers, str(tmp_path / "two.json")), batch=8)
    refused(lambda: run_list(two, good), "the model has 2 inputs")
    assert np.array_equal(host(run_list(m, good)[0][0]), want)  # the model is still usable

    # rois_from_detections_list: outputs pre-filled; a refused call writes nothing
    rows = torch.rand((2, 10, 6), device="cuda")
    counts = cuda_i32([10, 10])
    regions, count = cuda_i32(np.full((8, 6), 77)), cuda_i32([77])
    wh = (C.c_int * 4)(320, 240, 64, 48)

    def rfd(n=2, frame_wh=wh, sel=(0.0, -1, 0.0), stream=1):
        s = None if sel is None else C.byref(_lib.RoiSelect(*sel))
        _lib.check(_lib.lib().snnb_rois_from_detections_list(ctx.h, rows.data_ptr(), counts.data_ptr(), n, 10, frame_wh, s, regions.data_ptr(), 8,
                                                             count.data_ptr(), stream), "snnb_rois_from_detections_list")

    def refused_rfd(text, **kw):
        before = ctx.launches
        with pytest.raises(SnnbError) as e:
            rfd(**kw)
        assert text in str(e.value), str(e.value)
        assert ctx.launches == before and (host(regions) == 77).all() and int(host(count)[0]) == 77

    refused_rfd("snnb_rois_from_detections_list: null frame_wh", frame_wh=None)
    refused_rfd("snnb_rois_from_detections_list: null sel", sel=None)
    refused_rfd("frame 1: size 64 x 0; width and height must be >= 1", frame_wh=(C.c_int * 4)(320, 240, 64, 0))
    refused_rfd("frame 0: size -1 x 240", frame_wh=(C.c_int * 4)(-1, 240, 64, 48))
    refused_rfd("num_frames 257 is more than 256", n=257, frame_wh=(C.c_int * 514)(*([8] * 514)))
    refused_rfd("num_frames 0", n=0)
    g2 = torch.cuda.CUDAGraph()

    def capture_rfd():
        with torch.cuda.graph(g2, capture_error_mode="relaxed"):
            rfd(stream=torch.cuda.current_stream().cuda_stream)
    before = ctx.launches
    with pytest.raises(SnnbError) as e:
        capture_rfd()
    assert "being captured" in str(e.value) and ctx.launches == before and (host(regions) == 77).all()
    rfd()  # the same arguments, valid: it runs
    assert int(host(count)[0]) == 8
