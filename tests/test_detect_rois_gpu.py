"""snnb_model_detect_rois / detect_rois_list (MixedInferenceCore.detect_rois / detect_rois_list): detection on regions of device frames.

Each frame's rows and count must equal tests/_region_merge.py's merge_region_rows (the float32 restatement of the mapping and the per-frame merge
in include/snnb.h) applied to each slot's own detections: the rows detect_frames(format="rgba8") returns on the same model handle for
that slot's crop of libyuv's RGBA8 image (P010: detect_torch of the restated 10-bit model input of the crop), max_rows 100. That is bit
identity, so the gather, the mapping, the stable sort and the NMS are all held to the header."""
import ctypes as C

import numpy as np
import pytest

import _region_merge as region_merge
from oracle import yuv10
from shadernn_b200 import _lib, core
from shadernn_b200._lib import SnnbError
from test_detect_gpu import yolo_path
from test_frames_gpu import NORM, expected_rgba, host, laid_out, load, packed, random_yuv, set_params
from test_p010_gpu import laid_out10, random_yuv10
from test_p010_gpu import set_params as set_params10

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

HW = (416, 416)
MEAN4, NORM4 = NORM["yolov3tiny"]
FH, FW = 301, 437  # odd frames
B = 8
# {frame, row, x, y, width, height} over two FH x FW frames: edges, 1 x 1, the model's size, a duplicate region, and invalid slots
REGIONS = [(0, 0, 0, 0, 200, 150),  # top-left corner
           (0, 1, FW - 220, FH - 180, 220, 180),  # touching the right and bottom edges
           (1, 2, 10, 11, 416, 290),  # wide
           (1, 3, 57, 44, 1, 1),  # 1 x 1
           (0, 4, 0, 0, 200, 150),  # the same region as slot 0: its boxes are suppressed by slot 0's
           (1, 5, 0, 0, FW, FH),  # the whole frame
           (2, 6, 0, 0, 10, 10),  # frame out of range
           (0, 7, FW - 5, 0, 10, 10)]  # outside the frame


def cuda_i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda()


def yolo(ctx, model_dir, kind, batch=B, **kw):
    kw = dict({"fuse": True, "use_cuda_graph": True}, **kw)
    return core.MixedInferenceCore(ctx, yolo_path(model_dir, kind, HW), batch=batch, input_hw=HW, **kw)


def crop(images, roi):
    f, _, x, y, w, h = (int(v) for v in roi)
    return np.ascontiguousarray(images[f][y:y + h, x:x + w])


def want_slot_rows(m, images, regions, count, sizes, linear, detect=None):
    """Each valid slot's rows [B, 100, 6] and counts [B]: detect_frames(format="rgba8") of its crop on m, one call per crop size (or
    detect(crops) for the crops of one size)."""
    rows, counts = np.zeros((m.batch, 100, 6), np.float32), np.zeros(m.batch, np.int32)
    used = m.batch if count is None else min(max(count, 0), m.batch)
    valid = [i for i, r in enumerate(regions) if region_merge.roi_valid(r, i, used, sizes)]
    crops = {i: crop(images, regions[i]) for i in valid}
    for hw in sorted({c.shape[:2] for c in crops.values()}):
        slots = [i for i in valid if crops[i].shape[:2] == hw]
        batch = [crops[i] for i in slots] + [crops[slots[0]]] * (m.batch - len(slots))
        if detect is None:
            r, c = m.detect_frames(torch.from_numpy(np.stack(batch)).cuda(), format="rgba8", linear=linear, mean4=MEAN4, norm4=NORM4)
        else:
            r, c = detect(batch)
        r, c = host(r), host(c)
        for k, i in enumerate(slots):
            rows[i], counts[i] = r[k], c[k]
    return rows, counts


def raw_detect(m, f, num_frames, rois, count=None, max_rows=100, out=None, stream=None):
    rows, counts = out if out is not None else (torch.empty((num_frames, max_rows, 6), dtype=torch.float32, device="cuda"),
                                                torch.empty(num_frames, dtype=torch.int32, device="cuda"))
    ptr = lambda t: None if t is None else (t if isinstance(t, int) else t.data_ptr())  # noqa: E731
    _lib.check(_lib.lib().snnb_model_detect_rois(m.h, C.byref(f), num_frames, ptr(rois), ptr(count), ptr(rows), max_rows, ptr(counts),
                                                 stream if stream is not None else m._torch_stream()), "snnb_model_detect_rois")
    return rows, counts


def sentinel(num_frames, max_rows, extra=7):
    """rows and counts inside larger buffers filled with NaN / -7, so that an unwritten element and a write outside show."""
    rows = torch.full((num_frames * max_rows * 6 + extra,), float("nan"), device="cuda")
    counts = torch.full((num_frames + extra,), -7, dtype=torch.int32, device="cuda")
    return rows, counts


def check_sentinel(rows, counts, num_frames, max_rows, want_rows, want_counts):
    r, c = host(rows), host(counts)
    n = num_frames * max_rows * 6
    assert np.array_equal(r[:n].reshape(num_frames, max_rows, 6), want_rows) and np.array_equal(c[:num_frames], want_counts)
    assert np.isnan(r[n:]).all() and (c[num_frames:] == -7).all(), "written outside [num_frames][max_rows]"


def frames_of(fmt, n, hw, seed):
    """(keep-alive, snnb_frames, per-frame RGBA8 images; P010: per-frame 10-bit planes)."""
    if fmt == "p010":
        y, u, v = random_yuv10(n, hw[0], hw[1], seed=seed)
        keep, f = laid_out10(y, u, v, pitch_align=64)
        return keep, f, (y, u, v)
    y, u, v = random_yuv(n, hw[0], hw[1], seed=seed)
    rgba = expected_rgba("nv12", y, u, v, "bt601")
    keep, f = laid_out(fmt, y, u, v, rgba=rgba)
    return keep, f, rgba


def p010_detect(m, planes, linear):
    """detect_torch of the restated model input of each crop of 10-bit frames: detect(batch) for want_slot_rows."""
    y, u, v = planes
    tex = [yuv10.texels(y[i:i + 1], u[i:i + 1], v[i:i + 1], "bt601")[0] for i in range(y.shape[0])]

    def detect(batch):
        x = np.concatenate([yuv10.model_input(t[None], HW, 3, linear, MEAN4, NORM4) for t in batch])
        return m.detect_torch(torch.from_numpy(np.ascontiguousarray(x)).cuda())
    return tex, detect


@pytest.mark.parametrize("kind", ["planted", "allpass"])
@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("fmt", ["nv12", "nv21", "i420", "rgba8", "p010"])
def test_every_frame_equals_the_merge_of_detect_frames_of_each_crop(ctx, model_dir, fmt, linear, kind):
    m = yolo(ctx, model_dir, kind)
    keep, f, images = frames_of(fmt, 3, (FH, FW), seed=len(fmt) * 7 + linear)  # three frames: frame 2 has no region
    (set_params10 if fmt == "p010" else set_params)(f, linear=linear, mean4=MEAN4, norm4=NORM4)
    sizes = [(FH, FW)] * 3
    regions = REGIONS[:6] + [(3, 6, 0, 0, 10, 10), (0, 7, FW - 5, 0, 10, 10)]  # frame 3 of three: out of range
    detect = None
    if fmt == "p010":
        images, detect = p010_detect(m, images, linear)
    slot_rows, slot_counts = want_slot_rows(m, images, regions, None, sizes, linear, detect)
    if kind == "allpass":
        assert slot_counts.max() == 100  # heavy suppression across slots, and equal scores
    for max_rows in (100, 17):
        rows, counts = sentinel(3, max_rows)
        raw_detect(m, f, 3, cuda_i32(regions), max_rows=max_rows, out=(rows, counts))
        want, wc = region_merge.merge_region_rows(slot_rows, slot_counts, regions, None, sizes, max_rows)
        check_sentinel(rows, counts, 3, max_rows, want, wc)
        assert wc[2] == 0 and wc[:2].sum() > 0
    # slot 4 repeats slot 0's region, so its boxes are all suppressed: without it (an invalid slot) frame 0 comes out the same
    alone = list(regions)
    alone[4] = (9, 4, 0, 0, 1, 1)
    rows, counts = raw_detect(m, f, 3, cuda_i32(regions))
    got, gc = raw_detect(m, f, 3, cuda_i32(alone))
    assert np.array_equal(host(got), host(rows)) and np.array_equal(host(gc), host(counts))


def test_all_slots_on_one_frame_with_all_pass_heads(ctx, model_dir):
    m = yolo(ctx, model_dir, "allpass", batch=16)
    y, u, v = random_yuv(2, 480, 640, seed=3)
    rgba = expected_rgba("nv12", y, u, v, "bt601")
    rng = np.random.default_rng(5)
    regions = [(1, i, int(rng.integers(0, 300)), int(rng.integers(0, 200)), 300 + i, 250 + i) for i in range(16)]
    regions[3] = regions[2]  # equal scores across slots: the tie goes to the lower slot
    rows, counts = m.detect_rois(packed("nv12", y, u, v), cuda_i32(regions), mean4=MEAN4, norm4=NORM4)
    slot_rows, slot_counts = want_slot_rows(m, rgba, regions, None, [(480, 640)] * 2, True)
    assert (slot_counts == 100).all()
    want, wc = region_merge.merge_region_rows(slot_rows, slot_counts, regions, None, [(480, 640)] * 2, 100)
    assert np.array_equal(host(rows), want) and np.array_equal(host(counts), wc) and wc[0] == 0 and wc[1] > 0


def test_counted_calls_equal_the_call_at_the_chosen_size(ctx, model_dir):
    m = yolo(ctx, model_dir, "planted")
    y, u, v = random_yuv(2, FH, FW, seed=9)
    src = packed("nv12", y[:, :FH - 1, :FW - 1], u[:, :(FH - 1) // 2, :(FW - 1) // 2], v[:, :(FH - 1) // 2, :(FW - 1) // 2])
    regions = [(r[0] % 2, r[1], r[2] // 2, r[3] // 2, max(r[4] // 2, 1), max(r[5] // 2, 1)) for r in REGIONS]
    r = cuda_i32(regions)
    m.set_count_batches([2, 4])
    for k, size in ((1, 2), (3, 4), (5, B), (B, B), (0, 0)):
        got, gc = m.detect_rois(src, r, cuda_i32([k]), mean4=MEAN4, norm4=NORM4)
        got, gc = host(got), host(gc)
        if size == 0:
            assert not got.any() and not gc.any()
            continue
        m.set_batch(size)
        want, wc = m.detect_rois(src, r[:size], cuda_i32([k]), mean4=MEAN4, norm4=NORM4)
        m.set_batch(B)
        assert np.array_equal(got, host(want)) and np.array_equal(gc, host(wc)), k
    m.set_count_batches([])


def test_list_form_mixed_sizes_and_equal_to_the_batch_form(ctx, model_dir):
    m = yolo(ctx, model_dir, "planted")
    shapes = [(FH, FW), (240, 320), (481, 641)]
    frames, images = [], []
    for i, (h, w) in enumerate(shapes):
        y, u, v = random_yuv(1, h, w, seed=40 + i)
        images.append(expected_rgba("nv12", y, u, v, "bt601")[0])
        frames.append(torch.from_numpy(images[-1]).cuda())
    regions = [(0, 0, 0, 0, 200, 150), (1, 1, 0, 0, 320, 240), (2, 2, 100, 100, 381, 300), (1, 3, 200, 100, 120, 140),
               (2, 4, 0, 0, 641, 481), (1, 5, 0, 0, 400, 100), (0, 6, 3, 3, 50, 60), (2, 7, 600, 400, 41, 81)]  # slot 5: wider than frame 1
    rows, counts = m.detect_rois_list(frames, cuda_i32(regions), format="rgba8", mean4=MEAN4, norm4=NORM4)
    slot_rows, slot_counts = want_slot_rows(m, images, regions, None, shapes, True)
    want, wc = region_merge.merge_region_rows(slot_rows, slot_counts, regions, None, shapes, 100)
    assert np.array_equal(host(rows), want) and np.array_equal(host(counts), wc)
    # equal sizes: the list form is the batch form byte for byte
    y, u, v = random_yuv(2, FH, FW, seed=50)
    rgba = expected_rgba("nv12", y, u, v, "bt601")
    r = cuda_i32(REGIONS)
    batch = m.detect_rois(torch.from_numpy(rgba).cuda(), r, format="rgba8", mean4=MEAN4, norm4=NORM4)
    lst = m.detect_rois_list([torch.from_numpy(rgba[i]).cuda() for i in range(2)], r, format="rgba8", mean4=MEAN4, norm4=NORM4)
    assert all(np.array_equal(host(a).view(np.uint8), host(b).view(np.uint8)) for a, b in zip(batch, lst))


def test_whole_frame_regions_agree_with_detect_frames(ctx, model_dir):
    # (0 + x * W) / W is not always x in float32, so the coordinates agree to a couple of ulps, not bit for bit
    m = yolo(ctx, model_dir, "planted", batch=2)
    y, u, v = random_yuv(2, 480, 640, seed=60)
    src = packed("nv12", y, u, v)
    want, wc = (host(t) for t in m.detect_frames(src, mean4=MEAN4, norm4=NORM4))
    got, gc = (host(t) for t in m.detect_rois(src, cuda_i32([(0, 0, 0, 0, 640, 480), (1, 1, 0, 0, 640, 480)]), mean4=MEAN4, norm4=NORM4))
    assert np.array_equal(gc, wc) and wc.sum() > 0
    assert np.array_equal(got[..., :2], want[..., :2])
    np.testing.assert_array_max_ulp(got[..., 2:], want[..., 2:], maxulp=4)


def test_tiles_and_a_whole_frame_region(ctx, model_dir):
    m = yolo(ctx, model_dir, "planted", batch=16)
    y, u, v = random_yuv(1, 720, 1280, seed=70)
    rgba = expected_rgba("nv12", y, u, v, "bt601")
    tiles = core.tile_rois((720, 1280), (416, 416), 64)
    regions = np.concatenate([tiles, [[0, len(tiles), 0, 0, 1280, 720]]]).astype(np.int32)
    assert len(regions) <= 16
    regions = np.concatenate([regions, np.zeros((16 - len(regions), 6), np.int32)])
    count = len(tiles) + 1
    rows, counts = m.detect_rois(packed("nv12", y, u, v), cuda_i32(regions), cuda_i32([count]), mean4=MEAN4, norm4=NORM4)
    slot_rows, slot_counts = want_slot_rows(m, rgba, regions, count, [(720, 1280)], True)
    want, wc = region_merge.merge_region_rows(slot_rows, slot_counts, regions, count, [(720, 1280)], 100)
    assert np.array_equal(host(rows), want) and np.array_equal(host(counts), wc) and wc[0] > 0


def test_chains_on_a_new_stream_equal_the_synchronised_chains(ctx, model_dir):
    det = yolo(ctx, model_dir, "planted", batch=16)
    first = yolo(ctx, model_dir, "planted", batch=2)
    y, u, v = random_yuv(2, 720, 1280, seed=80)
    src = packed("nv12", y, u, v)
    tiles = np.concatenate([core.tile_rois((720, 1280), (416, 416), 64, frame=f) for f in range(2)])[:14]
    tiles = np.concatenate([tiles, [[0, 14, 0, 0, 1280, 720], [1, 15, 0, 0, 1280, 720]]]).astype(np.int32)
    want_tiled = [host(t) for t in det.detect_rois(src, cuda_i32(tiles), mean4=MEAN4, norm4=NORM4)]
    frames = [src[0], src[1]]
    r1, c1 = first.detect_frame_list(frames, mean4=MEAN4, norm4=NORM4)
    rois, count = ctx.rois_from_detections(r1, c1, [(720, 1280)] * 2, 16, expand=0.5)
    want_zoom = [host(t) for t in det.detect_rois_list(frames, rois, count, mean4=MEAN4, norm4=NORM4)]
    torch.cuda.synchronize()

    def chain(stream):
        with torch.cuda.stream(stream):
            torch.cuda._sleep(100_000_000)
            x = torch.empty_like(src)
            x.copy_(src)
            tiled = det.detect_rois(x, cuda_i32(tiles), mean4=MEAN4, norm4=NORM4)
            fl = [x[0], x[1]]
            r, c = first.detect_frame_list(fl, mean4=MEAN4, norm4=NORM4)
            ro, co = ctx.rois_from_detections(r, c, [(720, 1280)] * 2, 16, expand=0.5)
            zoom = det.detect_rois_list(fl, ro, co, mean4=MEAN4, norm4=NORM4)
            return [t.clone() for t in tiled + zoom]

    got = [host(t) for t in chain(torch.cuda.Stream())]
    assert all(np.array_equal(g, w) for g, w in zip(got, want_tiled + want_zoom))
    assert want_tiled[1].sum() + want_zoom[1].sum() > 0


@pytest.mark.parametrize("precision,fuse,graph", [("fp32x3", False, False), ("fp32x3", True, False), ("fp32x3", True, True), ("fp16", True, True),
                                                  ("fp16", False, False)])
def test_precisions_and_graph_modes(ctx, model_dir, precision, fuse, graph):
    m = yolo(ctx, model_dir, "planted", precision=precision, fuse=fuse, use_cuda_graph=graph)
    y, u, v = random_yuv(2, FH, FW, seed=90)
    rgba = expected_rgba("nv12", y, u, v, "bt601")
    keep, f = laid_out("nv12", y, u, v)
    set_params(f, mean4=MEAN4, norm4=NORM4)
    rows, counts = raw_detect(m, f, 2, cuda_i32(REGIONS))
    slot_rows, slot_counts = want_slot_rows(m, rgba, REGIONS, None, [(FH, FW)] * 2, True)
    want, wc = region_merge.merge_region_rows(slot_rows, slot_counts, REGIONS, None, [(FH, FW)] * 2, 100)
    assert np.array_equal(host(rows), want) and np.array_equal(host(counts), wc)


def test_launch_count(ctx, model_dir):
    m = yolo(ctx, model_dir, "planted")
    y, u, v = random_yuv(2, FH, FW, seed=95)
    keep, f = laid_out("nv12", y, u, v)
    set_params(f, mean4=MEAN4, norm4=NORM4)
    r = cuda_i32(REGIONS)
    raw_detect(m, f, 2, r)
    before = ctx.launches
    raw_detect(m, f, 2, r)
    assert ctx.launches - before == m.launches_per_forward + 7  # the input, three decode kernels and three merge kernels


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")  # the refused call leaves the caller's capture empty, as it should
def test_refusals_launch_nothing_and_write_nothing(ctx, model_dir):
    m = yolo(ctx, model_dir, "planted")
    y, u, v = random_yuv(2, FH, FW, seed=99)
    keep, f = laid_out("nv12", y, u, v)
    set_params(f, mean4=MEAN4, norm4=NORM4)
    r, cnt = cuda_i32(REGIONS), cuda_i32([4])
    want = [host(t) for t in raw_detect(m, f, 2, r)]
    rows, counts = sentinel(2, 100)

    def refused(text, call):
        before = ctx.launches
        with pytest.raises(SnnbError) as e:
            call()
        assert text in str(e.value), str(e.value)
        assert ctx.launches == before, "a refused call launched kernels"
        assert np.isnan(host(rows)).all() and (host(counts) == -7).all(), "a refused call wrote"

    def run(frames=f, n=2, rois=r, count=None, rows_p=rows, counts_p=counts, max_rows=100, stream=None):
        return raw_detect(m, frames, n, rois, count, max_rows, out=(rows_p, counts_p), stream=stream)

    resnet = _resnet(ctx, model_dir)
    refused("no YOLO output; use snnb_model_run_rois", lambda: raw_detect(resnet, f, 2, r, out=(rows, counts)))
    refused("max_rows 0 is outside 1..100", lambda: run(max_rows=0))
    refused("max_rows 101 is outside 1..100", lambda: run(max_rows=101))
    refused("null rois", lambda: run(rois=None))
    refused("rows 0: null data pointer", lambda: run(rows_p=None))
    refused("counts 0: null data pointer", lambda: run(counts_p=None))
    refused("unregistered host memory", lambda: run(rows_p=np.zeros(1200, np.float32).ctypes.data))
    refused("pinned host memory", lambda: run(counts_p=torch.zeros(2, dtype=torch.int32).pin_memory()))
    refused("is not aligned to its 4-byte elements", lambda: run(rows_p=rows.data_ptr() + 2))
    refused("is not aligned to its 4-byte elements", lambda: run(counts_p=counts.data_ptr() + 1))
    refused("is not aligned to its 4-byte elements", lambda: run(rois=r.data_ptr() + 2))
    refused("is not aligned to its 4-byte elements", lambda: run(count=cnt.data_ptr() + 1))
    refused("unregistered host memory", lambda: run(rois=np.asarray(REGIONS, np.int32).ctypes.data))
    refused("num_frames 0", lambda: run(n=0))
    g = torch.cuda.CUDAGraph()

    def capture():
        with torch.cuda.graph(g, capture_error_mode="relaxed"):
            run(stream=torch.cuda.current_stream().cuda_stream)
    refused("being captured", capture)
    fl = _lib.FrameList()
    images = (_lib.FrameImage * 1)()
    fl.format, fl.images = _lib.FRAME_NV12, images
    for n in (0, 257):
        fl.count = n

        def call_list():
            _lib.check(_lib.lib().snnb_model_detect_rois_list(m.h, C.byref(fl), r.data_ptr(), None, rows.data_ptr(), 100, counts.data_ptr(), 1),
                       "snnb_model_detect_rois_list")
        refused("count %d; a list holds 1 to 256 frames" % n, call_list)
    # run_rois keeps refusing YOLO models and names the new call
    outs, obufs, _ = m._device_outputs("test", None, "nhwc", 1.0, 0.0, False)
    with pytest.raises(SnnbError) as e:
        _lib.check(_lib.lib().snnb_model_run_rois(m.h, C.byref(f), 2, r.data_ptr(), None, obufs, 0, None, 1), "snnb_model_run_rois")
    assert "detection on regions is not supported" in str(e.value) and "snnb_model_detect_rois" in str(e.value)
    # the model still gives the same answer
    assert all(np.array_equal(host(a), b) for a, b in zip(raw_detect(m, f, 2, r), want))


def _resnet(ctx, model_dir):
    return load(ctx, model_dir, "resnet18", (64, 64), B, fuse=True, use_cuda_graph=True)
