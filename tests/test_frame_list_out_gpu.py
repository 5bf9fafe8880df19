"""Output lists (snnb_model_transform_frame_list / transform_luma_list / segment_frame_list; MixedInferenceCore.transform_frame_list /
transform_luma_list / segment_frame_list): a frame list in, one separately allocated output per image out, each at its own size.

Out image i must be bit-identical to what the batch call on the same handle writes when it is fed a batch whose every frame is input
image i (test_frame_list_gpu's `repeated`) and writes a batch-sized output of out image i's size; every slot of that output is the same.
Each out image lives in its own device buffer between sentinel bytes, with padded rows, so a byte written outside the rows shows."""
import ctypes as C

import numpy as np
import pytest

from shadernn_b200 import _lib, core, modelzoo
from shadernn_b200._lib import SnnbError
from test_frame_list_gpu import MATRICES, frame_list, image, repeated
from test_frames_gpu import host, load
from test_luma_gpu import MEAN as LMEAN, NORM as LNORM, espcn
from test_segment_gpu import conv_model

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

FILL = 0xA5
GUARD = 64  # sentinel bytes before and after each out allocation
FORMATS = {"nv12": 0, "nv21": 1, "i420": 2, "rgba8": 3, "p010": 16}
_paths = {}


def plane_shapes(fmt, h, w):
    """(rows, row bytes) of each used plane of one h x w frame"""
    ch, cw = (h + 1) // 2, (w + 1) // 2
    return {"rgba8": [(h, 4 * w)], "i420": [(h, w), (ch, cw), (ch, cw)], "p010": [(h, 2 * w), (ch, 4 * cw)]}.get(fmt, [(h, w), (ch, 2 * cw)])


class OutFrames:
    """n images of h x w in `fmt` in ONE device buffer of FILL bytes: rows `pad` bytes longer than their data (even for P010), GUARD
    bytes before the first image and after the last."""

    def __init__(self, fmt, n, h, w, pad=0):
        self.fmt, self.n, self.h, self.w = fmt, n, h, w
        self.shapes = plane_shapes(fmt, h, w)
        self.pitches = [(b + pad + 1) // 2 * 2 if fmt == "p010" else b + pad for _, b in self.shapes]
        self.offs, cur = [], GUARD
        for (rows, _), pitch in zip(self.shapes, self.pitches):
            self.offs.append(cur)
            cur += rows * pitch
        self.stride = cur - GUARD
        self.buf = torch.full((GUARD + n * self.stride + GUARD,), FILL, dtype=torch.uint8, device="cuda")

    def ptr(self, p):
        return self.buf.data_ptr() + self.offs[p]

    def image(self):
        """its snnb_frame_out_image (n = 1)"""
        im = _lib.FrameOutImage()
        for p in range(len(self.shapes)):
            im.plane[p], im.pitch[p] = self.ptr(p), self.pitches[p]
        im.width, im.height = self.w, self.h
        return im

    def batch(self, linear, scale, offset):
        """its snnb_frames_out"""
        o = _lib.FramesOut()
        o.format, o.width, o.height, o.linear_filter, o.scale, o.offset = FORMATS[self.fmt], self.w, self.h, int(bool(linear)), scale, offset
        for p in range(len(self.shapes)):
            o.plane[p], o.pitch[p], o.image_stride[p] = self.ptr(p), self.pitches[p], self.stride
        return o

    def planes(self):
        """The rows of each plane [n, rows, row bytes]; asserts that every other byte still holds FILL."""
        b = host(self.buf)
        untouched = np.ones(b.shape, bool)
        out = []
        for (rows, cols), pitch, off in zip(self.shapes, self.pitches, self.offs):
            idx = off + np.arange(self.n)[:, None, None] * self.stride + np.arange(rows)[None, :, None] * pitch + np.arange(cols)[None, None, :]
            out.append(b[idx])
            untouched[idx] = False
        assert (b[untouched] == FILL).all(), "bytes outside the rows were written"
        return out


class OutLabels:
    """n label planes of h x w in ONE device buffer of FILL bytes, rows `pad` bytes longer than w, GUARD bytes on both sides"""

    def __init__(self, n, h, w, pad=0):
        self.n, self.h, self.w, self.pitch = n, h, w, w + pad
        self.stride = h * self.pitch
        self.buf = torch.full((2 * GUARD + n * self.stride,), FILL, dtype=torch.uint8, device="cuda")

    def image(self):
        return _lib.LabelsImage(self.buf.data_ptr() + GUARD, self.pitch, self.w, self.h)

    def batch(self, linear, threshold):
        o = _lib.LabelsOut()
        o.width, o.height, o.plane, o.pitch, o.image_stride = self.w, self.h, self.buf.data_ptr() + GUARD, self.pitch, self.stride
        o.linear_filter, o.threshold = int(bool(linear)), float(threshold)
        return o

    def labels(self):
        b = host(self.buf)
        idx = GUARD + np.arange(self.n)[:, None, None] * self.stride + np.arange(self.h)[None, :, None] * self.pitch + np.arange(self.w)[None, None, :]
        untouched = np.ones(b.shape, bool)
        untouched[idx] = False
        assert (b[untouched] == FILL).all(), "bytes outside the rows were written"
        return b[idx]


def out_list(fmt, outs, linear, scale, offset):
    images = (_lib.FrameOutImage * max(1, len(outs)))(*[o.image() for o in outs])
    return _lib.FrameOutList(FORMATS[fmt], len(outs), images, int(bool(linear)), scale, offset), images


def labels_list(outs, linear, threshold):
    images = (_lib.LabelsImage * max(1, len(outs)))(*[o.image() for o in outs])
    return _lib.LabelsList(len(outs), images, int(bool(linear)), threshold), images


def call(name, m, *args, stream=None):
    _lib.check(getattr(_lib.lib(), name)(m.h, *args, stream if stream is not None else m._torch_stream()), name)


def assert_same(got, want, what):
    for p, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and np.array_equal(g, w), "%s: plane %d: %d bytes differ" % (what, p, int((g != w).sum()) if g.shape == w.shape else -1)


def check_transform(m, entry, batch_entry, in_fmt, made, matrices, out_fmt, out_sizes, linear, out_linear, mean4, norm4, scale, offset, pads=None):
    """Runs the list entry point and, per image, its batch reference; compares every out image with slot 0 .. B-1 of the reference."""
    B = len(made)
    frames = [f for _, f in made]
    fl, keep = frame_list(in_fmt, frames, matrices, linear, mean4, norm4)
    outs = [OutFrames(out_fmt, 1, h, w, pad=(pads[i] if pads else 0)) for i, (h, w) in enumerate(out_sizes)]
    ol, keep2 = out_list(out_fmt, outs, out_linear, scale, offset)
    call(entry, m, C.byref(fl), C.byref(ol))
    got = [o.planes() for o in outs]
    for i, (f, mat) in enumerate(zip(frames, matrices)):
        ref = OutFrames(out_fmt, B, *out_sizes[i], pad=3)
        call(batch_entry, m, C.byref(repeated(f, mat, linear, mean4, norm4)), C.byref(ref.batch(out_linear, scale, offset)))
        want = ref.planes()
        for n in (0, B - 1):
            assert_same([g[0] for g in got[i]], [w[n] for w in want], "image %d against slot %d" % (i, n))
    return got


def candy(ctx, model_dir, batch, **kw):
    return load(ctx, model_dir, "candy", (48, 64), batch, **kw)


def rgba4(ctx, model_dir, batch, **kw):
    if "rgba4" not in _paths:
        b = modelzoo.Builder(seed=44)
        b.conv(b.input(40, 24, 4), 4, 3)
        _paths["rgba4"] = modelzoo.write_model(b.layers, "%s/list_out_rgba4.json" % model_dir)
    return core.MixedInferenceCore(ctx, _paths["rgba4"], batch=batch, **kw)


# (H, W, pitch alignment) of 6 input images, and the 6 out sizes: the model's (48 x 64: sampled directly), odd, 1 x 1, larger, smaller
IN_SIZES = [(48, 64, 1), (91, 121, 256), (1, 1, 1), (100, 90, 64), (33, 17, 32), (64, 48, 1)]
OUT_SIZES = [(48, 64), (33, 17), (1, 1), (91, 150), (20, 30), (48, 64)]
PADS = [0, 5, 1, 64, 3, 17]


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("in_fmt,out_fmt", [("nv12", "nv12"), ("nv21", "i420"), ("i420", "rgba8"), ("rgba8", "nv21"), ("p010", "p010"), ("nv12", "p010"),
                                            ("p010", "rgba8")])
def test_transform_equals_the_batch_call_per_image(ctx, model_dir, in_fmt, out_fmt, linear):
    m = candy(ctx, model_dir, 6, fuse=True, use_cuda_graph=True)
    made = [image(in_fmt, h, w, seed=20 + i, pitch_align=a) for i, (h, w, a) in enumerate(IN_SIZES)]
    check_transform(m, "snnb_model_transform_frame_list", "snnb_model_transform_frames", in_fmt, made, [MATRICES[i % 4] for i in range(6)], out_fmt,
                    OUT_SIZES, linear, not linear, (0.0,) * 4, (1.0,) * 4, 1.0, 0.0, pads=PADS)


@pytest.mark.parametrize("out_fmt", ["nv12", "rgba8", "p010"])
@pytest.mark.parametrize("name", ["espcn", "rgba4"])
def test_transform_1_and_4_channel_outputs(ctx, model_dir, name, out_fmt):
    m = espcn(ctx, model_dir, hw=(24, 40), batch=4) if name == "espcn" else rgba4(ctx, model_dir, 4)
    made = [image("nv12", h, w, seed=30 + i, pitch_align=a) for i, (h, w, a) in enumerate([(24, 40, 1), (51, 33, 64), (2, 2, 1), (80, 120, 128)])]
    check_transform(m, "snnb_model_transform_frame_list", "snnb_model_transform_frames", "nv12", made, MATRICES, out_fmt,
                    [(24, 40), (7, 9), (72, 120), (80, 120)], True, True, (0.0,) * 4, (1.0 / 255.0,) * 4, 300.0, -20.0, pads=[2, 0, 9, 1])


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("in_fmt,out_fmt", [("nv12", "nv12"), ("nv21", "i420"), ("i420", "nv21"), ("p010", "p010")])
def test_luma_equals_the_batch_call_per_image_and_in_place_equals_out_of_place(ctx, model_dir, in_fmt, out_fmt, linear):
    m = espcn(ctx, model_dir, hw=(24, 40), batch=4)
    sizes = [(24, 40, 1), (47, 63, 64), (1, 1, 1), (90, 160, 32)]
    made = [image(in_fmt, h, w, seed=40 + i, pitch_align=a) for i, (h, w, a) in enumerate(sizes)]
    mean4, norm4 = (LMEAN,) * 4, (LNORM,) * 4
    check_transform(m, "snnb_model_transform_luma_list", "snnb_model_transform_luma", in_fmt, made, ["bt601"] * 4, out_fmt,
                    [(48, 80), (47, 63), (3, 5), (45, 80)], linear, linear, mean4, norm4, 219.0, 16.0, pads=[0, 7, 2, 11])
    # in place: out image i is input image i itself, and equals the out-of-place result at the input's own size
    frames = [f for _, f in made]
    outs = [OutFrames(in_fmt, 1, f.height, f.width) for f in frames]
    fl, keep = frame_list(in_fmt, frames, ["bt601"] * 4, linear, mean4, norm4)
    ol, keep2 = out_list(in_fmt, outs, linear, 219.0, 16.0)
    call("snnb_model_transform_luma_list", m, C.byref(fl), C.byref(ol))
    want = [o.planes() for o in outs]
    images = (_lib.FrameOutImage * 4)()
    for i, f in enumerate(frames):
        images[i].plane, images[i].pitch, images[i].width, images[i].height = f.plane, f.pitch, f.width, f.height
    call("snnb_model_transform_luma_list", m, C.byref(fl), C.byref(_lib.FrameOutList(FORMATS[in_fmt], 4, images, int(linear), 219.0, 16.0)))
    for i, ((buf, f), w) in enumerate(zip(made, want)):
        b = host(buf).reshape(-1).view(np.uint8)
        base = buf.data_ptr()
        for p, ((rows, cols), wp) in enumerate(zip(plane_shapes(in_fmt, f.height, f.width), w)):
            off = f.plane[p] - base
            idx = off + np.arange(rows)[:, None] * f.pitch[p] + np.arange(cols)[None, :]
            assert np.array_equal(b[idx], wp[0]), "image %d plane %d: in place differs from out of place" % (i, p)


def test_python_wrappers(ctx, model_dir):
    m = espcn(ctx, model_dir, hw=(24, 40), batch=3)
    from test_frames_gpu import packed, random_yuv
    ts = [packed("nv12", *random_yuv(1, h, w, seed=50 + h))[0] for h, w in ((24, 40), (60, 90), (12, 20))]
    hw = [(48, 80), (60, 90), (4, 6)]
    got = m.transform_luma_list(ts, mean=LMEAN, norm=LNORM, out_scale=219.0, out_offset=16.0, out_hw=hw)
    for i, t in enumerate(ts):
        want = m.transform_luma(t[None].expand(3, -1, -1), mean=LMEAN, norm=LNORM, out_scale=219.0, out_offset=16.0, out_hw=hw[i])
        assert np.array_equal(host(got[i]), host(want)[0]), i
    same = [t.clone() for t in ts]
    ref = m.transform_luma_list(ts, mean=LMEAN, norm=LNORM)
    assert all(a is b for a, b in zip(m.transform_luma_list(same, mean=LMEAN, norm=LNORM, out=same), same))
    for r, s in zip(ref, same):
        assert np.array_equal(host(r), host(s))
    c = candy(ctx, model_dir, 3)
    got = c.transform_frame_list(ts, out_format="rgba8", out_hw=[(10, 12), (48, 64), (5, 3)])
    assert [tuple(g.shape) for g in got] == [(10, 12, 4), (48, 64, 4), (5, 3, 4)]
    for i, t in enumerate(ts):
        want = c.transform_frames(t[None].expand(3, -1, -1), out_format="rgba8", out_hw=got[i].shape[:2])
        assert np.array_equal(host(got[i]), host(want)[0]), i
    s = conv_model(ctx, model_dir, 3, 5, batch=3)
    labels = s.segment_frame_list(ts)
    for i, t in enumerate(ts):
        assert np.array_equal(host(labels[i]), host(s.segment_frames(t[None].expand(3, -1, -1)))[0]), i
    with pytest.raises(ValueError):
        m.transform_luma_list(ts[:2])


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("classes,luma", [(5, False), (21, False), (1, False), (5, True), (1, True)])
def test_segment_equals_the_batch_call_per_image(ctx, model_dir, classes, luma, linear):
    m = conv_model(ctx, model_dir, 1 if luma else 3, classes, batch=5)
    made = [image("nv12", h, w, seed=60 + i, pitch_align=a) for i, (h, w, a) in enumerate([(24, 40, 1), (91, 121, 64), (1, 1, 1), (50, 70, 32), (13, 7, 1)])]
    frames = [f for _, f in made]
    sizes = [(24, 40), (91, 121), (1, 97), (25, 41), (60, 20)]
    mean4, norm4 = (LMEAN,) * 4, (LNORM,) * 4
    threshold = 0.0
    fl, keep = frame_list("nv12", frames, MATRICES + ["bt601"], True, mean4, norm4)
    outs = [OutLabels(1, h, w, pad=i * 3) for i, (h, w) in enumerate(sizes)]
    ll, keep2 = labels_list(outs, linear, threshold)
    _lib.check(_lib.lib().snnb_model_segment_frame_list(m.h, C.byref(fl), int(luma), C.byref(ll), m._torch_stream()), "snnb_model_segment_frame_list")
    got = [o.labels() for o in outs]
    for i, (f, mat) in enumerate(zip(frames, MATRICES + ["bt601"])):
        ref = OutLabels(5, *sizes[i], pad=1)
        _lib.check(_lib.lib().snnb_model_segment_frames(m.h, C.byref(repeated(f, mat, True, mean4, norm4)), int(luma), C.byref(ref.batch(linear, threshold)),
                                                        m._torch_stream()), "snnb_model_segment_frames")
        want = ref.labels()
        assert np.array_equal(got[i][0], want[0]) and np.array_equal(got[i][0], want[4]), "image %d" % i
    if classes > 1:
        assert len(np.unique(got[1])) > 1


@pytest.mark.parametrize("precision", ["fp32x3", "fp16"])
def test_graph_and_fused_models_and_a_new_stream(ctx, model_dir, precision):
    m = candy(ctx, model_dir, 4, fuse=True, use_cuda_graph=True, precision=precision)
    made = [image("nv12", h, w, seed=70 + i, pitch_align=a) for i, (h, w, a) in enumerate([(48, 64, 1), (72, 128, 64), (9, 11, 1), (100, 60, 32)])]
    sizes = [(48, 64), (144, 256), (9, 11), (50, 30)]
    got = check_transform(m, "snnb_model_transform_frame_list", "snnb_model_transform_frames", "nv12", made, MATRICES, "nv12", sizes, True, True,
                          (0.0,) * 4, (1.0,) * 4, 1.0, 0.0)
    fl, keep = frame_list("nv12", [f for _, f in made], MATRICES)
    outs = [OutFrames("nv12", 1, h, w) for h, w in sizes]
    ol, keep2 = out_list("nv12", outs, True, 1.0, 0.0)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(100_000_000)
        call("snnb_model_transform_frame_list", m, C.byref(fl), C.byref(ol), stream=s.cuda_stream)
    for g, o in zip(got, outs):
        assert_same([p[0] for p in o.planes()], [p[0] for p in g], "on a new stream")


def tiny(ctx, tmp_path, batch):
    b = modelzoo.Builder(seed=5)
    b.batchnorm(b.input(2, 2, 3))
    return core.MixedInferenceCore(ctx, modelzoo.write_model(b.layers, str(tmp_path / "tiny_out.json")), batch=batch)


def test_list_of_256_images_is_accepted_and_257_is_refused(ctx, tmp_path):
    m = tiny(ctx, tmp_path, 256)
    made = [image("nv12", 1 + i % 7, 1 + i % 5, seed=i) for i in range(257)]
    frames = [f for _, f in made]
    fl, keep = frame_list("nv12", frames[:256], [MATRICES[i % 4] for i in range(256)])
    outs = [OutFrames("nv12", 1, 1 + i % 3, 2 + i % 4) for i in range(257)]
    ol, keep2 = out_list("nv12", outs[:256], True, 100.0, 0.0)
    call("snnb_model_transform_frame_list", m, C.byref(fl), C.byref(ol))
    for i in (0, 5, 255):
        ref = OutFrames("nv12", 256, outs[i].h, outs[i].w)
        call("snnb_model_transform_frames", m, C.byref(repeated(frames[i], MATRICES[i % 4], True, (0.0,) * 4, (1.0,) * 4)), C.byref(ref.batch(True, 100.0, 0.0)))
        assert_same([p[0] for p in outs[i].planes()], [p[i] for p in ref.planes()], "image %d" % i)
    big, keep3 = frame_list("nv12", frames, [MATRICES[i % 4] for i in range(257)])
    bol, keep4 = out_list("nv12", outs, True, 100.0, 0.0)
    with pytest.raises(SnnbError, match="count 257"):
        call("snnb_model_transform_frame_list", m, C.byref(big), C.byref(bol))


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")
def test_refusals_launch_nothing_and_write_nothing(ctx, model_dir, tmp_path):
    m = candy(ctx, model_dir, 3, fuse=True, use_cuda_graph=True)
    lm = espcn(ctx, model_dir, hw=(24, 40), batch=3)
    sm = conv_model(ctx, model_dir, 3, 5, batch=3)
    made = [image("nv12", h, w, seed=80 + i, pitch_align=64) for i, (h, w) in enumerate([(24, 40), (30, 50), (10, 12)])]
    frames = [f for _, f in made]
    fl, keep = frame_list("nv12", frames, MATRICES[:3])
    made10 = [image("p010", 10, 12, seed=i) for i in range(3)]
    fl10, keep10 = frame_list("p010", [f for _, f in made10], MATRICES[:3])
    outs = [OutFrames("nv12", 1, 20, 30) for _ in range(3)]
    labels = [OutLabels(1, 20, 30) for _ in range(3)]

    def refused(fn, text):
        before = ctx.launches
        with pytest.raises(SnnbError) as e:
            fn()
        assert text in str(e.value), str(e.value)
        assert ctx.launches == before, "a refused call launched kernels"
        for o in outs:
            assert (host(o.buf) == FILL).all(), "a refused call wrote"
        for o in labels:
            assert (host(o.buf) == FILL).all(), "a refused call wrote"

    def ol(fmt="nv12", n=3, **kw):
        lst, images = out_list(fmt, outs[:n], True, 1.0, 0.0)
        for k, (i, val) in kw.items():
            if k in ("plane", "pitch"):
                getattr(images[i], k)[val[0]] = val[1]
            else:
                setattr(images[i], k, val)
        ol.keep = images
        return lst

    tf = lambda model, f, o: call("snnb_model_transform_frame_list", model, C.byref(f) if f is not None else None, C.byref(o) if o is not None else None)  # noqa: E731
    tl = lambda f, o: call("snnb_model_transform_luma_list", lm, C.byref(f), C.byref(o))  # noqa: E731
    for name, run in (("snnb_model_transform_frame_list", lambda o: tf(m, fl, o)), ("snnb_model_transform_luma_list", lambda o: tl(fl, o))):
        refused(lambda: run(ol(n=2)), "%s: out count 2; the out list must hold one image per frame (3)" % name)
        o = ol()
        o.images = None
        refused(lambda: run(o), "%s: null out images" % name)
        o = ol()
        o.format = 4
        refused(lambda: run(o), "%s: unknown out frame format 4" % name)
        refused(lambda: run(ol(width=(1, 0))), "%s: image 1: out frame size 0 x 20; width and height must be >= 1" % name)
        refused(lambda: run(ol(pitch=(2, (1, 29)))), "%s: image 2 out plane 1: pitch 29 is less than its row's 30 bytes" % name)
        refused(lambda: run(ol(plane=(0, (0, np.zeros(4096, np.uint8).ctypes.data)))), "image 0 out plane 0: ")
        pinned = torch.zeros(4096, dtype=torch.uint8).pin_memory()
        refused(lambda: run(ol(plane=(1, (1, pinned.data_ptr())))), "pinned host memory")
        p10 = [OutFrames("p010", 1, 10, 12) for _ in range(3)]
        o10, k10 = out_list("p010", p10, True, 1.0, 0.0)
        k10[1].pitch[0] = 25
        src = fl10 if "luma" in name else fl
        refused(lambda: (tf(m, src, o10) if "frame_list" in name else tl(src, o10)), "image 1 out plane 0: P010 pitch 25 and image stride 0 must be even")
        refused(lambda: call(name, m if "frame_list" in name else lm, C.byref(fl), None), "%s: null out" % name)
        g = torch.cuda.CUDAGraph()

        def capture():
            with torch.cuda.graph(g, capture_error_mode="relaxed"):
                run(ol())
        refused(capture, "being captured")
    refused(lambda: tf(m, frame_list("nv12", frames[:2], MATRICES[:2])[0], ol(n=2)), "count 2; the list must hold the model's batch of 3 images")
    refused(lambda: tf(sm, fl, ol()), "output 0 has 5 channels; frames are written from 1 (grey), 3 (RGB) or 4 (RGBA)")
    refused(lambda: tf(m, None, ol()), "snnb_model_transform_frame_list: null frames")
    # luma: bit depths, RGBA8 on either side, a 3-channel model, and an out plane on another image's source chroma
    refused(lambda: tl(fl, ol(fmt="p010")), "the bit depths differ")
    refused(lambda: tl(fl10, ol()), "the bit depths differ")
    refused(lambda: tl(fl, ol(fmt="rgba8")), "out format RGBA8 has no Y plane")
    rgba = [image("rgba8", 10, 12, seed=i) for i in range(3)]
    refused(lambda: tl(frame_list("rgba8", [f for _, f in rgba], MATRICES[:3])[0], ol()), "RGBA8 frames have no Y plane")
    refused(lambda: call("snnb_model_transform_luma_list", m, C.byref(fl), C.byref(ol())), "the model input has 3 channels; the Y plane feeds exactly 1")
    refused(lambda: tl(fl, ol(plane=(1, (0, frames[0].plane[1] + 8)))), "image 1 out plane 0 overlaps image 0 source chroma plane 1")
    refused(lambda: tl(fl, ol(plane=(2, (1, frames[2].plane[1])))), "image 2 out plane 1 overlaps image 2 source chroma plane 1")
    # segment
    sl = lambda model, lst, luma=0: call("snnb_model_segment_frame_list", model, C.byref(fl), luma, C.byref(lst) if lst is not None else None)  # noqa: E731

    def ll(n=3, **kw):
        lst, images = labels_list(labels[:n], True, 0.5)
        for k, (i, val) in kw.items():
            setattr(images[i], k, val)
        ll.keep = images
        return lst

    name = "snnb_model_segment_frame_list"
    refused(lambda: sl(sm, ll(n=2)), "%s: out count 2; the out list must hold one image per frame (3)" % name)
    o = ll()
    o.images = None
    refused(lambda: sl(sm, o), "%s: null out images" % name)
    refused(lambda: sl(sm, None), "%s: null out" % name)
    refused(lambda: sl(sm, ll(height=(1, 0))), "%s: image 1: label plane size 30 x 0; width and height must be >= 1" % name)
    refused(lambda: sl(sm, ll(pitch=(2, 29))), "%s: image 2: label plane pitch 29 is less than its width 30" % name)
    refused(lambda: sl(sm, ll(plane=(0, np.zeros(4096, np.uint8).ctypes.data))), "image 0 label plane 0: ")
    refused(lambda: sl(sm, ll(), luma=1), "the model input has 3 channels; the Y plane feeds exactly 1")
    from test_rois_gpu import load_yolo
    yolo = load_yolo(ctx, model_dir, "planted", batch=3)
    refused(lambda: sl(yolo, ll()), "output 0 is a YOLO detection list")
    refused(lambda: tf(yolo, fl, ol()), "output 0 is a YOLO detection list")
    # the models are still usable
    tf(m, fl, ol())
    sl(sm, ll())
    torch.cuda.synchronize()
