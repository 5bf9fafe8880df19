"""Count-sized region batches (snnb_model_set_count_batches, MixedInferenceCore.set_count_batches): once sizes are declared, run_rois and
run_rois_list with a device-side count run the forward pass at the size a selector kernel picks from the count on the GPU, through one
CUDA graph of conditional (IF) nodes per model batch.

The oracle is the same handle after set_batch(s), s the size the count selects (snnb_debug_count_body, held to a restatement on the CPU),
with no sizes declared: slot i < s of the counted call must equal it byte for byte, in every output dtype and the classes, and every slot
>= the count must be zero. Also: a count of 0 runs no forward pass, calls without a count are unchanged, counted calls queued back to back
on a caller's stream each see their own count, the detector chain on a new stream equals the synchronised chain, and refused calls change
nothing."""
import ctypes as C

import numpy as np
import pytest

from shadernn_b200 import _lib
from shadernn_b200._lib import SnnbError
from test_count_batches_cpu import restated
from test_frames_gpu import NORM, host, load
from test_partial_batch_gpu import nv12
from test_rois_gpu import cuda_i32, load_yolo

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

HW, B = (112, 112), 64
SIZES = [1, 4, 8, 16, 32]
COUNTS = [1, 3, 4, 5, 8, 9, 16, 17, 32, 33, 63, 64, 100, -2]
MEAN4, NORM4 = NORM["resnet18"]
FH, FW, NF = 180, 320, 4  # NV12 frames of the batch form
LIST_HW = [(180, 320), (96, 128), (240, 200), (120, 160)]  # the frame list's mixed sizes
DTYPES = [None, torch.float16, torch.uint8]


def test_driver_version_is_on_record():
    v = C.c_int()
    assert C.CDLL("libcuda.so.1").cuDriverGetVersion(C.byref(v)) == 0  # what cudaDriverGetVersion reports
    print("CUDA driver version %d.%d (conditional graph nodes need 12.3)" % (v.value // 1000, v.value % 1000 // 10))
    assert v.value >= 12030


def regions(sizes_hw, n, seed):
    """n caller-made regions, each inside its frame (frame i % len(sizes_hw)), of varied sizes and origins."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        f = i % len(sizes_hw)
        h, w = sizes_hw[f]
        rw, rh = int(rng.integers(1, w + 1)), int(rng.integers(1, h + 1))
        out.append((f, i, int(rng.integers(0, w - rw + 1)), int(rng.integers(0, h - rh + 1)), rw, rh))
    return cuda_i32(out)


def classifier(ctx, model_dir, batch=B, **kw):
    opts = dict(fuse=True, use_cuda_graph=True)
    opts.update(kw)
    return load(ctx, model_dir, "resnet18", HW, batch, **opts)


def call(m, frames, rois, count, out_dtype=None):
    """run_rois (frames a batch tensor) or run_rois_list (frames a list): (output 0, classes), both on the host."""
    kw = dict(mean4=MEAN4, norm4=NORM4, out_dtype=out_dtype, want_classes=True)
    c = None if count is None else cuda_i32([count])
    out, cls = (m.run_rois_list if isinstance(frames, list) else m.run_rois)(frames, rois, c, **kw)
    return host(out), host(cls)


def same(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape)
    assert got.tobytes() == want.tobytes(), "%s: %d of %d bytes differ" % (what, int((got.view(np.uint8) != want.view(np.uint8)).sum()), got.nbytes)


def check_counts(m, frames, rois, sizes, counts, dtypes=DTYPES):
    """Each count's counted call (sizes declared) against set_batch(s) with the same count and no declaration; returns the counted results."""
    b = m.batch
    m.set_count_batches(sizes)
    got = {(c, dt): call(m, frames, rois, c, dt) for c in counts for dt in dtypes}
    m.set_count_batches([])
    for c in counts:
        s = restated(sizes, b, c)
        used = min(max(c, 0), b)
        if s:
            m.set_batch(s)
        for dt in dtypes:
            out, cls = got[(c, dt)]
            assert not out[used:].view(np.uint8).any() and not cls[used:].any(), (c, dt)
            if s:
                want, wcls = call(m, frames, rois[:s], c, dt)
                same(out[:s], want, "count %d, size %d, dtype %s" % (c, s, dt))
                same(cls[:s], wcls, "classes, count %d" % c)
                assert (cls[:used] >= 1).all(), c
        m.set_batch(b)
    return got


def test_run_rois_bit_exact_against_set_batch(ctx, model_dir):
    m = classifier(ctx, model_dir)
    frames = nv12(FH, FW, 1, n=NF)
    check_counts(m, frames, regions([(FH, FW)] * NF, B, 2), SIZES, COUNTS)
    m.close()


def test_run_rois_list_bit_exact_against_set_batch(ctx, model_dir):
    m = classifier(ctx, model_dir)
    flist = [nv12(h, w, 10 + i) for i, (h, w) in enumerate(LIST_HW)]
    check_counts(m, flist, regions(LIST_HW, B, 3), SIZES, [1, 5, 16, 33, 64, 0])
    m.close()


@pytest.mark.parametrize("kw", [dict(precision="fp16"), dict(fuse=False)], ids=["fp16", "unfused"])
def test_other_model_options(ctx, model_dir, kw):
    m = classifier(ctx, model_dir, **kw)
    frames = nv12(FH, FW, 4, n=NF)
    check_counts(m, frames, regions([(FH, FW)] * NF, B, 5), SIZES, [1, 4, 9, 33, 64], dtypes=[None])
    m.close()


def test_a_batch_below_some_declared_sizes(ctx, model_dir):
    m = classifier(ctx, model_dir)
    m.set_batch(12)
    frames = nv12(FH, FW, 6, n=NF)
    rois = regions([(FH, FW)] * NF, 12, 7)
    assert [restated([4, 8, 16], 12, c) for c in (1, 4, 5, 8, 9, 12, 20)] == [4, 4, 8, 8, 12, 12, 12]  # bodies 4, 8 and 12
    check_counts(m, frames, rois, [4, 8, 16], [1, 4, 5, 8, 9, 12, 20], dtypes=[None])
    m.close()


def test_count_zero_runs_no_forward_pass(ctx, model_dir):
    from torch.profiler import ProfilerActivity, profile
    m = classifier(ctx, model_dir)
    frames = nv12(FH, FW, 8, n=NF)
    rois = regions([(FH, FW)] * NF, B, 9)
    m.set_count_batches(SIZES)
    for c in (0, 1):  # build and warm up
        call(m, frames, rois, c)

    def kernels(count):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out, cls = call(m, frames, rois, count)
            torch.cuda.synchronize()
        return [e.key for e in prof.key_averages()], out, cls
    names0, out, cls = kernels(0)
    assert not out.view(np.uint8).any() and not cls.any()
    assert any("count_select_kernel" in n for n in names0) and any("roi_clear_kernel" in n for n in names0), names0
    assert not any("conv" in n or "gap_dense" in n for n in names0), [n for n in names0 if "conv" in n or "gap_dense" in n]
    names1, _, _ = kernels(1)
    assert any("conv" in n for n in names1)  # the profiler does see the forward pass's kernels inside the IF bodies
    m.close()


def test_calls_without_a_count_are_unchanged(ctx, model_dir):
    m = classifier(ctx, model_dir)
    frames = nv12(FH, FW, 11, n=NF)
    rois = regions([(FH, FW)] * NF, B, 12)
    plain, counted = call(m, frames, rois, None), call(m, frames, rois, 5)
    m.set_count_batches(SIZES)
    got = call(m, frames, rois, None)
    same(got[0], plain[0], "no count, sizes declared"), same(got[1], plain[1], "no count, sizes declared")
    m.set_count_batches([])
    for what, got, want in (("no count, cleared", call(m, frames, rois, None), plain), ("count, cleared", call(m, frames, rois, 5), counted)):
        same(got[0], want[0], what), same(got[1], want[1], what)
    m.close()


def test_redeclaring_and_clearing(ctx, model_dir):
    m = classifier(ctx, model_dir)
    frames = nv12(FH, FW, 13, n=NF)
    rois = regions([(FH, FW)] * NF, B, 14)
    check_counts(m, frames, rois, [8, 16], [3, 9, 20], dtypes=[None])
    check_counts(m, frames, rois, [2, 40], [3, 9, 20, 41], dtypes=[None])  # new sizes replace the old ones, graphs rebuilt
    base = ctx.launches
    m.set_count_batches([16])
    call(m, frames, rois, 3)
    counted = ctx.launches - base
    m.set_count_batches([])
    base = ctx.launches
    call(m, frames, rois, 3)
    assert counted == ctx.launches - base + 1  # the selector; the forward pass is counted at the model's batch either way
    m.close()


def test_counted_calls_queued_on_a_caller_stream(ctx, model_dir):
    m = classifier(ctx, model_dir)
    frames = nv12(FH, FW, 15, n=NF)
    rois = regions([(FH, FW)] * NF, B, 16)
    m.set_count_batches(SIZES)
    counts = [33, 1, 0, 9, 64, 4, 17]
    want = [call(m, frames, rois, c) for c in counts]  # synchronised, one at a time
    s = torch.cuda.Stream()
    got = []
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)  # the host queues every call long before the first one runs
        for c in counts:
            cnt = torch.empty(1, dtype=torch.int32, device="cuda")
            cnt.fill_(c)  # written by a kernel on the caller's stream
            got.append(m.run_rois(frames, rois, cnt, mean4=MEAN4, norm4=NORM4, want_classes=True))
    s.synchronize()
    for c, (out, cls), (wout, wcls) in zip(counts, got, want):
        same(host(out), wout, "count %d" % c), same(host(cls), wcls, "classes, count %d" % c)
    m.close()


def test_detector_chain_on_a_new_stream(ctx, model_dir):
    det = load_yolo(ctx, model_dir, "planted", batch=len(LIST_HW))
    m = classifier(ctx, model_dir)
    m.set_count_batches(SIZES)
    dmean, dnorm = NORM["yolov3tiny"]
    flist = [nv12(h, w, 20 + i) for i, (h, w) in enumerate(LIST_HW)]

    def chain(min_score):
        r, c = det.detect_frame_list(flist, mean4=dmean, norm4=dnorm)
        rois, count = ctx.rois_from_detections(r, c, LIST_HW, B, min_score=min_score)
        out, cls = m.run_rois_list(flist, rois, count, mean4=MEAN4, norm4=NORM4, want_classes=True)
        return out, cls, count
    seen = set()
    for min_score in (0.0, 0.3, 0.6, 0.9):
        torch.cuda.synchronize()
        want = [host(t) for t in chain(min_score)]
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)
            got = chain(min_score)
        s.synchronize()
        for g, w in zip(got, want):
            same(host(g), w, "min_score %g" % min_score)
        seen.add(int(want[2][0]))
    assert len(seen) >= 2, seen  # the thresholds leave different counts
    det.close(), m.close()


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")
def test_refusals_change_nothing(ctx, model_dir):
    m = classifier(ctx, model_dir)
    frames = nv12(FH, FW, 17, n=NF)
    rois = regions([(FH, FW)] * NF, B, 18)
    m.set_count_batches([4, 16])
    want = call(m, frames, rois, 3)
    base = ctx.launches
    call(m, frames, rois, 3)
    per_call = ctx.launches - base
    for bad, text in (([4, 2], "sizes[1] = 2; sizes must be strictly increasing"), ([4, 4], "sizes[1] = 4"), ([0, 4], "sizes[0] = 0"),
                      ([8, B + 1], "sizes[1] = %d; sizes must be strictly increasing, from 1 to the loaded batch of %d" % (B + 1, B)),
                      (list(range(1, 35)), "34 sizes; 0 to 32 may be declared")):
        with pytest.raises(SnnbError) as e:
            m.set_count_batches(bad)
        assert text in str(e.value), str(e.value)
    base = ctx.launches
    got = call(m, frames, rois, 3)
    assert ctx.launches - base == per_call  # the declaration (and its graph) survived
    same(got[0], want[0], "after refusals"), same(got[1], want[1], "classes after refusals")

    eager = classifier(ctx, model_dir, use_cuda_graph=False)
    with pytest.raises(SnnbError, match="loaded without use_cuda_graph"):
        eager.set_count_batches([4])
    eager.close()

    # a counted call while the context's stream is being captured
    lib = _lib.lib()
    out, obufs, classes = m._device_outputs("test", None, "nhwc", 1.0, 0.0, True)
    for o in (out[0], classes):
        o.view(torch.uint8).fill_(0x5A)
    f, n = m._frames_any("test", frames, "nv12", "bt601", True, MEAN4, NORM4)
    cnt = cuda_i32([3])
    torch.cuda.synchronize()
    base = ctx.launches
    _lib.check(lib.snnb_graph_capture_begin(ctx.h))
    rc = lib.snnb_model_run_rois(m.h, C.byref(f), n, rois.data_ptr(), cnt.data_ptr(), obufs, 1, classes.data_ptr(), None)
    msg = lib.snnb_last_error().decode()
    g = C.c_void_p()
    if lib.snnb_graph_capture_end(ctx.h, C.byref(g)) == 0:
        lib.snnb_graph_destroy(g)
    assert rc != 0 and "is being captured (snnb_graph_capture_begin)" in msg, msg
    assert ctx.launches == base
    assert (host(out[0]).view(np.uint8) == 0x5A).all() and (host(classes).view(np.uint8) == 0x5A).all()
    got = call(m, frames, rois, 3)
    same(got[0], want[0], "after the refused capture")
    m.close()
