"""The sampled restatement behind test_bench_exact_gpu.py, without a GPU: exact.f(..., at=S) is exact.f(...) at S bit for bit, the
chosen pixels cover every tile of every convolution launch of the benchmark's batches, and a defect confined to one tile is caught."""
import numpy as np
import pytest

import test_bench_exact_gpu as tb
import test_conv_plan as cp
from oracle import exact, oracle
from shadernn_b200 import modelzoo

RNG = np.random.default_rng(5)


def _x(n, h, w, c, lo=-1.0, hi=1.0, seed=0):
    return exact.stored(np.random.default_rng(seed).uniform(lo, hi, (n, h, w, c)), False)


def _at(n, oh, ow, count, seed=1):
    """`count` random output pixels in random order, with repeats, plus the four corners of the last image."""
    rng = np.random.default_rng(seed)
    at = [rng.integers(0, d, count) for d in (n, oh, ow)]
    return tuple(np.concatenate([a, [n - 1] * 4 if i == 0 else ([0, 0, d - 1, d - 1] if i == 1 else [0, d - 1, 0, d - 1])])
                 for i, (a, d) in enumerate(zip(at, (n, oh, ow))))


def _same(full, part, at):
    for f, p in zip(full, part):
        assert p.dtype == np.float64 and np.array_equal(f[at], p, equal_nan=True), np.max(np.abs(f[at] - p))
        assert np.array_equal(np.signbit(f[at]), np.signbit(p))


BN = {"gamma": RNG.uniform(0.5, 1.5, 24), "beta": RNG.uniform(-0.5, 0.5, 24), "mean": RNG.uniform(-0.2, 0.2, 24), "var": RNG.uniform(0.5, 2, 24)}


# (kernel, form, n, h, w, ic, oc, k, stride, pad, pad_mode, residual, act): every K order, the three pad modes, stride 2, a residual,
# and more output pixels than exact.ROWS so that the full restatement spans several row blocks
CONV_CASES = [
    ("igemm", "fp32x3", 2, 40, 37, 20, 24, 3, 1, 1, "constant", False, "relu"),
    ("igemm", "fp16w", 2, 19, 21, 70, 24, 3, 2, 1, "replicate", True, "leakyRelu"),
    ("igemm", "fp16", 3, 9, 11, 16, 24, 1, 1, 0, "constant", True, ""),
    ("rowwin", "fp32x3", 2, 41, 30, 3, 24, 5, 1, 2, "reflect", False, "tanh"),
    ("rowwin", "fp16w", 1, 23, 29, 4, 24, 3, 2, 1, "constant", False, "SiLU"),
    ("feed", "fp32x3", 2, 33, 35, 3, 24, 7, 2, 3, "constant", False, "relu6"),
    ("simt", "simt", 2, 15, 13, 9, 24, 3, 1, 1, "reflect", True, "sigmoid"),
]


@pytest.mark.parametrize("case", CONV_CASES, ids=["%s-%s-k%d-s%d-%s%s" % (c[0], c[1], c[7], c[8], c[10], "-res" if c[11] else "") for c in CONV_CASES])
def test_conv2d_sampled_equals_full(case):
    kernel, form, n, h, w, ic, oc, k, s, p, mode, res, act = case
    x = _x(n, h, w, ic)
    wt = RNG.uniform(-0.5, 0.5, (oc, ic, k, k)).astype(np.float32)
    b = RNG.uniform(-0.1, 0.1, oc).astype(np.float32)
    oh, ow = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    r = _x(n, oh, ow, oc, seed=3) if res else None
    kw = dict(act=act, alpha=0.1, residual=r, form=form, kernel=kernel, half_out=form == "fp16", pad_mode=mode)
    full = exact.conv2d(x, wt, b, BN, s, p, p, (oh, ow), **kw)
    at = _at(n, oh, ow, 300)
    _same(full, exact.conv2d(x, wt, b, BN, s, p, p, (oh, ow), at=at, **kw), at)


def test_layers_sampled_equal_full():
    n, h, w, c = 2, 13, 17, 24
    x, y = _x(n, h, w, c), _x(n, h, w, c, seed=2)
    g, be = RNG.uniform(0.5, 1.5, c), RNG.uniform(-0.5, 0.5, c)
    wd = RNG.uniform(-0.5, 0.5, (c, 3, 3)).astype(np.float32)
    dk = RNG.uniform(-0.5, 0.5, (7, c)).astype(np.float32)
    at = _at(n, h, w, 120)
    for act in ("", "relu", "leakyRelu", "tanh", "sigmoid"):
        for half in (False, True):
            _same(exact.add(x, y, act, 0.1, half), exact.add(x, y, act, 0.1, half, at), at)
            _same(exact.batchnorm(x, BN, act, 0.1, half), exact.batchnorm(x, BN, act, 0.1, half, at), at)
            _same(exact.activation(x, act, 0.1, half), exact.activation(x, act, 0.1, half, at), at)
            _same(exact.instancenorm(x * 40 + 3, g, be, act, 0.1, half), exact.instancenorm(x * 40 + 3, g, be, act, 0.1, half, at), at)
    for s, p in ((1, 1), (2, 1), (2, 0)):
        ohw = ((h + 2 * p - 3) // s + 1, (w + 2 * p - 3) // s + 1)
        a2 = _at(n, *ohw, 60)
        _same(exact.depthwise(x, wd, None, BN, s, p, p, ohw, "relu6"), exact.depthwise(x, wd, None, BN, s, p, p, ohw, "relu6", at=a2), a2)
    for k, s in ((2, 2), (3, 2), (3, 1)):
        ohw = (-(-h // s), -(-w // s))
        a2 = _at(n, *ohw, 60)
        _same(exact.maxpool(x, k, s, ohw), exact.maxpool(x, k, s, ohw, a2), a2)
        _same(exact.avgpool(x, k, s, ohw, True), exact.avgpool(x, k, s, ohw, True, a2), a2)
    for mode in ("constant", "replicate", "reflect"):
        a2 = _at(n, h + 3, w + 1, 60)
        _same(exact.pad(x, 0, 2, (h + 3, w + 1), mode), exact.pad(x, 0, 2, (h + 3, w + 1), mode, a2), a2)
    _same(exact.concat(x, y), exact.concat(x, y, at), at)
    a2 = _at(n, 2 * h, 2 * w, 80)
    _same(exact.upsample_nearest(x, (2 * h, 2 * w)), exact.upsample_nearest(x, (2 * h, 2 * w), a2), a2)
    _same(exact.subpixel(x[..., :4], 2), exact.subpixel(x[..., :4], 2, at=a2), a2)
    _same(exact.model_input(x, True), exact.model_input(x, True, at), at)
    _same(exact.model_input(x, False), exact.model_input(x, False, at), at)
    flat = x[:, :1, :1, :]
    a3 = (np.array([1, 0, 1]), np.zeros(3, int), np.zeros(3, int))
    _same(exact.dense(flat, dk, None, "relu", "fp16w"), exact.dense(flat, dk, None, "relu", "fp16w", at=a3), a3)


def test_sampler_is_seeded_and_covers_its_boxes():
    n, oh, ow = 3, 37, 29
    a = exact.sample_pixels(n, oh, ow, [(16, 5, 1), (8, 8, 1)], [1, 2, 3])
    assert all(np.array_equal(u, v) for u, v in zip(a, exact.sample_pixels(n, oh, ow, [(16, 5, 1), (8, 8, 1)], [1, 2, 3])))
    assert not all(np.array_equal(u, v) for u, v in zip(a, exact.sample_pixels(n, oh, ow, [(16, 5, 1), (8, 8, 1)], [1, 2, 4])))
    _assert_covers(a, n, oh, ow, (16, 5, 1), 2)
    _assert_covers(a, n, oh, ow, (8, 8, 1), 2)
    whole = exact.sample_pixels(2, 1, 1, [(1, 1, 2)], 0)  # a box of fewer pixels than asked for: all of them
    assert list(whole[0]) == [0, 1]


def _assert_covers(at, n, oh, ow, box, per_box, tiles=None):
    """At least min(per_box, box pixels) chosen pixels in every box of the grid, and every edge pixel of every image."""
    ni, oy, ox = at
    tw, th, tn = box
    tx, ty, tnn = tiles or (-(-ow // tw), -(-oh // th), -(-n // tn))
    assert (tx, ty, tnn) == (-(-ow // tw), -(-oh // th), -(-n // tn))
    tile = ((ni // tn) * ty + oy // th) * tx + ox // tw
    got = np.bincount(tile, minlength=tx * ty * tnn)
    nb, yb, xb = np.indices((tnn, ty, tx)).reshape(3, -1)
    size = np.minimum(tn, n - nb * tn) * np.minimum(th, oh - yb * th) * np.minimum(tw, ow - xb * tw)
    assert got.size == tx * ty * tnn and np.all(got >= np.minimum(size, per_box)), np.nonzero(got < np.minimum(size, per_box))[0][:10]
    mark = np.zeros((n, oh, ow), bool)
    mark[ni, oy, ox] = True
    assert mark[:, 0].all() and mark[:, -1].all() and mark[:, :, 0].all() and mark[:, :, -1].all()


def _model_shapes(key, batch):
    """oracle.Model and per-layer NHWC shapes, up to the last Conv2D, of a bench model at its default size (torch on the CPU)."""
    import tempfile
    fn, hw, _, _ = modelzoo.MODELS[key]
    with tempfile.TemporaryDirectory() as d:
        path, layers = modelzoo.build(key, d)
        om = oracle.Model(path)
    last = max(i for i, l in enumerate(layers) if l["type"] == "Conv2D")
    outs = modelzoo.torch_forward(layers, modelzoo.synthetic_input(key, 1, hw), upto=last)
    return om, [None if o is None else (batch,) + tuple(np.shape(o)[1:]) for o in outs]


@pytest.mark.parametrize("key", sorted({c[0] for c in tb.bench_cases()}))
def test_sample_covers_every_tile_of_every_bench_convolution(built, key):
    pytest.importorskip("torch")
    batches = sorted({c[1] for c in tb.bench_cases() if c[0] == key})
    om, shapes1 = _model_shapes(key, 1)
    fusion = tb.fused_convs(om)
    assert fusion
    seen = set()
    for batch in batches:
        shapes = [None if s is None else (batch,) + s[1:] for s in shapes1]
        for precision in tb.FORMS:
            for j in fusion:
                p = tb.conv_plan(tb.conv_query(om, j, fusion, shapes), batch, precision, cp.SMS)
                box = tb.tile_box(p)
                assert box is not None, (key, j, p["path"])  # every bench convolution runs on a tensor-core kernel
                n, oh, ow, _ = shapes[j]
                at = tb.choose_pixels(key, j, shapes[j], box)
                if p["path"] == cp.IGEMM:
                    tiles = (p["tiles_x"], p["tiles_y"], p["tiles_n"])
                else:
                    assert p["tiles_x"] == -(-ow // 128)
                    tiles = (p["tiles_x"], oh, n)
                _assert_covers(at, n, oh, ow, box, 2, tiles)
                seen.add((p["path"], p["ksplit"] > 1, p["sk"]))
    assert seen


def _tile_defect_case():
    """A 3-image, multi-tile Conv2D with a residual on conv_umma_kernel in fp32x3: inputs with positive lo halves and positive
    weights, so that every defect below moves an output by far more than its bound."""
    n, h, w, ic, oc, k = 3, 26, 30, 32, 24, 3
    hi = exact.f16(np.random.default_rng(0).uniform(0.5, 1.5, (n, h, w, ic))).astype(np.float32)
    x = hi + np.abs(exact.f16(np.random.default_rng(1).uniform(0.3, 1.0, hi.shape) * 2.0 ** -12 * hi)).astype(np.float32)
    wt = np.random.default_rng(2).uniform(0.05, 0.5, (oc, ic, k, k)).astype(np.float32)
    res = _x(n, h, w, oc, seed=4)
    p = cp.plan((h, w, ic), (h, w, oc), k, 1, 1, 1, residual=True, n=n)
    assert p["path"] == cp.IGEMM and p["tiles_x"] * p["tiles_y"] * p["tiles_n"] > 4
    return x, wt, res, p, (n, h, w)


def test_tile_local_defects_are_caught():
    x, wt, res, p, (n, h, w) = _tile_defect_case()
    conv = lambda xx, ww, rr, form="fp32x3": exact.conv2d(xx, ww, None, None, 1, 1, 1, (h, w), residual=rr, form=form)
    ref, bound = conv(x, wt, res)
    box = tb.tile_box(p)
    at = tb.choose_pixels("defects", 0, (n, h, w, wt.shape[0]), box)
    assert exact.check(ref[at], ref[at], bound[at], "")[1] == 0
    w_lost = wt.copy()
    w_lost[:, :, 1, 2] = 0  # one K block: the 64-channel block of tap (1, 2)
    defects = {
        "lost K block": conv(x, w_lost, res)[0],
        "dropped lo-term product": conv(exact.f16(x).astype(np.float32), wt, res)[0],
        "fp16-rounded store": exact.f16(ref),
        "residual of the neighbouring image": conv(x, wt, np.roll(res, 1, axis=0))[0],
    }
    n0, y0, x0, nn, hy, wx = exact.box_grid(n, h, w, box)
    edge = np.zeros((n, h, w), bool)
    edge[:, 0] = edge[:, -1] = edge[:, :, 0] = edge[:, :, -1] = True

    def tile_mask(t):
        mask = np.zeros((n, h, w), bool)
        mask[n0[t]:n0[t] + nn[t], y0[t]:y0[t] + hy[t], x0[t]:x0[t] + wx[t]] = True
        return mask

    # the last tile of the last image, whole; and the middle tile of the middle image without its edge pixels, which stay right, so
    # that only the tile's random pixels can see the defect there
    middle = np.nonzero(n0 == n // 2)[0]
    assert box[2] == 1 and len(middle) >= 3
    tiles = {"last tile": tile_mask(len(n0) - 1), "middle tile, off the edges": tile_mask(middle[len(middle) // 2]) & ~edge}
    for where, mask in tiles.items():
        assert mask.any()
        for what, bad in defects.items():
            got = np.where(mask[..., None], bad, ref)
            assert exact.check(got[at], ref[at], bound[at], what)[1] > 0, (what, where)


def test_case_table_is_the_benchmark():
    import bench
    from shadernn_b200 import parallel
    cases = tb.bench_cases()
    assert {(c[0], c[1]) for c in cases if c[3] == 0} == {(v[0], v[1]) for v in bench.WORKLOADS.values()}
    assert {c[2] for c in cases if c[3] == 0} == set(tb.FORMS) and len([c for c in cases if c[3] == 0]) == len(bench.WORKLOADS) * len(tb.FORMS)
    strong = {c[0]: c[1] for c in cases if c[3] != 0}
    assert strong == {"mobilenetv2": 8, "yolov3tiny": 2, "candy": 1}
    for key, count in strong.items():
        assert parallel.shard_range(bench.WORKLOADS[key][1], tb.WORLD, tb.WORLD - 1)[1] == count
    assert all(c[0] in modelzoo.MODELS for c in cases)
