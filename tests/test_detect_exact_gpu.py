"""The YOLO decode, score order and NMS held to oracle/exact.py's two statements of them, on every detection entry point.

- The float32 contract decides: the rows of detect_device and detect_torch must equal exact.yolo_contract of the engine's own stored
  heads (layer_output of the two head layers) bit for bit: counts, order and every float.
- The float64 definition checks the contract: every row value lies within exact.yolo_define's bound, and every threshold, order and
  suppression decision whose float64 margin exceeds its bound is the one the contract made (exact.yolo_decisions). No decision inside
  its bound is asserted from float64.
- The host path (run() + boxes(n)) takes glibc's expf: its rows are held to the definition's bounds and to the contract's decisions
  wherever they are certain.

Planted heads: two model inputs go through a 1x1 identity Conv2D each into a YOLO layer, so the stored heads are the planted values (an
identity product of storage-representable values is exact in every form; the test asserts it). The planting searches values the
form can store for a score of exactly 0.35f (rejected) and one fp32 ulp above, an IoU of exactly 0.45f (kept) and one ulp above, exact
score ties across heads and anchors, and values past fp16's range (w, h = inf; score exactly 1) and NaN pixels. Where the form's
spacing cannot hit an exact edge the fixture straddles it instead. On the 13x13 / 26x26 pair in fp32x3 both exact edges must lie on the
decision path. The all-pass pair's walk must run past 256 candidates, with candidates suppressed by boxes kept in earlier
128-candidate steps. A YOLOv3-tiny with planted head biases also goes through detect_frames, detect_frame_list, detect_rois and
detect_rois_list, restated from its stored heads after each call. Each call asserts the detection kernels it launched; the module
fails if one of COVERED was never launched (test_detect_exact_cpu.py holds COVERED to the library's kernels)."""
import os

import numpy as np
import pytest

import _region_merge as region_merge
from oracle import exact
from shadernn_b200 import core, modelzoo

pytestmark = pytest.mark.gpu

FORMS = ("fp32x3", "fp16w", "fp16")
f32 = np.float32
COVERED = ["yolo_select_kernel", "yolo_rank_kernel", "yolo_nms_kernel", "yolo_candidates_kernel", "roi_merge_gather_kernel<batch>",
           "roi_merge_gather_kernel<list>", "roi_merge_rank_kernel", "roi_merge_nms_kernel"]
SEEN = {}  # kernel -> the first case that launched it
WORST = {}  # (entry point, form) -> worst |err| / bound
DECISIONS = {}  # form -> [certain, inside]


# ---- planting (CPU) ----------------------------------------------------------------------------------------------------------------
def representable(v, half):
    """The values of v the storage keeps unchanged (exact.stored's fixed points)."""
    v = np.asarray(v, f32)
    return np.unique(v[exact.stored(v, half) == v])


def near_values(x, half, n=4000):
    """Storable values around x: fp16 neighbours in fp16 storage, a fine grid (the hi + lo pairs) otherwise."""
    if half:
        h = np.float16(x).view(np.uint16).astype(np.int64)
        return representable(np.arange(h - n // 2, h + n // 2).astype(np.uint16).view(np.float16).astype(f32), half)
    return representable(f32(x) + np.arange(-n // 2, n // 2) * abs(f32(x)) * f32(2.0 ** -22), half)


def score_edge(half):
    """(d4, d5) pairs around the 0.35f threshold: {"exact": contract score == 0.35f, "above": one fp32 ulp above (or the nearest
    above), "below": the nearest below}, searched over storable values."""
    d5s = representable(np.linspace(0.5, 3.0, 64).astype(f32), half)
    best = {}
    for d5 in d5s:
        t = -np.log((1 / 0.35 - 1) / (1 + np.exp(-float(d5))))
        d4 = near_values(t, half)
        s, _, _ = exact.yolo_score32(d4, np.full(d4.shape, d5, f32))
        for key, sel, target in (("exact", s == exact.YOLO_CONF, 0), ("above", s > exact.YOLO_CONF, 1), ("below", s < exact.YOLO_CONF, -1)):
            if not sel.any():
                continue
            gap = np.abs(s[sel].view(np.int32).astype(np.int64) - exact.YOLO_CONF.view(np.int32).astype(np.int64) - target)
            k = int(np.argmin(gap))
            if key not in best or gap[k] < best[key][2]:
                best[key] = (float(d4[sel][k]), float(d5), int(gap[k]))
    return best


# the fp32 boxes of cells with values d [k, 6] at one grid position (yolo_decode32 on a one-image, k-cell list)
def box32(d, gx, gy, gc, yi, gw, gh):
    c = {"d": np.asarray(d, f32).reshape(1, -1, 6), "yi": np.full(len(d), yi), "gx": np.full(len(d), gx), "gy": np.full(len(d), gy),
         "gc": np.asarray(gc).repeat(len(d)) if np.ndim(gc) == 0 else np.asarray(gc), "gw": np.full(len(d), gw), "gh": np.full(len(d), gh)}
    return exact.yolo_decode32(c)[2][0]


def iou_edge(half, gw, gh):
    """Two boxes of cell (1, 1) of head 0, anchors gc = 1 and 2: (dA, dB) six values each with the contract IoU == 0.45f ("exact") and
    the nearest above ("above"), searched over B's storable d2 near where the IoU crosses 0.45, for a few d3. Both boxes are small and
    score above every background cell, so that A is kept and no box but A can suppress B."""
    dA = np.array([0.0, 0.0, -1.0, -1.0, 6.0, 6.0], f32)
    a = box32(dA[None], 1, 1, 1, 0, gw, gh)[0]

    def ious(d2, d3):
        dB = np.tile(np.array([0.0, 0.0, 0.0, d3, 5.0, 6.0], f32), (len(d2), 1))
        dB[:, 2] = d2
        return exact.yolo_iou32(a[None], box32(dB, 1, 1, 2, 0, gw, gh)), dB
    best = {}
    for d3 in representable(np.linspace(-3.0, 0.0, 41).astype(f32), half):
        coarse = np.linspace(-3.0, 3.0, 6001).astype(f32)
        iou, _ = ious(coarse, d3)
        for x in np.flatnonzero(np.diff(np.sign(iou.astype(np.float64) - 0.45)) != 0):
            d2 = near_values(coarse[x], half, 4000)
            iou, dB = ious(d2, d3)
            bits = iou.view(np.int32).astype(np.int64) - exact.YOLO_IOU.view(np.int32).astype(np.int64)
            for key, target in (("exact", 0), ("above", 1)):
                sel = bits >= target
                if not sel.any():
                    continue
                k = int(np.argmin(np.where(sel, np.abs(bits - target), 1 << 40)))
                if key not in best or abs(bits[k] - target) < best[key][2]:
                    best[key] = (dA, dB[k].copy(), int(abs(bits[k] - target)))
    return best


def planted(g0, g1, c, n, half, seed, allpass=False):
    """Heads [n, gh, gw, c] of two grids g0 = (gh, gw), g1 with the planted cells, and what they reached: {"score": {"exact" / "above" /
    "below": ulps from the target}, "iou": {...}, "cells": {"score": {key: scan index on head 0}, "iou": {key: (image, scan of A, scan
    of B)}}}. Background cells pass sparsely, so that no image fills 100 rows before its lowest planted score. All-pass heads have
    boxes large enough that the greedy walk suppresses candidates with boxes kept in earlier 128-candidate steps."""
    rng = np.random.default_rng(seed)
    h = [rng.uniform(-1.5, 1.5, (n,) + tuple(g) + (c,)).astype(f32) for g in (g0, g1)]
    for t in h:
        if allpass:
            t[..., 4:18:6] = rng.uniform(2, 5, t[..., 4:18:6].shape)
            t[..., 5:18:6] = 4.0
            for k in (2, 3, 8, 9, 14, 15):  # boxes several cells wide: the walk runs past 128 candidates
                t[..., k] = rng.uniform(3.0, 4.5, t[..., k].shape)
        else:
            t[..., 4:18:6] = np.where(rng.uniform(size=t[..., 4:18:6].shape) < 0.03, rng.uniform(0, 4, t[..., 4:18:6].shape), -6.0)
    if not allpass:
        reached = {"score": {}, "iou": {}, "cells": {"score": {}, "iou": {}}}
        edges = score_edge(half)
        # score edges on head 0, image by image, at cells that nothing else touches (their boxes are small and apart)
        for k, (key, (d4, d5, gap)) in enumerate(sorted(edges.items())):
            for t in h:
                gy, gx = (k + 2) % t.shape[1], (2 * k) % t.shape[2]
                t[:, gy, gx, 12:18] = [0.0, 0.0, -3.0, -3.0, d4, d5]
            reached["score"][key] = gap
            reached["cells"]["score"][key] = (((k + 2) % g0[0]) * g0[1] + (2 * k) % g0[1]) * 3 + 2
        ie = iou_edge(half, g0[1], g0[0])
        for k, (key, (dA, dB, gap)) in enumerate(sorted(ie.items())):
            if k < n:  # pair k in image k: cell (1, 1) of head 0, its anchor 0 rejected
                h[0][k, 1, 1, 0:6], h[0][k, 1, 1, 6:12], h[0][k, 1, 1, 12:18] = [0, 0, 0, 0, -6, 0], dA, dB
                reached["cells"]["iou"][key] = (k, (g0[1] + 1) * 3 + 1, (g0[1] + 1) * 3 + 2)
            reached["iou"][key] = gap
        # exact score ties: the same (d4, d5) on both heads and on several anchors, far apart
        tie = representable(np.array([2.5, 2.0], f32), half)
        if tie.size == 2:
            for t in h:
                t[:, -1, -1, 4:6], t[:, -1, -1, 16:18], t[:, 0, -1, 10:12] = tie[::-1], tie[::-1], tie[::-1]
        # past fp16's range (stored saturated): w = inf, h = inf, score exactly 1; and a NaN pixel
        big = f32(131008.0 if not half else 65504.0)
        h[1][:, -1, 0, 0:6] = [0.0, 0.0, 100.0, -1.0, 3.0, 3.0]
        h[1][:, -1, 0, 6:12] = [0.5, -0.5, -1.0, big, 2.5, 3.0]
        h[1][:, -1, 0, 12:18] = [-big, big, -1.0, -1.0, big, 3.0]
        h[1][:, 0, 0, :] = np.nan
    else:
        reached = {}
    return [exact.stored(t, half) for t in h], reached


def walk_end(path, max_rows):
    """Where the greedy walk stops in the sorted list: after the max_rows-th kept box, or at the end of the list."""
    return int(path["kept"][-1]) + 1 if len(path["kept"]) == max_rows else len(path["order"])


def cross_step(heads, paths, max_rows):
    """Per image, the candidates past the first 128-candidate step of yolo_greedy_nms that a box kept in an earlier step suppresses: the
    kernel's test against kept[] rather than against the step's own candidates."""
    _, _, box, _ = exact.yolo_decode32(exact.yolo_cells(heads[0], heads[1]))
    out = []
    for n, p in enumerate(paths):
        o, kept = p["order"], p["kept"]
        b, hits = box[n, o], 0
        for j in sorted(set(range(128, walk_end(p, max_rows))) - set(kept.tolist())):
            early = kept[kept < (j // 128) * 128]
            hits += int((exact.yolo_iou32(b[early], b[j]) > exact.YOLO_IOU).any())
        out.append(hits)
    return out


def edges_on_path(heads, paths, cells, max_rows):
    """The planted exact edges that lie on the contract's decision path, as {"score": images, "iou": images}. The exact-0.35f cell counts
    where it is rejected with fewer than max_rows rows kept, so that passing it would have made a row. The exact-0.45f pair counts where A
    is kept, B comes after it within the walk, the pair's fp32 IoU is 0.45f, and B is kept: no other kept box suppresses it either."""
    _, score, box, _ = exact.yolo_decode32(exact.yolo_cells(heads[0], heads[1]))
    on = {"score": [], "iou": []}
    for n, p in enumerate(paths):
        s = cells["score"].get("exact")
        if s is not None and score[n, s] == exact.YOLO_CONF and len(p["kept"]) < max_rows:
            on["score"].append(n)
    if "exact" in cells["iou"]:
        n, a, b = cells["iou"]["exact"]
        o, kept = paths[n]["order"], paths[n]["kept"]
        ks = o[kept]
        pa, pb = np.flatnonzero(o == a), np.flatnonzero(o == b)
        if (a in ks and b in ks and pa.size and pb.size and pa[0] < pb[0] < walk_end(paths[n], max_rows)
                and exact.yolo_iou32(box[n, a], box[n, b]) == exact.YOLO_IOU):
            on["iou"].append(n)
    return on


def identity_model(tmp, g0, g1, c, precision, tag):
    """Two inputs [gh, gw, c] -> 1x1 identity Conv2D each (no bias, no BN, linear) -> YOLO."""
    b = modelzoo.Builder(3)
    heads = []
    for i, (gh, gw) in enumerate((g0, g1)):
        x = b.input(gw, gh, c, index=i)
        heads.append(b.conv(x, c, 1, 1, "valid", "linear", bias=False, bn=False))
        b.layers[heads[-1]]["_w"]["kernel"] = np.eye(c, dtype=f32).reshape(c, c, 1, 1)
    b.yolo(*heads)
    path = os.path.join(tmp, "%s_%s.json" % (tag, precision))
    modelzoo.write_model(b.layers, path, split=True)
    return path, heads


# ---- holding rows --------------------------------------------------------------------------------------------------------------------
def same_bits(a, b):
    """Bit-identical float32 arrays; any NaN matches any NaN (the device's and numpy's NaN payloads differ)."""
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32))


YOLO_DEVICE = ["yolo_select_kernel", "yolo_rank_kernel", "yolo_nms_kernel"]


def expect_launches(ctx, tail, why):
    """The launches since the last call end with `tail` (the entry point's own detection kernels, after its input and forward pass)."""
    names = ctx.debug_launches(clear=True)
    assert names[-len(tail):] == tail, (why, tail, names[-len(tail) - 2:])
    for k in names:
        SEEN.setdefault(k, why)


def worst(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), ratio)


def hold_values(got, scan, defn, n, key, why):
    """Rows' score, x, y, w, h against the definition at their cells: within the bound where it is finite, the same value where not."""
    ratio = 0.0
    for j, f in enumerate(("score", "x", "y", "w", "h")):
        ref, e = defn[f][n, scan], defn["e_" + f][n, scan]
        g = got[:, 1 + j].astype(np.float64)
        inf = np.isinf(ref)
        assert np.array_equal(np.isnan(g), np.isnan(ref)) and np.array_equal(g[inf], ref[inf]), (why, f, "non-finite values")
        fin = np.isfinite(ref)
        r, bad = exact.check(g[fin], ref[fin], e[fin], f)
        assert bad == 0, "%s: %s: %d values outside the bound, worst |err|/bound %.3g" % (why, f, bad, r)
        ratio = max(ratio, r)
    worst(key, ratio)


def hold_contract(rows, counts, heads, max_rows, form, key, why, check_decisions=True):
    """Device rows and counts against yolo_contract of the stored heads (bit for bit), and the contract against the definition."""
    want, wc, near, paths = exact.yolo_contract(heads[0], heads[1], max_rows)
    assert not near.any(), "%s: an exp lies within reach of an fp32 rounding midpoint: %d cells" % (why, int(near.sum()))
    assert np.array_equal(counts, wc), (why, counts, wc)
    for n in range(len(wc)):
        if not same_bits(rows[n], want[n]):
            bad = np.flatnonzero(~np.all(rows[n].view(np.uint32) == want[n].view(np.uint32), axis=1))
            raise AssertionError("%s: image %d: %d rows differ from the contract, first at %d: got %r want %r" % (
                why, n, bad.size, bad[0], rows[n, bad[0]], want[n, bad[0]]))
    if not check_decisions:
        return want, wc, paths, None
    defn = exact.yolo_define(heads[0], heads[1])
    dec = exact.yolo_decisions(heads[0], heads[1], paths, max_rows, defn=defn)
    for n, d in enumerate(dec):
        assert not d["wrong"], "%s: image %d: certain decisions the contract made the other way: %s" % (why, n, d["wrong"][:5])
        c = DECISIONS.setdefault(form, [0, 0])
        c[0] += sum(d["certain"].values())
        c[1] += sum(d["inside"].values())
        hold_values(want[n, :wc[n]], paths[n]["order"][paths[n]["kept"]], defn, n, key, why)
    return want, wc, paths, (defn, dec)


def hold_host(m, paths, defn, dec, max_rows, form, why):
    """run() + boxes(n): the contract's rows up to the first one an inside-bound decision may move, within the definition's bounds,
    and the same count when no decision on the path is inside its bound."""
    for n, d in enumerate(dec):
        got = m.boxes(n, max_rows)
        kept = paths[n]["order"][paths[n]["kept"]]
        k = d["first_uncertain"]
        if k == len(kept):
            assert len(got) == len(kept), (why, n, len(got), len(kept))
        assert len(got) >= k, (why, n, len(got), k)
        assert np.all(got[:k, 0] == 0), (why, n)
        hold_values(got[:k], kept[:k], defn, n, ("host", form), why + " host image %d" % n)


# ---- planted heads, through detect_device, detect_torch and the host path ---------------------------------------------------------------
# (head 0 grid, head 1 grid, channels, batch, max_rows list, all-pass)
SHAPES = [((13, 13), (26, 26), 18, 5, (1, 7, 100), False),
          ((7, 11), (14, 22), 20, 1, (7, 100), False),
          ((5, 9), (3, 4), 255, 5, (100,), False),
          ((64, 64), (128, 128), 18, 1, (100,), True)]


@pytest.mark.parametrize("precision", FORMS)
@pytest.mark.parametrize("shape", SHAPES, ids=["13x13-26x26", "7x11-14x22-c20", "5x9-3x4-c255", "allpass-64-128"])
def test_planted_heads(ctx, tmp_path, shape, precision):
    import torch
    from shadernn_b200 import _lib
    g0, g1, c, n, max_rows_list, allpass = shape
    half = precision == "fp16"
    h_in, reached = planted(g0, g1, c, n, half, seed=c + g0[0], allpass=allpass)
    path, head_ids = identity_model(str(tmp_path), g0, g1, c, precision, "planted_%dx%d_%d" % (g0[0], g0[1], c))
    m = core.MixedInferenceCore(ctx, path, batch=n, precision=precision)
    try:
        tag = "%dx%d/%dx%d c%d batch %d %s" % (g0 + g1 + (c, n, precision))
        if reached:
            print("%s: score edge %s, IoU edge %s (ulps from the target)" % (tag, reached["score"], reached["iou"]))
            if precision == "fp32x3" and shape == SHAPES[0]:
                assert reached["score"].get("exact") == 0 and reached["iou"].get("exact") == 0, reached
        m.set_input(h_in[1], 1)
        ctx.debug_launches(clear=True)
        m.run(h_in[0], want_classes=False)
        expect_launches(ctx, ["yolo_candidates_kernel"], tag + " host")
        heads = [m.layer_output(i) for i in head_ids]
        for i in range(2):
            assert same_bits(heads[i], h_in[i]), "%s: head %d is not the planted values: %d differ" % (
                tag, i, int(np.sum((heads[i] != h_in[i]) & ~(np.isnan(heads[i]) & np.isnan(h_in[i])))))
        xs = [torch.from_numpy(np.ascontiguousarray(h)).cuda() for h in h_in]
        for max_rows in max_rows_list:
            why = "%s max_rows %d" % (tag, max_rows)
            rows, counts = m.detect_torch(xs, max_rows=max_rows)
            torch.cuda.synchronize()
            expect_launches(ctx, YOLO_DEVICE, why + " detect_torch")
            want, wc, paths, dd = hold_contract(rows.cpu().numpy(), counts.cpu().numpy(), heads, max_rows, precision, ("detect_torch", precision), why)
            if max_rows == max_rows_list[-1]:
                hold_host(m, paths, dd[0], dd[1], max_rows, precision, why)
                if reached:  # the exact edges the fixture reached, on the decision path
                    on = edges_on_path(heads, paths, reached["cells"], max_rows)
                    print("%s: exact edges on the decision path in images: 0.35f %s, 0.45f %s" % (tag, on["score"], on["iou"]))
                    if precision == "fp32x3" and shape == SHAPES[0]:
                        assert on["score"] == list(range(n)) and on["iou"] == [reached["cells"]["iou"]["exact"][0]], on
                if allpass:
                    hits = cross_step(heads, paths, max_rows)
                    print("%s: the walk ends at %d of %d candidates; %d suppressed by boxes kept in earlier steps" % (
                        tag, walk_end(paths[0], max_rows), len(paths[0]["order"]), hits[0]))
                    assert walk_end(paths[0], max_rows) > 256 and hits[0] > 0, hits
            # detect_device: the raw call into caller buffers on the context's stream
            keep, ins = m._device_inputs("detect_device", xs, "nhwc", None, None)
            r2, c2 = torch.full_like(rows, float("nan")), torch.full_like(counts, -7)
            _lib.check(_lib.lib().snnb_model_detect_device(m.h, ins, len(keep), r2.data_ptr(), max_rows, c2.data_ptr(), m._torch_stream()),
                       "snnb_model_detect_device")
            torch.cuda.synchronize()
            expect_launches(ctx, YOLO_DEVICE, why + " detect_device")
            assert same_bits(r2.cpu().numpy(), want) and np.array_equal(c2.cpu().numpy(), wc), why + " detect_device"
            WORST[("detect_device", precision)] = WORST[("detect_torch", precision)]  # the same rows, bit for bit
        if allpass:
            assert int(wc.min()) == 100 and len(paths[0]["order"]) > 256, (wc, len(paths[0]["order"]))
    finally:
        m.close()


# ---- YOLOv3-tiny with planted biases, through the frame and region entry points -------------------------------------------------------------
def tiny(ctx, model_dir, batch):
    from test_detect_gpu import yolo_path
    hw = (128, 160)
    path = yolo_path(model_dir, "planted", hw)
    m = core.MixedInferenceCore(ctx, path, batch=batch, input_hw=hw)
    ids = [i for i in range(m.num_layers) if m.layer_info(i)[2][-1] == 18]
    return m, ids, hw


def test_frame_and_region_entry_points(ctx, model_dir):
    import torch
    m, ids, hw = tiny(ctx, model_dir, 4)
    try:
        assert len(ids) == 2, ids
        rng = np.random.default_rng(5)
        mean4, norm4 = [120.0, 110.0, 100.0, 0.0], [1 / 60.0, 1 / 60.0, 1 / 60.0, 1.0]
        frames = rng.integers(0, 256, (4, hw[0], hw[1], 4), dtype=np.uint8)
        fr = torch.from_numpy(frames).cuda()
        kw = dict(format="rgba8", mean4=mean4, norm4=norm4)
        for what, call in (("detect_frames", lambda: m.detect_frames(fr, **kw)),
                           ("detect_frame_list", lambda: m.detect_frame_list([fr[i] for i in range(4)], **kw))):
            rows, counts = call()
            torch.cuda.synchronize()
            expect_launches(ctx, YOLO_DEVICE, what)
            heads = [m.layer_output(i) for i in ids]
            _, wc, _, _ = hold_contract(rows.cpu().numpy(), counts.cpu().numpy(), heads, 100, "fp32x3", (what, "fp32x3"), what)
            assert wc.sum() > 0, what
        # regions: two frames of 300 x 410, four slots (one invalid); each used slot's heads decoded by the contract, then merged
        big = rng.integers(0, 256, (2, 300, 410, 4), dtype=np.uint8)
        regions = np.array([(0, 0, 0, 0, 200, 150), (1, 1, 50, 40, 160, 128), (0, 2, 0, 0, 200, 150), (0, 3, 400, 0, 20, 20)], np.int32)
        rois = torch.from_numpy(regions).cuda()
        fb = torch.from_numpy(big).cuda()
        for what, form, call in (("detect_rois", "batch", lambda: m.detect_rois(fb, rois, **kw)),
                                 ("detect_rois_list", "list", lambda: m.detect_rois_list([fb[0], fb[1]], rois, **kw))):
            rows, counts = call()
            torch.cuda.synchronize()
            expect_launches(ctx, YOLO_DEVICE + ["roi_merge_gather_kernel<%s>" % form, "roi_merge_rank_kernel", "roi_merge_nms_kernel"], what)
            heads = [m.layer_output(i) for i in ids]
            slot_rows, slot_counts, _, _ = exact.yolo_contract(heads[0], heads[1], 100)
            want, wc = region_merge.merge_region_rows(slot_rows, slot_counts, regions, None, [(300, 410)] * 2, 100)
            assert np.array_equal(counts.cpu().numpy(), wc) and same_bits(rows.cpu().numpy(), want), what
            assert wc.sum() > 0, what
    finally:
        m.close()


def test_every_detection_kernel_was_launched():
    for key in sorted(WORST):
        print("%-18s %-7s worst |err|/bound %.3g" % (key + (WORST[key],)))
    for form, (certain, inside) in sorted(DECISIONS.items()):
        print("%-7s decisions: %d certain, %d inside their bound" % (form, certain, inside))
    for key in COVERED:
        print("%-32s %s" % (key, SEEN.get(key, "NOT LAUNCHED")))
    missing = [k for k in COVERED if k not in SEEN]
    assert not missing, missing
