"""The detection table without a GPU: its coverage list against the library's kernels, and oracle/exact.py's YOLO statements it relies
on. yolo_contract must agree with the C++ oracle's decode (glibc expf) within yolo_define's bounds and with the same certain decisions,
and with decodeCell on hand-worked cells; float32 simulations (the contract, an FMA-contracted score, numpy's float32 exp) must
sit inside the bounds; the planting search must reach its edges in each storage form; and each simulation mutated as a plausible bug
must differ from the contract on the planted fixtures or make a certain decision the other way."""
import math

import numpy as np
import pytest

from oracle import exact, oracle

import test_cuda_core_exact_cpu as cc
import test_detect_exact_gpu as table

f32 = np.float32
DETECT = ("yolo_", "roi_merge_")


def test_every_detection_kernel_has_a_case():
    have = cc._library_kernels()
    det = sorted(k for k in have if k.startswith(DETECT))
    assert "yolo_nms_kernel" in det and "roi_merge_nms_kernel" in det, det
    families = {k.split("<")[0] for k in table.COVERED}
    missing = [k for k in det if k.split("<")[0] not in families]
    assert not missing, "detection kernels without a case in test_detect_exact_gpu.py: %s" % missing
    assert not [k for k in families if k not in have], "COVERED names kernels the library does not have"


def random_heads(seed, n=3, g0=(13, 13), g1=(26, 26), c=18, scale=1.5):
    rng = np.random.default_rng(seed)
    return [rng.normal(0, scale, (n,) + g + (c,)).astype(f32) for g in (g0, g1)]


# ---- the contract against decodeCell and the oracle --------------------------------------------------------------------------------------
def decode_cell(d, yi, gx, gy, gc, gw, gh):
    """decodeCell (layers.cpp) worked out one scalar fp32 operation at a time, exp correctly rounded."""
    e = lambda x: f32(math.exp(float(x)))  # noqa: E731
    d = [f32(v) for v in d]
    ml = d[5] if d[5] > -exact.FLT_MAX else -exact.FLT_MAX
    prob = f32(1) / (f32(1) + e(-d[4]) * (f32(1) + e(-ml)))
    ai = exact.YOLO_MASKS[gc + 3 * yi]
    bw, bh = f32(exact.YOLO_ANCHORS[2 * ai]), f32(exact.YOLO_ANCHORS[2 * ai + 1])
    net_w, net_h = f32(exact.YOLO_SCALE[yi] * gw), f32(exact.YOLO_SCALE[yi] * gh)
    cx = (f32(gx) + f32(1) / (f32(1) + e(-d[0]))) / f32(gw)
    cy = (f32(gy) + f32(1) / (f32(1) + e(-d[1]))) / f32(gh)
    w, h = e(d[2]) * bw / net_w, e(d[3]) * bh / net_h
    return prob, np.array([cx - w / f32(2), cy - h / f32(2), w, h], f32)


def test_contract_matches_decode_cell_by_hand():
    h0, h1 = random_heads(3, n=1, g0=(7, 11), g1=(3, 4))
    c = exact.yolo_cells(h0, h1)
    _, score, box, _ = exact.yolo_decode32(c)
    for s in (0, 5, 7 * 11 * 3 - 1, 7 * 11 * 3, 7 * 11 * 3 + 3 * 4 * 3 - 1, 100):
        yi, gx, gy, gc, gw, gh = (int(c[k][s]) for k in ("yi", "gx", "gy", "gc", "gw", "gh"))
        h = (h0, h1)[yi][0, gy, gx, gc * 6:gc * 6 + 6]
        prob, b = decode_cell(h, yi, gx, gy, gc, gw, gh)
        assert prob.view(np.uint32) == score[0, s].view(np.uint32) and np.array_equal(b.view(np.uint32), box[0, s].view(np.uint32)), s


def test_contract_agrees_with_the_oracle_within_bounds():
    h0, h1 = random_heads(4)
    rows, counts, near, paths = exact.yolo_contract(h0, h1, 100)
    assert not near.any()
    defn = exact.yolo_define(h0, h1)
    dec = exact.yolo_decisions(h0, h1, paths, 100, defn=defn)
    checked = 0
    for n in range(len(h0)):
        assert not dec[n]["wrong"], dec[n]["wrong"][:5]
        ref = oracle.yolo(h0[n], h1[n])
        k = dec[n]["first_uncertain"]
        kept = paths[n]["order"][paths[n]["kept"]]
        if k == len(kept):
            assert len(ref) == len(kept)
        for j, f in enumerate(("score", "x", "y", "w", "h")):
            err = np.abs(ref[:k, 1 + j].astype(np.float64) - defn[f][n, kept[:k]])
            assert np.all(err <= defn["e_" + f][n, kept[:k]]), (n, f)
            err = np.abs(rows[n, :k, 1 + j].astype(np.float64) - defn[f][n, kept[:k]])
            assert np.all(err <= defn["e_" + f][n, kept[:k]]), (n, f)
        checked += k
    assert checked >= 150, checked


# ---- the bounds hold float32 simulations ------------------------------------------------------------------------------------------------
def exp_np32(x):
    with np.errstate(over="ignore", under="ignore"):
        return np.exp(np.asarray(x, f32)), np.zeros(np.shape(x), bool)


def fma_decode(c):
    """yolo_decode32 with the score's 1 + e4 (1 + e5) contracted into one rounding."""
    cls, score, box, near = exact.yolo_decode32(c)
    d = c["d"]
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        ml = np.where(d[..., 5] > -exact.FLT_MAX, d[..., 5], -exact.FLT_MAX)
        e4, e5 = exact.exp_cr(-d[..., 4])[0], exact.exp_cr(-ml)[0]
        score = (f32(1) / f32(np.float64(e4) * np.float64(f32(1) + e5) + 1.0)).astype(f32)
    return cls, score, box, near


@pytest.mark.parametrize("variant", ["contract", "fma", "numpy_exp"])
def test_bounds_hold_float32_simulations(variant):
    for seed, scale, g0, g1 in ((5, 1.5, (13, 13), (26, 26)), (6, 6.0, (7, 11), (14, 22)), (7, 40.0, (5, 9), (3, 4))):
        h0, h1 = random_heads(seed, 2, g0, g1, scale=scale)
        c = exact.yolo_cells(h0, h1)
        _, score, box, _ = fma_decode(c) if variant == "fma" else exact.yolo_decode32(c, exp_np32 if variant == "numpy_exp" else exact.exp_cr)
        defn = exact.yolo_define(h0, h1)
        for j, f in enumerate(("score", "x", "y", "w", "h")):
            got = (score if f == "score" else box[..., j - 1]).astype(np.float64)
            ref, e = defn[f], defn["e_" + f]
            fin = np.isfinite(ref)
            assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(got[np.isinf(ref)], ref[np.isinf(ref)]), (variant, f)
            r, bad = exact.check(got[fin], ref[fin], e[fin], f)
            assert bad == 0, (variant, seed, f, bad, r)
        if scale > 6:
            continue
        # the IoU bound holds the fp32 IoU of the simulated boxes (boxes of normal fp32 size)
        b64 = np.stack([defn[k] for k in "xywh"], -1)[0, :60]
        e64 = np.stack([defn["e_" + k] for k in "xywh"], -1)[0, :60]
        i64, ie = exact.yolo_iou64(b64[:, None], e64[:, None], b64[None], e64[None])
        i32 = exact.yolo_iou32(box[0, :60, None], box[0, None, :60]).astype(np.float64)
        ok = np.isfinite(i64)
        assert np.all(np.abs(i32[ok] - i64[ok]) <= ie[ok]), variant


# ---- the planting search -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("half", [False, True], ids=["split", "fp16"])
def test_planting_reaches_its_edges(half):
    s, i = table.score_edge(half), table.iou_edge(half, 13, 13)
    assert {"above", "below"} <= set(s) and {"exact", "above"} <= set(i), (s, i)
    if not half:
        assert s["exact"][2] == 0 and s["above"][2] == 0 and i["exact"][2] == 0 and i["above"][2] == 0, (s, i)
    for d4, d5, _ in s.values():  # what the search chose is what the storage keeps
        assert exact.stored(f32(d4), half) == f32(d4) and exact.stored(f32(d5), half) == f32(d5)
    for dA, dB, _ in i.values():
        assert np.array_equal(exact.stored(dB, half), dB)


# ---- mutations ---------------------------------------------------------------------------------------------------------------------
def sim(h0, h1, max_rows, mutation=None):
    """yolo_contract with one plausible bug."""
    f = f32
    if mutation == "pitch_c":  # 255-channel heads stored with a 256-channel pitch, read with pitch 255
        pads = [np.concatenate([h, np.zeros(h.shape[:3] + (256 - h.shape[3],), f)], -1) for h in (h0, h1)]
        c = exact.yolo_cells(pads[0], pads[1], pitch=(255, 255))
    else:
        c = exact.yolo_cells(h0, h1)
    cls, score, box, _ = exact.yolo_decode32(c)
    d = c["d"]
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        if mutation in ("product", "fma_score"):
            ml = np.where(d[..., 5] > -exact.FLT_MAX, d[..., 5], -exact.FLT_MAX)
            e4, e5 = exact.exp_cr(-d[..., 4])[0], exact.exp_cr(-ml)[0]
            if mutation == "product":
                score = (f(1) / ((f(1) + e4) * (f(1) + e5))).astype(f)
            else:
                score = (f(1) / f(np.float64(e4) * np.float64(f(1) + e5) + 1.0)).astype(f)
        if mutation in ("masks", "netw", "gxgy", "centre"):
            yi, gx, gy, gw, gh = c["yi"], c["gx"], c["gy"], c["gw"], c["gh"]
            mi = 1 - yi if mutation == "masks" else yi
            a = np.array(exact.YOLO_ANCHORS, f)[np.array(exact.YOLO_MASKS)[c["gc"] + 3 * mi][:, None] * 2 + np.arange(2)]
            gsz = np.stack([gw, gh], 1)
            if mutation == "netw":  # head 0's grid for both heads' net size
                gsz0 = np.array([[gw[0], gh[0]]]).repeat(len(gw), 0)
                net = (np.array(exact.YOLO_SCALE)[yi][:, None] * gsz0).astype(f)
            else:
                net = (np.array(exact.YOLO_SCALE)[yi][:, None] * gsz).astype(f)
            g = np.stack([gy, gx] if mutation == "gxgy" else [gx, gy], 1).astype(f)
            cxy = (g + f(1) / (f(1) + exact.exp_cr(-d[..., 0:2])[0])) / gsz.astype(f)
            wh = exact.exp_cr(d[..., 2:4])[0] * a / net
            box = np.concatenate([cxy if mutation == "centre" else cxy - wh / f(2), wh], -1).astype(f)
    n = score.shape[0]
    rows, counts = np.zeros((n, max_rows, 6), f), np.zeros(n, np.int64)
    for i in range(n):
        p = np.flatnonzero(score[i] >= exact.YOLO_CONF if mutation == "score_ge" else score[i] > exact.YOLO_CONF)
        o = p[np.lexsort((-p, -score[i, p]))] if mutation == "unstable" else p[np.argsort(-score[i, p], kind="stable")]
        if mutation == "max_rows_first":
            o = o[:max_rows]
        b = box[i, o]
        if mutation in ("iou_ge", "suppressed", "step128"):
            alive, kept = np.ones(len(o), bool), []
            for j in range(len(o)):
                if len(kept) == max_rows:
                    break
                if mutation == "step128":  # boxes kept in earlier 128-candidate steps are forgotten
                    alive[j] = not any(k // 128 == j // 128 and exact.yolo_iou32(b[k], b[j]) > exact.YOLO_IOU for k in kept)
                elif mutation == "suppressed":  # every earlier box suppresses, kept or not
                    alive[j] = not (j and (exact.yolo_iou32(b[:j], b[j]) > exact.YOLO_IOU).any())
                else:
                    alive[j] = not any(exact.yolo_iou32(b[k], b[j]) >= exact.YOLO_IOU for k in kept)
                if alive[j]:
                    kept.append(j)
            kept = np.array(kept, np.int64)
        else:
            kept = exact.yolo_nms32(b, cls[i, o], max_rows)
        k = o[kept]
        rows[i, :len(k), 1], rows[i, :len(k), 2:] = score[i, k], box[i, k]
        counts[i] = len(k)
    return rows, counts


def fixtures():
    """The GPU table's planted heads in fp32x3 (split storage), with the max_rows each runs at: the fixtures the device is held on."""
    out = []
    for g0, g1, c, n, mrl, allpass in table.SHAPES:
        h, _ = table.planted(g0, g1, c, n, False, seed=c + g0[0], allpass=allpass)
        out += [(h, mr) for mr in mrl]
    return out


_FIX = []


def caught(mutation):
    if not _FIX:
        _FIX.extend(fixtures())
    for h, mr in _FIX:
        want, wc, _, paths = exact.yolo_contract(h[0], h[1], mr)
        got, gc = sim(h[0], h[1], mr, mutation)
        if not (np.array_equal(gc, wc) and np.array_equal(got.view(np.uint32), want.view(np.uint32))):
            return True
    return False


def test_the_simulation_is_the_contract():
    for h, mr in fixtures()[:4]:
        want, wc, _, _ = exact.yolo_contract(h[0], h[1], mr)
        got, gc = sim(h[0], h[1], mr)
        assert np.array_equal(gc, wc) and np.array_equal(got.view(np.uint32), want.view(np.uint32))


MUTATIONS = ["score_ge", "iou_ge", "product", "masks", "netw", "gxgy", "centre", "unstable", "suppressed", "step128", "max_rows_first",
             "pitch_c", "fma_score"]


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutations_fall_outside(mutation):
    assert caught(mutation), "%s: the planted fixtures do not tell it from the contract" % mutation


@pytest.mark.parametrize("mutation", ["product", "masks", "netw", "gxgy", "centre"])
def test_value_mutations_fall_outside_the_float64_bounds(mutation):
    # the decode's mistakes are caught by the definition alone: some row value of the mutated decode lies outside its bound
    h0, h1 = random_heads(9, 2, (7, 11), (14, 22))
    defn = exact.yolo_define(h0, h1)
    rows, counts = sim(h0, h1, 100, mutation)
    _, _, _, paths = exact.yolo_contract(h0, h1, 100)
    bad = 0
    for n in range(2):
        kept = paths[n]["order"][paths[n]["kept"]]
        k = min(len(kept), int(counts[n]))
        for j, f in enumerate(("score", "x", "y", "w", "h")):
            bad += int(np.sum(np.abs(rows[n, :k, 1 + j] - defn[f][n, kept[:k]]) > defn["e_" + f][n, kept[:k]]))
    assert bad > 0, mutation


def test_the_gpu_fixtures_reach_the_decision_edges():
    # what test_planted_heads asserts on the device, checked here on the fixtures themselves (fp32x3 storage)
    for g0, g1, c, n, mrl, allpass in table.SHAPES:
        h, reached = table.planted(g0, g1, c, n, False, seed=c + g0[0], allpass=allpass)
        _, _, _, paths = exact.yolo_contract(h[0], h[1], mrl[-1])
        if allpass:
            assert table.walk_end(paths[0], 100) > 256 and table.cross_step(h, paths, 100)[0] > 0
        elif (g0, g1) == table.SHAPES[0][:2]:
            on = table.edges_on_path(h, paths, reached["cells"], mrl[-1])
            assert on["score"] == list(range(n)) and on["iou"] == [reached["cells"]["iou"]["exact"][0]], on


def test_iou_bound_covers_an_overlap_at_zero():
    # b starts 1e-7 past a's right edge, both x within 1e-6: an fp32 evaluation may find an overlap of up to ~1e-6 of a unit height
    a, b = np.array([0.0, 0.0, 1.0, 1.0]), np.array([1.0 + 1e-7, 0.0, 1.0, 1.0])
    e = np.array([1e-6, 0.0, 0.0, 0.0])
    iou, bound = exact.yolo_iou64(a, e, b, e)
    b32 = np.array([1.0 - 9e-7, 0.0, 1.0, 1.0], f32)
    assert iou == 0 and float(exact.yolo_iou32(a.astype(f32), b32)) <= bound
    far = np.array([1.1, 0.0, 1.0, 1.0])
    assert exact.yolo_iou64(a, e, far, e) == (0.0, 0.0)  # certainly apart: both evaluations return 0
