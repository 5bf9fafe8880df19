"""The per-operator C ABI table (test_ops_exact_gpu.py) without a GPU: every per-operator entry point include/snnb.h declares has a row,
the convolution rows' host plans (snnb_debug_conv_launch with the query snnb_conv2d_launch makes) reach every conv variant the GPU
test requires, and on the table's own shapes each plausible misreading of an operation falls outside oracle/exact.py's bound
somewhere, so the GPU table would catch it."""
import os
import re

import numpy as np
import pytest

from oracle import exact

import test_ops_exact_gpu as table

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32, f64 = np.float32, np.float64
SMS = 132  # H100 SXM


def _exceeds(got, ref, bound):
    with np.errstate(invalid="ignore", over="ignore"):
        return exact.check(got, ref, bound, "mutation")[1] > 0


# ---- the table covers the surface --------------------------------------------------------------------------------------------
def declared_entry_points():
    with open(os.path.join(ROOT, "include", "snnb.h")) as f:
        src = f.read()
    names = re.findall(r"^int (snnb_\w+)\(", src, re.M)
    op = re.compile(r"snnb_(\w+_launch|argmax1|tensor_(upload|download)_\w+|weights_pack_\w+|graph_capture_\w+)$")
    return [n for n in names if op.match(n) and not n.startswith("snnb_debug_")]


def test_every_declared_operator_entry_point_has_a_row():
    declared = declared_entry_points()
    assert "snnb_conv2d_launch" in declared and "snnb_argmax1" in declared and "snnb_tensor_download_c4hw4" in declared, declared
    missing = [n for n in declared if n not in table.ENTRY_POINTS]
    assert not missing, "declared in snnb.h without a row in test_ops_exact_gpu.py: %s" % missing
    assert not [n for n in table.ENTRY_POINTS if n not in declared], "ENTRY_POINTS names calls snnb.h does not declare"


def test_conv_rows_reach_every_variant(built):
    seen = {}
    for c in table.CONV:
        for form in table.FORMS:
            v = table.plan_variant(table.conv_plan(c, form, SMS))
            assert v["path"] != "none", (c.why, form)
            for key in table.variant_keys(v):
                seen.setdefault(key, c.why)
    missing = [k for k in table.expected_conv_variants() if k not in seen]
    assert not missing, missing
    sk = [c for c in table.CONV if c.algo == "tcgen05-streamk"]
    for c in sk:  # a partial last wave: whole tiles do not divide into the SMs
        p = table.conv_plan(c, "fp32x3", SMS)
        assert p["sk"] and p["sk_dp"] > 0 and p["tiles_x"] * p["tiles_y"] * p["tiles_n"] * p["tiles_oc"] % SMS, (c.why, p)


def test_conv_rows_are_asymmetric_with_every_bottom_and_right_padding(built):
    by_path = {}
    for c in table.CONV:
        assert c.h != c.w and c.px != c.py, c.why
        assert 0 <= c.B < c.k and 0 <= c.R < c.k, c.why
        path = table.plan_variant(table.conv_plan(c, "fp32x3", SMS))["path"]
        by_path.setdefault((path, c.k), []).append(c)
        if c.row != (c.s, c.px):
            assert path != "rowwin", c.why
    for path in ("igemm", "simt"):
        rows = by_path[(path, 3)]
        assert {c.B for c in rows} == {0, 1, 2} and {c.R for c in rows} == {0, 1, 2}, path
        assert {c.px > c.py for c in rows} == {True, False}, path  # pads both ways round
    assert {c.px > c.py for c in by_path[("rowwin", 3)]} == {True, False}
    acts = {(c.act, c.alpha) for c in table.CONV}
    assert {a for a, _ in acts} >= {"", "relu", "relu6", "tanh", "sigmoid", "leakyRelu", "SiLU"}
    assert {al for a, al in acts if a == "leakyRelu"} - {0.1}, "a leaky alpha other than 0.1"
    assert any(c.k == 1 for c in by_path.get(("igemm", 1), [])) and any(c.k == 1 for c in by_path.get(("rowwin", 1), []))


def test_depthwise_rows_reach_every_kernel():
    got = set()
    for why, n, h, w, c, k, s, px, py, B, R, *_ in table.DW:
        assert h != w and px != py and 0 <= B < k and 0 <= R < k, why
        got.add(table.dw_kernel(*table.dw_out(h, w, k, s, px, py, B, R), k, s))
    assert got == set(table.DW_KERNELS), sorted(got)


# ---- misreadings fall outside the bounds ---------------------------------------------------------------------------------------
def _conv_case(c, seed):
    x, wt, bias, bn, res = table.conv_operands(c, seed)
    return exact.stored(x, False), wt, bias, bn, None if res is None else exact.stored(res, False)


def _restate(c, x, wt, bias, bn, res, path, form="fp32x3", px=None, py=None, mode=None, residual=True):
    """exact.conv2d of row c on the kernel `path`, at the row's output size whatever pads or mode replace the row's."""
    px, py, mode = c.px if px is None else px, c.py if py is None else py, c.mode if mode is None else mode
    return exact.conv2d(x, wt, bias, bn, c.s, px, py, table.conv_out(c), c.act, c.alpha, residual=res if residual else None,
                        form="simt" if path == "simt" else form, kernel=table.KERNEL_OF_PATH[path], pad_mode=mode)


SMALL = [(i, c) for i, c in enumerate(table.CONV) if c.n * c.h * c.w <= 4000]


@pytest.mark.parametrize("i,c", SMALL, ids=[c.why for _, c in SMALL])
def test_swapped_pads_fall_outside_the_conv_bound(built, i, c):
    path = table.plan_variant(table.conv_plan(c, "fp32x3", SMS))["path"]
    x, wt, bias, bn, res = _conv_case(c, 100 + i)
    for kernel in sorted({path, "simt"}):  # the kernel's own restatement, and the CUDA-core one
        ref, bound = _restate(c, x, wt, bias, bn, res, kernel)
        swapped, _ = _restate(c, x, wt, bias, bn, res, kernel, px=c.py, py=c.px)
        assert _exceeds(swapped, ref, bound), (c.why, kernel)


@pytest.mark.parametrize("row", table.DW, ids=[r[0] for r in table.DW])
def test_swapped_pads_fall_outside_the_depthwise_bound(row):
    why, n, h, w, c, k, s, px, py, B, R, act, alpha, bias_on, bn_on = row
    rng = np.random.default_rng(1)
    x = exact.stored(rng.uniform(-1, 1, (n, h, w, c)), False)
    wk = rng.standard_normal((c, k, k)).astype(f32) / k
    ohw = table.dw_out(h, w, k, s, px, py, B, R)
    ref, bound = exact.depthwise(x, wk, None, None, s, px, py, ohw, act, alpha)
    assert _exceeds(exact.depthwise(x, wk, None, None, s, py, px, ohw, act, alpha)[0], ref, bound), why


def test_residual_after_the_activation_falls_outside(built):
    rows = [(i, c) for i, c in enumerate(table.CONV) if c.res]
    assert {table.plan_variant(table.conv_plan(c, "fp32x3", SMS))["path"] for _, c in rows} >= {"igemm", "simt"}
    for i, c in rows:
        x, wt, bias, bn, res = _conv_case(c, 100 + i)
        path = table.plan_variant(table.conv_plan(c, "fp32x3", SMS))["path"]
        ref, bound = _restate(c, x, wt, bias, bn, res, path)
        after = _restate(c, x, wt, bias, bn, res, path, residual=False)[0] + res
        assert _exceeds(after, ref, bound), c.why


def _folded(wt, bias, bn, eps=1e-3, clamp=True):
    """pack.cpp's BN fold with its epsilon or its clamp changed."""
    g, be, m, v = (np.asarray(bn[k], f32) for k in ("gamma", "beta", "mean", "var"))
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.sqrt(v + f32(eps))
        if clamp:
            s = np.maximum(s, f32(1e-4))
        scale = (g / s).astype(f32)
        return (wt * scale[:, None, None, None]).astype(f32), ((bias - m) * scale + be).astype(f32)


@pytest.mark.parametrize("eps,clamp", [(1e-3, False), (1e-5, True)], ids=["no clamp", "eps 1e-5"])
def test_bn_fold_misreadings_fall_outside(built, eps, clamp):
    rows = [(i, c) for i, c in enumerate(table.CONV) if c.bn and c.n * c.h * c.w <= 4000]
    assert {table.plan_variant(table.conv_plan(c, "fp32x3", SMS))["path"] for _, c in rows} >= {"igemm", "simt", "rowwin"}
    for i, c in rows:
        x, wt, bias, bn, res = _conv_case(c, 100 + i)
        assert bn["var"][1] == f32(-1e-3)
        path = table.plan_variant(table.conv_plan(c, "fp32x3", SMS))["path"]
        ref, bound = _restate(c, x, wt, bias, bn, res, path)
        wm, bm = _folded(wt, bias, bn, eps, clamp)
        with np.errstate(invalid="ignore", over="ignore"):
            got = _restate(c, x, wm, bm, None, res, path)[0]
        assert _exceeds(got, ref, bound), c.why
        if clamp:  # the ordinary channels alone show the epsilon
            keep = [j for j in range(c.oc) if j != 1]
            assert _exceeds(got[..., keep], ref[..., keep], bound[..., keep]), c.why
    rng = np.random.default_rng(5)
    x = exact.stored(rng.uniform(-3, 3, (2, 9, 11, 20)), False)
    bn = table.bn_params(rng, 20)
    ref, bound = exact.batchnorm(x, bn, "relu6")
    g, be, m, v = (bn[k].astype(f64) for k in ("gamma", "beta", "mean", "var"))
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.sqrt(v + eps)
        s = np.maximum(s, 1e-4) if clamp else s
        got = exact.act64(g / s * (x - m) + be, "relu6", 0.0)
    assert _exceeds(got, ref, bound)


def test_dense_read_as_in_out_falls_outside():
    why, n, h, w, c, n_out, act = table.DENSE[table.DENSE_SQUARE]
    assert h * w * c == n_out, why
    rng = np.random.default_rng(3)
    x = exact.stored(rng.uniform(-1, 1, (n, h, w, c)), False)
    kern = (rng.standard_normal((n_out, n_out)) / np.sqrt(n_out)).astype(f32)
    bias = rng.uniform(-0.2, 0.2, n_out).astype(f32)
    for form in table.FORMS:
        v = {"path": "igemm"}
        ref, bound = table.restate_dense(x, kern, bias, act, 0.0, v, form)
        assert not _exceeds(table.restate_dense(x, kern, bias, act, 0.0, v, form)[0], ref, bound)
        assert _exceeds(table.restate_dense(x, np.ascontiguousarray(kern.T), bias, act, 0.0, v, form)[0], ref, bound), form


def test_flatten_in_chw_order_falls_outside():
    rng = np.random.default_rng(4)
    for shape in ((2, 3, 5, 20), (2, 2, 3, 13)):
        x = exact.stored(rng.uniform(-1, 1, shape), False)
        ref, bound = exact.flatten(x)
        chw = x.transpose(0, 3, 1, 2).reshape(shape[0], 1, 1, -1)
        assert _exceeds(chw, ref, bound), shape
    for n, h, w, c, n_out, act in [r[1:] for r in table.DENSE if r[2] * r[3] > 1]:  # dense on an H x W > 1 input flattens too
        x = exact.stored(rng.uniform(-1, 1, (n, h, w, c)), False)
        kern = (rng.standard_normal((n_out, h * w * c))).astype(f32)
        v = {"path": "simt" if h * w * c < 16 else "igemm"}
        ref, bound = table.restate_dense(x, kern, None, act, 0.0, v, "fp32x3")
        chw = x.transpose(0, 3, 1, 2).copy()
        assert _exceeds(table.restate_dense(chw, kern, None, act, 0.0, v, "fp32x3")[0], ref, bound), (h, w, c)


def test_c4hw4_with_lane_and_block_swapped_differs():
    rng = np.random.default_rng(6)
    for c in table.C4HW4:
        x = rng.uniform(-1, 1, (3, 4, 5, c)).astype(f32)
        good = table.c4hw4_of(x)
        d = good.shape[1]
        perm = np.zeros((3, 4, 5, 4 * d), f32)
        perm[..., :c] = x
        assert np.array_equal(good, perm.reshape(3, 4, 5, d, 4).transpose(0, 3, 1, 2, 4))
        assert _exceeds(table.c4hw4_of(x, swap=True), good, np.zeros(good.shape)), c


def test_avgpool_k2_divisor_on_clipped_windows_falls_outside():
    rng = np.random.default_rng(7)
    clipped = 0
    for n, h, w, c, k, s in table.POOL:
        x = exact.stored(rng.uniform(-1, 1, (n, h, w, c)), False)
        ohw = ((h - 1) // s + 1, (w - 1) // s + 1)
        ref, bound = exact.avgpool(x, k, s, ohw)
        if (ohw[0] - 1) * s + k <= h and (ohw[1] - 1) * s + k <= w:
            continue
        clipped += 1
        got = np.zeros(ref.shape)
        for oy in range(ohw[0]):
            for ox in range(ohw[1]):
                got[:, oy, ox] = x[:, oy * s:oy * s + k, ox * s:ox * s + k].astype(f64).sum(axis=(1, 2)) / (k * k)
        assert _exceeds(got, ref, bound), (h, w, k, s)
    assert clipped >= 3
    assert {(k > s) - (k < s) for _, _, _, _, k, s in table.POOL} == {-1, 0, 1}  # k < s, k = s, k > s


def test_reflect_repeating_the_edge_falls_outside(built):
    rng = np.random.default_rng(8)
    pads = [r for r in table.PAD if r[8] == "reflect"]
    for n, h, w, c, px, py, oh, ow, mode in pads:
        x = exact.stored(rng.uniform(-1, 1, (n, h, w, c)), False)
        ref, bound = exact.pad(x, px, py, (oh, ow), "reflect")
        sym = np.pad(x, ((0, 0), (py, oh - h - py), (px, ow - w - px), (0, 0)), mode="symmetric")
        assert _exceeds(sym, ref, bound), (h, w, px, py)
    rows = [(i, c) for i, c in enumerate(table.CONV) if c.mode == "reflect"]
    assert rows
    for i, c in rows:
        x, wt, bias, bn, res = _conv_case(c, 100 + i)
        oh, ow = table.conv_out(c)
        ref, bound = _restate(c, x, wt, bias, bn, res, "simt")
        need_h, need_w = (oh - 1) * c.s + c.k, (ow - 1) * c.s + c.k
        xp = np.pad(x, ((0, 0), (c.py, max(need_h - c.h - c.py, 0)), (c.px, max(need_w - c.w - c.px, 0)), (0, 0)), mode="symmetric")
        got = _restate(c, xp, wt, bias, bn, res, "simt", px=0, py=0, mode="constant")[0]
        assert _exceeds(got, ref, bound), c.why


def test_softmax_without_max_subtraction_falls_outside():
    rng = np.random.default_rng(9)
    z = exact.stored(rng.uniform(-100, 100, (3, 2, 5, 37)), False)
    ref, bound = exact.softmax(z)
    with np.errstate(over="ignore", invalid="ignore"):
        e = np.exp(z - z.max(axis=-1, keepdims=True))
        assert not _exceeds(e / e.sum(axis=-1, keepdims=True, dtype=f32), ref, bound)
        e = np.exp(z)
        assert _exceeds(e / e.sum(axis=-1, keepdims=True, dtype=f32), ref, bound)


# ---- the SIMT bound holds the kernel's arithmetic ---------------------------------------------------------------------------
def simt_sim(x, wv, shift, c, px, py):
    """conv2d_simt_kernel in float32: per output, fmaf over K = (ky, kx, ic) in that order from 0, + bias, then the activation; the
    store of exact.stored."""
    n, h, w, ic = x.shape
    oh, ow = table.conv_out(c)
    ni, oy, ox = exact.pixels(None, n, oh, ow)
    acc = np.zeros((len(ni), wv.shape[0]), f32)
    for ky in range(c.k):
        for kx in range(c.k):
            X = exact.gather(x, ni, oy * c.s + ky - py, ox * c.s + kx - px, c.mode, dtype=f32)
            for ch in range(ic):  # fmaf: the product is exact in float64, one rounding of the sum
                acc = (X[:, ch:ch + 1].astype(f64) * wv[:, ch, ky, kx].astype(f64)[None] + acc.astype(f64)).astype(f32)
    v = (acc + shift[None]).astype(f32)
    if c.act == "leakyRelu":
        v = np.maximum(v, (v * f32(c.alpha)).astype(f32))
    else:
        v = exact.act64(v.astype(f64), c.act, c.alpha).astype(f32)
    return exact.stored(v, False).reshape(n, oh, ow, -1)


def test_simt_fma_chain_sits_inside_the_simt_bound(built):
    rows = [(i, c) for i, c in enumerate(table.CONV)
            if table.plan_variant(table.conv_plan(c, "fp32x3", SMS))["path"] == "simt" and not c.res and c.mode == "constant" and c.n * c.h * c.w <= 600]
    assert rows
    for i, c in rows[:2]:
        x, wt, bias, bn, _ = _conv_case(c, 100 + i)
        wv, shift = exact.fold(wt, bias, bn)
        ref, bound = _restate(c, x, wt, bias, bn, None, "simt")
        ratio, bad = exact.check(simt_sim(x, wv, shift, c, c.px, c.py), ref, bound, "simt")
        assert bad == 0, (c.why, ratio)
        assert _exceeds(simt_sim(x, wv, shift, c, c.py, c.px), ref, bound), c.why
