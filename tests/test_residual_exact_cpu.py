"""The fused-residual checks of test_residual_exact_gpu.py, without a GPU: its case table reaches every required key in every product
form on an H100's 132 SMs (each row needed for at least one), the residual sources and the tested convolutions are planned as the GPU
test expects, and the restatement it uses reports the epilogue's plausible residual defects, each confined to one tile."""
import functools
import tempfile

import numpy as np
import pytest

import test_conv_plan as cp
import test_residual_exact_gpu as tr
from oracle import exact, oracle

pytestmark = pytest.mark.usefixtures("built")

# (row, stream-K considered, seed: the row's index in its table, as the GPU test numbers its cases)
ROWS = [(row, False, i) for i, row in enumerate(tr.TABLE)] + [(row, True, i) for i, row in enumerate(tr.SK_TABLE)]


def _source_output(om, row, x):
    """The residual source's output for the stored input x: its float64 product plus bias (exact.conv2d), unrounded."""
    n, h, w, ic, oc, k, s, padding, mode, act, scale = row
    o = oracle.Model._offsets({"padding": padding}, k)
    px, py = (0, 0) if k == 1 else (o[0], o[2])
    lw = om.w[tr.SRC]
    return exact.conv2d(x, lw["kernel"], lw.get("bias"), None, s, px, py, tr.out_hw(row), form="simt", kernel="simt")[0]


@functools.lru_cache(maxsize=None)
def _keys(j, precision):
    """What ROWS[j] covers in `precision`: case_keys of its plan, and the residual-scale keys that the residuals of both GPU runs (the
    source's output on the same seeded inputs, in the form's storage) earn."""
    row, stream_k, seed = ROWS[j]
    half = precision == "fp16"
    with tempfile.TemporaryDirectory() as d:
        path = d + "/case.json"
        tr.write_case(row, path, seed)
        om = oracle.Model(path)
    res_keys = None
    for r in range(2):
        x = exact.model_input(tr.case_input(row, 1000 * seed + r), half)[0]
        got = set(tr.residual_keys(exact.stored(_source_output(om, row, x), half), precision))
        res_keys = got if res_keys is None else res_keys & got
    return tuple(tr.case_keys(row, precision, tr.case_plan(row, precision, cp.SMS, stream_k))) + tuple(res_keys)


def _covered(rows):
    return {key for j in rows for precision in tr.FORMS for key in _keys(j, precision)}


ALL = list(range(len(ROWS)))


def test_table_reaches_every_key():
    missing = [key for key in tr.required_keys() if key not in _covered(ALL)]
    assert not missing, "not covered: %s" % missing


@pytest.mark.parametrize("i", range(len(ROWS)))
def test_every_row_is_needed(i):
    # each row covers a key no other row does, so that removing or changing one shows up as a named missing key
    alone = _covered([i]) - _covered(ALL[:i] + ALL[i + 1:])
    assert alone & set(tr.required_keys()), ROWS[i]


def test_scale_rows_put_their_residual_at_scale():
    # the residual-scale keys come from the residual itself: the 1e-4 row's source output is mostly products, not its bias
    for j, (row, stream_k, seed) in enumerate(ROWS):
        if row[10] == 1e-4:
            assert all(tr.RES_SUBNORMAL + " [%s]" % f in _keys(j, f) for f in tr.FORMS), row
        if row[10] == 1.0:
            assert not any(tr.RES_SUBNORMAL in key or tr.RES_255 in key for f in tr.FORMS for key in _keys(j, f)), row


@pytest.mark.parametrize("row,stream_k,seed", ROWS, ids=["%s%d" % ("sk" if r[1] else "", r[2]) for r in ROWS])
def test_cases_are_planned_as_the_gpu_test_expects(row, stream_k, seed):
    n, h, w, ic, oc, k, s, padding, mode, act, scale = row
    for precision in tr.FORMS:
        p = tr.case_plan(row, precision, cp.SMS, stream_k)
        # the tested convolution: conv_umma_kernel with its residual, on a pre-padded copy when it pads by replicate / reflect
        assert p["path"] == cp.IGEMM and p["terms"] == exact.TERMS[precision], (row, precision, p)
        assert stream_k or not p["sk"], (row, precision)  # stream-K only where the planner is asked to consider it
        if mode is not None:
            assert p["pad_mode"] == cp.PAD_CONSTANT and p["pad_x"] == p["pad_y"] == 0 and p["prepad_h"] == (out := tr.out_hw(row))[0] - 1 + k \
                and p["prepad_w"] == out[1] - 1 + k, (row, p)
        # the residual source: a tensor-core convolution with zero padding and no residual of its own (the row window with <= 8
        # input channels), whose output the test reads back as the residual
        ps = tr.case_plan(row, precision, cp.SMS, stream_k, layer=tr.SRC)
        assert ps["path"] == (cp.ROWWIN if ic <= 8 else cp.IGEMM) and ps["prepad_h"] == 0, (row, precision, ps)
        assert ps == cp.reference_plan((h, w, ic), (*tr.out_hw(row), oc), k, s, ps["pad_x"], ps["pad_y"], pad_mode=tr.PAD_MODE[tr.src_mode(row)],
                                       may_feed=True,
                                       n=n, precision=precision, stream_k=stream_k)


def test_prepadded_small_channel_case_runs_the_implicit_gemm():
    # <= 8 input channels with replicate / reflect padding and a residual: the pre-pad probe (no residual) fits the row window, the
    # residual rules that out, and the implicit GEMM reads the pre-padded copy - whose channel extent is below its 64-channel box
    small = [row for row in tr.TABLE if row[3] <= 8]
    assert {row[8] for row in small} == {"reflect", "replicate"}
    for row in small:
        n, h, w, ic, oc, k, s, padding, mode, act, scale = row
        probe = cp.plan((h, w, ic), (*tr.out_hw(row), oc), k, s, k // 2, k // 2, pad_mode=tr.PAD_MODE[mode], n=n)
        assert probe["path"] == cp.ROWWIN
        assert tr.case_plan(row, "fp32x3", cp.SMS)["path"] == cp.IGEMM


# ---- defect sensitivity ----------------------------------------------------------------------------------------------------
def _defect_case(tmp, row, precision):
    """The Add of a case row restated as the GPU test restates it, from the input and a residual the source convolution would
    produce (float64 restatement, stored in the form's storage). Returns (restate(residual, at), ref, bound, residual, plan)."""
    n, h, w, ic, oc, k, s, padding, mode, act, scale = row
    path = str(tmp / ("defect_%s.json" % precision))
    tr.write_case(row, path, seed=7)
    om = oracle.Model(path)
    half = precision == "fp16"
    x = exact.model_input(tr.case_input(row, 7), half)[0].astype(np.float32)
    ohw = tr.out_hw(row)
    lw = om.w[tr.SRC]
    px, py = (0, 0) if k == 1 else (k // 2, k // 2)
    res = exact.stored(exact.conv2d(x, lw["kernel"], lw.get("bias"), None, s, px, py, ohw)[0], half).astype(np.float32)
    p = tr.case_plan(row, precision, cp.SMS)
    shape = (n, *ohw, oc)

    def restated(r, at=None):
        return tr.restate_case(om, x, r, tr.kernel_name(p), shape, precision, at)

    ref, bound = restated(res)
    return restated, ref, bound, res, p


def _middle_tile(p, shape):
    """Output pixels (at) of the middle pixel box of the first channel tile, and that tile's 128 channels."""
    n, oh, ow, oc = shape
    m = p["tiles_x"] * p["tiles_y"] * p["tiles_n"] // 2
    bx, by, bn = m % p["tiles_x"], (m // p["tiles_x"]) % p["tiles_y"], m // (p["tiles_x"] * p["tiles_y"])
    ni, oy, ox = np.meshgrid(np.arange(bn * p["tn"], min(n, (bn + 1) * p["tn"])), np.arange(by * p["th"], min(oh, (by + 1) * p["th"])),
                             np.arange(bx * p["tw"], min(ow, (bx + 1) * p["tw"])), indexing="ij")
    return (ni.ravel(), oy.ravel(), ox.ravel()), np.arange(0, min(oc, p["n_blk"]))


# one 128-channel tile of single images and one of stacked images (their rows of the GPU table)
DEFECT_ROWS = [next(r for r in tr.TABLE if r[:5] == (33, 32, 32, 64, 200)), next(r for r in tr.TABLE if r[0] == 500)]


@pytest.mark.parametrize("precision", tr.FORMS)
@pytest.mark.parametrize("row", DEFECT_ROWS, ids=["single", "stacked"])
def test_residual_defects_in_one_tile_are_caught(tmp_path, row, precision):
    restated, ref, bound, res, p = _defect_case(tmp_path, row, precision)
    assert p["n_blk"] == 128 and (p["tn"] > 1) == (row[0] == 500), p
    at, chans = _middle_tile(p, ref.shape)
    ni, oy, ox = at
    assert exact.check(ref, ref, bound, "")[1] == 0
    s0, s1 = chans[:64], chans[64:]
    assert len(s1) == 64

    def residual(edit):
        r = res.copy()
        edit(r)
        return r

    def zero_slab1(r):
        r[..., s1] = 0

    def slab0_for_slab1(r):
        r[..., s1] = res[..., s0]

    def previous_output(r):  # the staging buffer still holding slab 0's stored output
        r[..., s1] = exact.stored(ref[..., s0], precision == "fp16")

    def neighbour_image(r):
        r[:] = np.roll(res, 1, axis=0)

    def drop_lo(r):
        r[:] = exact.f16(res)

    def row_shift(r):
        r[:, :-1] = res[:, 1:]
        r[:, -1] = 0

    defects = {"residual missing from slab 1": (zero_slab1, s1), "slab 0's residual used for slab 1": (slab0_for_slab1, s1),
               "previous slab's output read back as the residual": (previous_output, s1),
               "a neighbouring image's residual": (neighbour_image, chans), "residual box shifted by one output row": (row_shift, chans)}
    if precision != "fp16":
        defects["residual lo plane dropped"] = (drop_lo, chans)
    for what, (edit, ch) in defects.items():
        bad_vals = restated(residual(edit), at)[0]
        got = ref.copy()
        got[ni[:, None], oy[:, None], ox[:, None], ch[None, :]] = bad_vals[:, ch]
        ratio, bad = exact.check(got, ref, bound, what)
        assert bad > 0, (what, precision, ratio)
