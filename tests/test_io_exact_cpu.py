"""The input / output transfer table without a GPU: its coverage list against the library's kernels, and the restatements of
oracle/exact.py it relies on. numpy float32 simulations of the kernels' own arithmetic (resize_u8_kernel contracted and not, quant_u8,
the arg-max) must sit inside the bounds, and each simulation mutated as a plausible bug must fall outside them somewhere in the data."""
import numpy as np
import pytest

from oracle import exact, oracle

import test_cuda_core_exact_cpu as cc
import test_io_exact_gpu as table

f32 = np.float32
# the transfer kernels' families (device-buffer kernels are templates over a type: the demangled name carries no arguments)
IO = ("split", "merge", "resize_u8", "device_input", "device_output", "argmax", "result_small")
MEAN4, NORM4 = table.MEAN4, table.NORM4


def test_every_transfer_kernel_has_a_case():
    have = cc._library_kernels()
    io = sorted(k for k in have if k.startswith(IO))
    assert "resize_u8_kernel" in io and "argmax_kernel" in io, io
    families = {k.split("<")[0] for k in table.COVERED}
    missing = [k for k in io if k.split("<")[0] not in families]
    assert not missing, "transfer kernels without a case in test_io_exact_gpu.py: %s" % missing
    assert not [k for k in families if k not in have], "COVERED names kernels the library does not have"


# ---- resize_u8_kernel ---------------------------------------------------------------------------------------------------------
def resize_sim(img, out_hw, mean4, norm4, linear, contract, half=False, mutation=None):
    """resize_u8_kernel in float32: resize_pos, resize_taps, ResizeTaps::blend (contract: the compiler fused the position's product
    and subtraction and each lerp's multiply-add), the normalisation and the store. mutation: a plausible bug."""
    n, sh, sw, c = img.shape
    oh, ow = out_hw
    ch = np.arange(c)
    mi = ch & 3 if mutation != "mean_by_c" else ch
    table_mean = np.concatenate([np.float32(mean4), np.float32(norm4), np.zeros(max(c, 8), f32)])  # U8Norm {mean[4], norm[4]}
    table_norm = np.concatenate([np.float32(norm4), np.zeros(max(c, 8), f32)])
    mean, norm = table_mean[mi].astype(f32), table_norm[mi].astype(f32)

    def pos(o, out, src):
        o = np.arange(o, dtype=f32)
        half_px = f32(0.5) if mutation != "no_half_pixel" else f32(0)
        q = (o + half_px) / f32(out)
        if not linear:
            return (q * f32(src)).astype(f32)
        if contract:
            return f32(np.float64(q) * src - 0.5)
        return ((q * f32(src)).astype(f32) - f32(0.5)).astype(f32)

    def taps(o, out, src):
        s = pos(o, out, src)
        if not linear:
            i = np.minimum(s.astype(np.int64), src - 1)
            return i, i, np.zeros(o, f32)
        f = np.floor(s)
        a = (s - f).astype(f32)
        i0 = np.clip(f.astype(np.int64), 0, src - 1)
        i1 = np.clip(f.astype(np.int64) + 1, 0, src - 1) if mutation != "x1_clamped_before" else np.clip(f.astype(np.int64), 0, src - 1) + 1
        return i0, i1, a

    x0, x1, ax = taps(ow, ow, sw)
    y0, y1, ay = taps(oh, oh, sh)
    src = np.zeros((n, sh + 1, sw + 1, c), f32)  # a tap past the edge reads 0
    src[:, :sh, :sw] = img

    def px(yy, xx):
        return src[:, yy][:, :, xx]
    p00, p01, p10, p11 = px(y0, x0), px(y0, x1), px(y1, x0), px(y1, x1)
    axb, ayb = ax[None, None, :, None], ay[None, :, None, None]
    if mutation == "swap_axy":  # the x lerps weighted by ay, the y lerp by ax
        axb, ayb = ayb, axb

    def lerp(a, b, t):
        if contract:
            return f32(np.float64(t) * np.float64((b - a).astype(f32)) + np.float64(a))
        return (a + (t * (b - a).astype(f32)).astype(f32)).astype(f32)
    v = p00 if not linear else lerp(lerp(p00, p01, axb), lerp(p10, p11, axb), ayb)
    return exact.stored(((v - mean).astype(f32) * norm).astype(f32), half)


# (source h, w, channels, output h, w): down, up, mixed, exact 2x / 3x both ways, 1 x N, N x 1, 1 x 1, a coarse source
SIZES = [(150, 233, 3, 64, 80), (40, 50, 3, 64, 80), (64, 96, 4, 32, 48), (90, 99, 1, 30, 33), (20, 30, 3, 40, 60), (8, 12, 20, 24, 36),
         (1, 57, 3, 16, 24), (45, 1, 4, 16, 24), (1, 1, 3, 16, 24), (1080, 1920, 3, 12, 20)]


@pytest.mark.parametrize("sh,sw,c,oh,ow", SIZES)
@pytest.mark.parametrize("linear", [True, False])
def test_resize_restatement_holds_the_kernel_arithmetic(sh, sw, c, oh, ow, linear):
    img = np.random.default_rng(sh * 7 + sw).integers(0, 256, (2, sh, sw, c), dtype=np.uint8)
    for half in (False, True):
        ref, bound = exact.resize_u8(img, (oh, ow), MEAN4, NORM4, linear, half)
        for contract in (False, True):
            got = resize_sim(img, (oh, ow), MEAN4, NORM4, linear, contract, half)
            ratio, bad = exact.check(got, ref, bound, "resize")
            assert bad == 0, (linear, half, contract, ratio)
        if not linear:
            mean = [MEAN4[i & 3] for i in range(c)]
            norm = [NORM4[i & 3] for i in range(c)]
            cands = exact.nearest_candidates(img, (oh, ow), mean, norm, half)
            assert np.any([got == v for v in cands], axis=0).all()


@pytest.mark.parametrize("linear", [True, False])
def test_resize_restatement_agrees_with_the_oracle(linear):
    img = np.random.default_rng(9).integers(0, 256, (2, 150, 233, 3), dtype=np.uint8)
    for out in ((64, 80), (300, 400)):
        ref, bound = exact.resize_u8(img, out, MEAN4, NORM4, linear, False)
        want = oracle.resize_normalize(img, out, MEAN4, NORM4, linear)
        assert exact.check(exact.stored(want, False), ref, bound, "resize")[1] == 0, out


def _outside(got, ref, bound):
    return exact.check(got, ref, bound, "mutation")[1] > 0


@pytest.mark.parametrize("mutation", ["no_half_pixel", "x1_clamped_before", "swap_axy", "mean_by_c"])
def test_resize_bound_catches_mutations(mutation):
    """Each mutation falls outside the bound on noisy images: the half-pixel offset, the right / bottom edge's second tap clamped before
    the + 1 (it reads past the edge), the two axes' weights swapped (on a non-square resize), mean and norm indexed by c (C = 20)."""
    img = np.random.default_rng(3).integers(0, 256, (2, 24, 31, 20), dtype=np.uint8)
    out = (40, 64)
    ref, bound = exact.resize_u8(img, out, MEAN4, NORM4, True, False)
    assert not _outside(resize_sim(img, out, MEAN4, NORM4, True, False), ref, bound)
    assert _outside(resize_sim(img, out, MEAN4, NORM4, True, False, mutation=mutation), ref, bound)
    if mutation in ("no_half_pixel", "mean_by_c"):
        ref, bound = exact.resize_u8(img, (12, 20), MEAN4, NORM4, False, False)
        assert _outside(resize_sim(img, (12, 20), MEAN4, NORM4, False, False, mutation=mutation), ref, bound)


# ---- storage, the NCHW tile -----------------------------------------------------------------------------------------------------
def test_stored_saturates_as_cvt_satfinite():
    v = np.array([1e6, -1e6, 100000.0, 65510.0, 65520.0, np.inf, -np.inf, np.nan, 2.0 ** -24 * 0.75, 65504.0], f32)
    split = exact.stored(v, False)
    assert np.array_equal(split[:7], f32([131008, -131008, 100000, 65510, 65520, 131008, -131008]))
    assert np.isnan(split[7]) and split[8] == f32(2.0 ** -24) and split[9] == 65504
    half = exact.stored(v, True)
    assert np.array_equal(half[:7], f32([65504, -65504, 65504, 65504, 65504, 65504, -65504])) and np.isnan(half[7])


def tiled_sim(x_nchw, transposed=False):
    """device_input_nchw_tiled_kernel<f32>: tiles of 32 pixels x 64 channels through shared memory, then NHWC (transposed: the tile's
    pixel and channel indices swapped on the way out)."""
    n, c, h, w = x_nchw.shape
    hw = h * w
    src = x_nchw.reshape(n, c, hw)
    out = np.zeros((n, hw, c), f32)
    for i in range(n):
        for p0 in range(0, hw, 32):
            for c0 in range(0, c, 64):
                s = np.zeros((64, 64), f32)  # the kernel's [64][33] tile, wide enough for the transposed read
                blk = src[i, c0:c0 + 64, p0:p0 + 32]
                s[:blk.shape[0], :blk.shape[1]] = blk
                for p in range(min(32, hw - p0)):
                    cs = np.arange(c0, min(c0 + 64, c))
                    out[i, p0 + p, cs] = s[p, cs - c0] if transposed else s[cs - c0, p]
    return exact.stored(out.reshape(n, h, w, c), False)


def test_tiled_transpose_mutation_is_caught():
    x = np.random.default_rng(4).uniform(-1, 1, (2, 70, 5, 9)).astype(f32)
    ref, bound = exact.model_input(x.transpose(0, 2, 3, 1), False)
    assert not _outside(tiled_sim(x), ref, bound)
    assert _outside(tiled_sim(x, transposed=True), ref, bound)


# ---- quant_u8 ----------------------------------------------------------------------------------------------------------------
def quant_sim(v, scale, offset, contract, away=False):
    v = np.asarray(v, f32)
    t = f32(np.float64(v) * f32(scale) + f32(offset)) if contract else ((v * f32(scale)).astype(f32) + f32(offset)).astype(f32)
    with np.errstate(invalid="ignore"):
        r = np.floor(np.abs(t) + f32(0.5)) * np.sign(t) if away else np.rint(t)
        return np.nan_to_num(np.minimum(np.maximum(r, 0), 255), nan=0.0)  # fminf(fmaxf(NaN, 0), 255) = 0


@pytest.mark.parametrize("scale,offset", table.QUANT)
def test_quant_restatement_holds_the_kernel_arithmetic(scale, offset):
    rng = np.random.default_rng(abs(int(scale * 10 + offset)))
    v = exact.stored(table.straddling(rng, (4000,), scale, offset), False)
    v[::3] = ((np.floor(v[::3] * 2 + offset) + 0.5 - offset) / 2).astype(f32) if scale == 2.0 else v[::3]
    v[5] = np.nan
    ref, bound = exact.quant_u8(v, scale, offset)
    for contract in (False, True):
        assert not _outside(quant_sim(v, scale, offset, contract), ref, bound), contract
    assert ref[5] == 0 and bound[5] == 0
    if scale == 2.0:  # exact ties: the bound is 0 there, and half away from zero lands on the odd neighbour
        assert _outside(quant_sim(v, scale, offset, False, away=True), ref, bound)
    v = exact.stored(rng.uniform(-50, 400, 4000), False)
    assert (exact.quant_u8(v, scale, offset)[1] == 0).mean() > 0.999  # only values within fp32 error of a half-integer go either way


# ---- arg-max -------------------------------------------------------------------------------------------------------------------
def argmax_sim(x, rule):
    """argmax_kernel's per-lane scan and warp reduction in numpy. rule "parent": best = -FLT_MAX, bi = INT_MAX, v > best (NaN never
    taken, an all-NaN image gives INT_MAX); "fixed": argmax_take / argmax_warp; "last": the fixed rule, keeping the last maximum."""
    n, c = x.shape
    none = 0x7fffffff
    out = np.zeros(n, np.int64)
    for i in range(n):
        lanes = []
        for lane in range(32):
            best, bi = (-3.402823466e+38, none) if rule == "parent" else (0.0, none)
            for ch in range(lane, c, 32):
                v = float(x[i, ch])
                if rule == "parent":
                    take = v > best
                else:
                    take = v == v and (bi == none or v > best or (rule == "last" and v == best))
                if take:
                    best, bi = v, ch
            lanes.append((best, bi))
        best, bi = lanes[0]
        for ob, oi in lanes[1:]:
            if rule == "parent":
                if ob > best or (ob == best and oi < bi):
                    best, bi = ob, oi
            elif oi != none and (bi == none or ob > best or (ob == best and (oi > bi if rule == "last" else oi < bi))):
                best, bi = ob, oi
        out[i] = bi if rule == "parent" else (0 if (np.isnan(x[i, 0]) or bi == none) else bi)
    return out


@pytest.mark.parametrize("c", [2, 31, 32, 33, 100])
def test_argmax_restatement(c):
    rng = np.random.default_rng(c)
    x = table.scores(rng, 40, c, table.ARGMAX_KINDS + ["nan0", "nan_later", "nan_all"])
    want, bound = exact.argmax(x)
    assert not bound.any()
    assert np.array_equal(argmax_sim(x, "fixed"), want)
    plain = table.scores(rng, 40, c, table.ARGMAX_KINDS)
    assert np.array_equal(exact.argmax(plain)[0], np.argmax(plain, axis=1))  # without NaN: the first maximum
    assert not np.array_equal(argmax_sim(plain, "last"), exact.argmax(plain)[0])  # the last maximum on ties
    assert not np.array_equal(argmax_sim(x, "parent"), want)  # the NaN rule before the fix
    allnan = np.full((1, c), np.nan, f32)
    assert exact.argmax(allnan)[0][0] == 0 and argmax_sim(allnan, "parent")[0] == 0x7fffffff


def test_argmax_is_max_element():
    """std::max_element: the running maximum moves on only when it compares below a later score."""
    def max_element(row):
        best = 0
        for j in range(1, len(row)):
            if row[best] < row[j]:
                best = j
        return best
    rng = np.random.default_rng(0)
    x = rng.integers(-2, 3, (500, 7)).astype(np.float64)
    x[rng.random(x.shape) < 0.2] = np.nan
    assert np.array_equal(exact.argmax(x)[0], [max_element(r) for r in x])
