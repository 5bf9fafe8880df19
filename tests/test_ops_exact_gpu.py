"""The per-operator C ABI (snnb_*_launch, snnb_weights_pack_*, snnb_tensor_upload / download_*, snnb_graph_capture_*) held to
oracle/exact.py's float64 restatements, at what only a caller of the ABI can reach: pad_x != pad_y on every convolution and depthwise
path (with H != W, so a swapped pair shows), output sizes chosen by the caller (every bottom and right padding B, R in [0, k - 1]),
the plan inputs only a descriptor sets (the forced algo, weights packed for another (stride, pad_x), the context's precision at each
launch), dense through a 1x1 implicit GEMM with images stacked per tile, and the ABI's refusals.

Each case uploads its operands and checks that the download is exact.stored of them bit for bit, restates the operation from the
downloaded tensors, launches it under set_precision("fp32x3") and ("fp16w"), and holds the output to the restatement within its
per-element bound (data moves bit-identical; outputs above SAMPLE_ABOVE pixels at exact.sample_pixels points). It asserts the kernels
launched (snnb_debug_launches) and, for convolutions, that last_conv_variant is the plan snnb_debug_conv_launch gives for the ABI's
own query: no pre-pad copy, no feed copy, the row window only for the pack descriptor's (stride, pad_x), stream-K when the algo asks.
The file prints the worst |err| / bound per entry point and conv variant and fails if an entry point, an expected conv variant or a
depthwise kernel was never launched (test_ops_exact_cpu.py holds the tables to the header and the plans to the variant list without
a GPU).
"""
import collections
import ctypes as C
import fnmatch

import numpy as np
import pytest

from oracle import exact
from shadernn_b200 import core
from shadernn_b200._lib import lib, vp

import test_conv_plan as cp

pytestmark = pytest.mark.gpu

FORMS = ("fp32x3", "fp16w")
SAMPLE_ABOVE = 20000  # output pixels above which a launch is restated at exact.sample_pixels points
PAD_MODE = {"none": cp.PAD_NONE, "constant": cp.PAD_CONSTANT, "replicate": cp.PAD_REPLICATE, "reflect": cp.PAD_REFLECT}
ALGO = {"auto": cp.AUTO, "simt": cp.ALGO_SIMT, "tcgen05": cp.TCGEN05, "tcgen05-streamk": cp.STREAMK}
PATH_NAME = ["none", "simt", "igemm", "rowwin", "rowwin-feed"]
KERNEL_OF_PATH = {"igemm": "igemm", "rowwin": "rowwin", "simt": "simt"}

# every entry point of the per-operator surface this file launches (test_ops_exact_cpu.py: each one the header declares)
ENTRY_POINTS = ["snnb_tensor_upload_nhwc", "snnb_tensor_download_nhwc", "snnb_tensor_upload_c4hw4", "snnb_tensor_download_c4hw4",
                "snnb_weights_pack_conv2d", "snnb_weights_pack_depthwise", "snnb_weights_pack_dense", "snnb_weights_pack_channels",
                "snnb_conv2d_launch", "snnb_depthwise_launch", "snnb_maxpool_launch", "snnb_avgpool_launch", "snnb_add_launch",
                "snnb_batchnorm_launch", "snnb_activation_launch", "snnb_dense_launch", "snnb_softmax_launch", "snnb_argmax1",
                "snnb_flatten_launch", "snnb_concat_launch", "snnb_upsample_launch", "snnb_pad_launch", "snnb_instancenorm_launch",
                "snnb_subpixel_launch", "snnb_graph_capture_begin", "snnb_graph_capture_end", "snnb_graph_launch"]
DW_KERNELS = ["depthwise_tma_kernel<1>", "depthwise_tma_kernel<2>", "depthwise_kernel<3, 1, 4>", "depthwise_kernel<3, 2, 4>", "depthwise_generic_kernel"]


def expected_conv_variants():
    """The conv variants the table must launch: SIMT; conv_umma with NB 32, 64, 128 in TERMS 2 and 3, stream-K and split-K in both
    forms; the row window in TERMS 2 and 3 with NB 32 and 64."""
    umma = ["conv_umma_kernel<%d, %d, false>" % (t, nb) for t in (2, 3) for nb in (32, 64, 128)]
    sk = ["conv_umma stream-K TERMS=%d" % t for t in (2, 3)]
    split = ["conv_umma split-K TERMS=%d" % t for t in (2, 3)]
    rowwin = ["conv_rowwin_kernel<%d, 0, %d>" % (t, nb) for t in (2, 3) for nb in (32, 64)]
    return ["simt"] + umma + sk + split + rowwin


def variant_keys(v):
    """The keys of expected_conv_variants a last_conv_variant record stands for."""
    if v["path"] == "igemm":
        keys = ["conv_umma_kernel<%d, %d, %s>" % (v["terms"], v["n_blk"], "true" if v["stream_k"] else "false")]
        if v["stream_k"]:
            keys.append("conv_umma stream-K TERMS=%d" % v["terms"])
        if v["ksplit"] > 1:
            keys.append("conv_umma split-K TERMS=%d" % v["terms"])
        return keys
    if v["path"] == "rowwin":
        return ["conv_rowwin_kernel<%d, %d, %d>" % (v["terms"], v["fks"], v["n_blk"])]
    return [v["path"]]


# ---- the tables --------------------------------------------------------------------------------------------------------------
# A convolution: input n x h x w x ic, oc filters of k x k, stride s, left / top pads (pad_x, pad_y) and bottom / right pads (B, R)
# that only the output size the caller allocates implies. row: the (stride, pad_x) the weights are packed for (default the launch's).
Conv = collections.namedtuple("Conv", "why n h w ic oc k s px py B R mode act alpha algo res bn row scale")


def conv(why, n, h, w, ic, oc, k, s, px, py, B, R, mode="constant", act="", alpha=0.0, algo="auto", res=False, bn=False, row=None, scale=1.0):
    return Conv(why, n, h, w, ic, oc, k, s, px, py, B, R, mode, act, alpha, algo, res, bn, row or (s, px), scale)


def conv_out(c):
    return (c.h + c.py + c.B - c.k) // c.s + 1, (c.w + c.px + c.R - c.k) // c.s + 1


CONV = [
    # conv_umma_kernel: NB 32 / 64 / 128, pads both ways round, every B and R of k = 3 and k = 5
    conv("igemm nb32 bn var -1e-3", 2, 13, 17, 16, 24, 3, 1, 1, 2, 0, 1, act="relu", bn=True),
    conv("igemm nb32 pads swapped", 2, 17, 13, 20, 24, 3, 1, 2, 0, 2, 0, act="leakyRelu", alpha=0.3),
    conv("igemm stride 2", 2, 11, 14, 32, 48, 3, 2, 0, 1, 1, 2, act="sigmoid"),
    conv("igemm stride 2 pads swapped", 2, 14, 11, 32, 64, 3, 2, 1, 0, 2, 1, act="relu6", bn=True),
    conv("igemm nb64", 4, 44, 45, 16, 48, 3, 1, 0, 1, 1, 2, act="tanh"),
    conv("igemm nb128 pads swapped", 4, 44, 45, 16, 96, 3, 1, 1, 0, 2, 1, act="SiLU", bn=True),
    conv("igemm oc 200", 1, 9, 12, 24, 200, 3, 1, 1, 0, 2, 2, act="tanh"),
    conv("igemm k5", 2, 12, 9, 16, 40, 5, 1, 3, 1, 4, 0, act="SiLU"),
    conv("igemm k5 stride 2", 2, 15, 19, 24, 32, 5, 2, 1, 4, 3, 2),
    conv("igemm k4 (even k)", 2, 10, 13, 16, 24, 4, 1, 2, 1, 3, 0, act="leakyRelu", alpha=-0.25),
    conv("igemm residual", 2, 10, 13, 32, 64, 3, 1, 2, 1, 1, 0, act="relu6", res=True),
    conv("igemm residual pads swapped", 2, 13, 10, 16, 24, 3, 1, 0, 2, 2, 1, act="tanh", res=True, bn=True),
    conv("igemm split-K", 2, 6, 8, 256, 64, 3, 1, 1, 0, 1, 2, act="relu"),
    conv("igemm stream-K partial wave", 1, 136, 128, 128, 32, 3, 1, 1, 0, 2, 1, algo="tcgen05-streamk"),
    conv("igemm forced, k1 pads", 2, 7, 10, 32, 40, 1, 1, 1, 2, 0, 0, algo="tcgen05"),
    conv("igemm k1 pads stride 2", 2, 11, 8, 16, 24, 1, 2, 2, 1, 0, 0, act="relu"),
    # conv_rowwin_kernel: IC <= 8, weights packed for the launch's (stride, pad_x)
    conv("rowwin nb32", 2, 15, 21, 3, 16, 3, 1, 1, 2, 1, 0, act="relu", bn=True),
    conv("rowwin nb32 pads swapped", 2, 21, 15, 8, 32, 3, 1, 2, 0, 0, 2, act="sigmoid"),
    conv("rowwin nb64 k5 stride 2", 2, 13, 18, 8, 48, 5, 2, 2, 1, 3, 1, act="leakyRelu", alpha=0.3),
    conv("rowwin nb64 k7 stride 2", 1, 20, 17, 4, 64, 7, 2, 3, 0, 6, 5, act="SiLU", bn=True),
    conv("rowwin k1 pads", 2, 9, 6, 4, 16, 1, 1, 2, 1, 0, 0),
    conv("rowwin forced", 2, 12, 9, 5, 40, 3, 2, 0, 1, 2, 0, algo="tcgen05", act="tanh"),
    # weights packed for another (stride, pad_x): never the row window
    conv("packed for (1, 1), launched pad_x 2", 2, 13, 18, 8, 24, 3, 1, 2, 1, 0, 2, row=(1, 1)),
    conv("packed for (2, 2), launched stride 1", 2, 10, 7, 4, 16, 3, 1, 2, 0, 1, 1, row=(2, 2), act="relu"),
    # conv2d_simt_kernel: forced on tensor-core shapes, AUTO's fallback for replicate / reflect, 9 <= IC <= 15, stride 3, even k
    conv("simt forced", 2, 11, 9, 32, 40, 3, 1, 0, 2, 2, 1, algo="simt", act="leakyRelu", alpha=0.3, bn=True),
    conv("simt forced residual", 2, 9, 11, 16, 24, 3, 2, 2, 1, 0, 2, algo="simt", act="relu", res=True),
    conv("simt forced rowwin shape", 2, 14, 11, 4, 16, 3, 1, 1, 2, 2, 0, algo="simt", act="relu6"),
    conv("simt reflect", 2, 9, 12, 16, 24, 3, 1, 2, 1, 1, 2, mode="reflect", act="tanh", bn=True),
    conv("simt reflect pads swapped k5", 2, 12, 9, 8, 16, 5, 2, 1, 3, 4, 0, mode="reflect"),
    conv("simt replicate", 2, 10, 7, 5, 12, 3, 2, 1, 2, 2, 0, mode="replicate", act="sigmoid"),
    conv("simt replicate residual", 2, 7, 10, 24, 16, 3, 1, 0, 1, 0, 1, mode="replicate", act="SiLU", res=True),
    conv("simt ic 12", 2, 12, 15, 12, 20, 3, 1, 2, 0, 1, 2, act="leakyRelu", alpha=-0.25),
    conv("simt stride 3", 2, 14, 17, 20, 16, 3, 3, 2, 0, 0, 2, act="relu"),
    conv("simt stride 3 pads swapped", 2, 17, 14, 9, 8, 5, 3, 0, 3, 3, 4),
    conv("simt k4", 2, 12, 15, 12, 20, 4, 1, 1, 2, 3, 0, act="relu6"),
    conv("simt k2 stride 2", 2, 9, 14, 10, 8, 2, 2, 1, 0, 1, 1, act="tanh"),
    conv("simt k1 pads", 2, 5, 8, 12, 8, 1, 2, 1, 0, 0, 0, act="sigmoid", bn=True),
]

# depthwise: (why, n, h, w, c, k, s, pad_x, pad_y, B, R, act, alpha, bias, bn)
DW = [
    ("tma s1", 2, 29, 37, 20, 3, 1, 0, 1, 2, 1, "relu6", 0.0, False, True),
    ("tma s1 pads swapped", 2, 37, 29, 136, 3, 1, 1, 0, 0, 2, "leakyRelu", 0.3, True, True),
    ("tma s2", 2, 31, 27, 136, 3, 2, 1, 0, 2, 0, "", 0.0, True, True),
    ("tma s2 pads swapped", 2, 25, 33, 20, 3, 2, 0, 2, 1, 2, "SiLU", 0.0, False, True),
    ("cuda-core s1", 2, 7, 5, 20, 3, 1, 1, 0, 2, 1, "tanh", 0.0, True, True),
    ("cuda-core s1 pads swapped", 2, 5, 7, 12, 3, 1, 0, 2, 1, 0, "relu", 0.0, False, True),
    ("cuda-core s2", 2, 5, 9, 20, 3, 2, 0, 1, 2, 2, "sigmoid", 0.0, True, False),
    ("cuda-core s2 pads swapped", 2, 9, 5, 24, 3, 2, 2, 0, 0, 1, "leakyRelu", -0.25, True, True),
    ("generic k5", 2, 17, 15, 24, 5, 2, 3, 1, 4, 0, "leakyRelu", 0.3, True, True),
    ("generic k5 pads swapped", 2, 15, 17, 20, 5, 1, 0, 4, 2, 3, "", 0.0, False, True),
    ("generic stride 3", 2, 20, 22, 20, 3, 3, 2, 0, 1, 2, "tanh", 0.0, True, False),
]


def dw_out(h, w, k, s, px, py, B, R):
    return (h + py + B - k) // s + 1, (w + px + R - k) // s + 1


def dw_kernel(oh, ow, k, s):
    """launch_depthwise's choice on split storage (depthwise_tma_supported's half-tile rule)."""
    if k == 3 and s in (1, 2):
        tw, th = (16, 8) if s == 1 else (8, 4)
        if ow * oh >= 0.5 * (-(-ow // tw) * tw) * (-(-oh // th) * th):
            return "depthwise_tma_kernel<%d>" % s
        return "depthwise_kernel<3, %d, 4>" % s
    return "depthwise_generic_kernel"


# dense: (why, n, input h, w, c, n_out, act); n_in = h w c
DENSE = [
    ("n_in 12 (simt)", 3, 1, 1, 12, 20, "relu"),
    ("n_in 12 from 2x3x2 softmax", 2, 2, 3, 2, 10, "softmax"),
    ("n_in 64 n1", 1, 1, 1, 64, 40, ""),
    ("n_in 64 n130 (two tiles)", 130, 1, 1, 64, 40, "tanh"),
    ("n_in 32 n256 softmax", 256, 1, 1, 32, 24, "softmax"),
    ("n_in 60 from 3x4x5", 2, 3, 4, 5, 7, "leakyRelu"),
    ("square 48", 4, 1, 1, 48, 48, "sigmoid"),
]
DENSE_SQUARE = 6  # the row with n_in == n_out
DENSE_ALPHA = 0.3

# pools at the start-inside limit: (n, h, w, c, k, s), out = (in - 1) // s + 1
POOL = [(2, 13, 11, 20, 2, 3), (2, 14, 10, 12, 3, 3), (2, 13, 16, 20, 5, 2), (2, 9, 12, 3, 3, 1), (1, 10, 7, 9, 2, 2)]
# upsample: (n, h, w, c, scale, bilinear, dh, dw): output floor(in scale) + (dh, dw)
UPSAMPLE = [(2, 5, 7, 12, 1.5, False, 1, -1), (2, 6, 5, 20, 1.7, False, -1, 1), (1, 7, 4, 3, 2.5, False, 1, 1),
            (2, 5, 7, 12, 1.5, True, 1, -1), (2, 6, 5, 20, 1.7, True, -1, 1), (1, 7, 4, 3, 2.5, True, 1, 1), (2, 4, 6, 9, 1.2, True, -1, -1)]
# pad: (n, h, w, c, pad_x, pad_y, out h, out w, mode)
PAD = [(2, 6, 7, 20, 1, 3, 11, 9, "constant"), (2, 6, 7, 3, 3, 1, 9, 12, "replicate"), (2, 5, 8, 12, 2, 4, 13, 11, "reflect"),
       (1, 4, 6, 3, 2, 7, 13, 9, "reflect"), (1, 6, 4, 5, 7, 1, 9, 13, "reflect"), (2, 5, 6, 8, 0, 2, 8, 7, "none"),
       (1, 4, 5, 3, 4, 2, 9, 12, "replicate")]
CONCAT = [(2, 5, 6, 3, 5), (2, 7, 4, 13, 20), (1, 3, 5, 8, 1)]
ACTS = [("", 0.0), ("relu", 0.0), ("relu6", 0.0), ("tanh", 0.0), ("sigmoid", 0.0), ("leakyRelu", 0.3), ("SiLU", 0.0)]
C4HW4 = [5, 6, 7]


# ---- running ------------------------------------------------------------------------------------------------------------------
class Run:
    """One context's launches under one precision: uploads checked bit for bit, the worst |err| / bound per entry point and variant."""

    def __init__(self, ctx, precision, seen):
        self.ctx, self.precision, self.seen = ctx, precision, seen
        self.keep = []

    def note(self, key, what, ratio):
        if self.seen.get(key, (None, -1.0))[1] < ratio:
            self.seen[key] = ("%s %s" % (what, self.precision), ratio)

    def tensor(self, x):
        """Upload x; the download must be exact.stored(x) bit for bit. Returns (tensor, the stored values)."""
        t = core.ImageTexture(self.ctx, *x.shape)
        t.upload(x)
        got = t.download()
        want = exact.stored(x, False)
        assert np.array_equal(got, want, equal_nan=True), ("upload", x.shape)
        self.note("snnb_tensor_upload_nhwc", "%s" % (x.shape,), 0.0)
        self.note("snnb_tensor_download_nhwc", "%s" % (x.shape,), 0.0)
        self.keep.append(t)
        return t, got

    def out(self, n, h, w, c):
        t = core.ImageTexture(self.ctx, n, h, w, c)
        self.keep.append(t)
        return t

    def launch(self, name, fn, *args):
        self.ctx.debug_launches(clear=True)
        rc = fn(*args)
        assert rc == 0, (name, rc, lib().snnb_last_error())
        self.ctx.sync()
        return self.ctx.debug_launches(clear=True)

    def hold(self, entry, what, got, ref, bound, launched, want, at=None):
        """got (downloaded) against (ref, bound); the launched kernels against the fnmatch patterns `want`."""
        assert len(launched) == len(want) and all(fnmatch.fnmatchcase(k, p) for k, p in zip(launched, want)), (what, launched, want)
        if at is not None:
            got = got[at]
        assert got.shape == ref.shape, (what, got.shape, ref.shape)
        ratio, bad = exact.check(got, ref, bound, entry)
        if bad:
            err = np.abs(got.astype(np.float64) - ref)
            k = np.unravel_index(np.argmax(np.where(err <= bound, 0, err / np.maximum(bound, 1e-300))), err.shape)
            raise AssertionError("%s %s: %d elements outside the bound, worst |err|/bound %.3g; at %s got %r ref %r bound %.3g (launched %s)" % (
                what, self.precision, bad, ratio, k, float(got[k]), float(ref[k]), float(bound[k]), launched))
        self.note(entry, what, ratio)
        return ratio


def sample_at(n, oh, ow, seed):
    return exact.sample_pixels(n, oh, ow, [(16, 8, 1), (8, 4, 1)], seed=seed) if n * oh * ow > SAMPLE_ABOVE else None


def bn_params(rng, c, clamp_channel=True):
    """BN of c channels; channel 1 at var = -1e-3, where var + 1e-3 is 0 and max(sqrt(.), 1e-4) applies (gamma ~ 1e-4 keeps the
    folded weights of that channel ordinary)."""
    bn = {"gamma": rng.uniform(0.5, 1.5, c), "beta": rng.uniform(-0.2, 0.2, c), "mean": rng.uniform(-0.2, 0.2, c), "var": rng.uniform(0.3, 1.5, c)}
    bn = {k: v.astype(np.float32) for k, v in bn.items()}
    if clamp_channel and c > 1:
        bn["var"][1] = np.float32(-1e-3)
        bn["gamma"][1] = np.float32(1.3e-4)
    return bn


def bn_ptrs(bn):
    return [None] * 4 if bn is None else [bn[k].ctypes.data_as(vp) for k in ("gamma", "beta", "mean", "var")]


def pack_conv(ctx, c, wt, bias, bn):
    d = core.conv_desc(c.ic, c.oc, c.k, c.row[0], c.row[1], c.py, c.mode, c.act, c.alpha, c.algo)
    wh = vp()
    rc = lib().snnb_weights_pack_conv2d(ctx.h, C.byref(d), wt.ctypes.data_as(vp), bias.ctypes.data_as(vp), *bn_ptrs(bn), C.byref(wh))
    assert rc == 0, lib().snnb_last_error()
    return core.Weights(wh)


def conv_plan(c, precision, sms):
    """snnb_debug_conv_launch with the query snnb_conv2d_launch makes."""
    oh, ow = conv_out(c)
    return cp.plan((c.h, c.w, c.ic), (oh, ow, c.oc), c.k, c.s, c.px, c.py, pad_mode=PAD_MODE[c.mode], residual=c.res, algo=ALGO[c.algo],
                   may_prepad=False, may_feed=False, row=c.row, n=c.n, precision=precision, stream_k=c.algo == "tcgen05-streamk", sms=sms)


def plan_variant(p):
    return {"path": PATH_NAME[p["path"]], "terms": p["terms"], "n_blk": p["n_blk"], "ksplit": p["ksplit"], "stream_k": p["sk"], "fks": p["fks"]}


def conv_operands(c, seed):
    rng = np.random.default_rng(seed)
    x = (rng.uniform(-1, 1, (c.n, c.h, c.w, c.ic)) * c.scale).astype(np.float32)
    wt = (rng.standard_normal((c.oc, c.ic, c.k, c.k)) / np.sqrt(c.ic * c.k * c.k)).astype(np.float32)
    bias = rng.uniform(-0.2, 0.2, c.oc).astype(np.float32)
    bn = bn_params(rng, c.oc) if c.bn else None
    res = rng.uniform(-1, 1, (c.n,) + conv_out(c) + (c.oc,)).astype(np.float32) if c.res else None
    return x, wt, bias, bn, res


def restate_conv(c, xin, wt, bias, bn, rin, v, precision, at=None):
    form = "simt" if v["path"] == "simt" else precision
    return exact.conv2d(xin, wt, bias, bn, c.s, c.px, c.py, conv_out(c), c.act, c.alpha, residual=rin, form=form, kernel=KERNEL_OF_PATH[v["path"]],
                        pad_mode=c.mode if c.mode != "none" else "constant", at=at)


def run_conv(r, c, seed, sms, w=None):
    """One snnb_conv2d_launch of table row c: returns its variant."""
    x, wt, bias, bn, res = conv_operands(c, seed)
    tin, xin = r.tensor(x)
    tres, rin = r.tensor(res) if c.res else (None, None)
    oh, ow = conv_out(c)
    tout = r.out(c.n, oh, ow, c.oc)
    w = w or pack_conv(r.ctx, c, wt, bias, bn)
    d = core.conv_desc(c.ic, c.oc, c.k, c.s, c.px, c.py, c.mode, c.act, c.alpha, c.algo)
    launched = r.launch("snnb_conv2d_launch", lib().snnb_conv2d_launch, r.ctx.h, C.byref(d), w.h, tin.h, tres.h if tres else None, tout.h)
    v = r.ctx.last_conv_variant()
    assert v == plan_variant(conv_plan(c, r.precision, sms)), (c.why, v)
    want = {"simt": "conv2d_simt_kernel", "igemm": "conv_umma_kernel*", "rowwin": "conv_rowwin_kernel"}[v["path"]]
    got = tout.download()
    at = sample_at(c.n, oh, ow, seed)
    ref, bound = restate_conv(c, xin, wt, bias, bn, rin, v, r.precision, at)
    ratio = r.hold("snnb_conv2d_launch", c.why, got, ref, bound, launched, [want], at)
    for key in variant_keys(v):
        r.note(key, c.why, ratio)
    return v


def run_depthwise(r, row, seed):
    why, n, h, w, c, k, s, px, py, B, R, act, alpha, bias_on, bn_on = row
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (n, h, w, c)).astype(np.float32)
    wk = rng.standard_normal((c, k, k)).astype(np.float32) / k
    bias = rng.uniform(-0.2, 0.2, c).astype(np.float32) if bias_on else None
    bn = bn_params(rng, c) if bn_on else None
    tin, xin = r.tensor(x)
    oh, ow = dw_out(h, w, k, s, px, py, B, R)
    tout = r.out(n, oh, ow, c)
    d = core.conv_desc(c, c, k, s, px, py, "constant", act, alpha)
    wh = vp()
    assert lib().snnb_weights_pack_depthwise(r.ctx.h, C.byref(d), wk.ctypes.data_as(vp), None if bias is None else bias.ctypes.data_as(vp),
                                             *bn_ptrs(bn), C.byref(wh)) == 0, lib().snnb_last_error()
    wobj = core.Weights(wh)
    r.note("snnb_weights_pack_depthwise", why, 0.0)
    launched = r.launch("snnb_depthwise_launch", lib().snnb_depthwise_launch, r.ctx.h, C.byref(d), wobj.h, tin.h, tout.h)
    got = tout.download()
    at = sample_at(n, oh, ow, seed)
    ref, bound = exact.depthwise(xin, wk, bias, bn, s, px, py, (oh, ow), act, alpha, at=at)
    kern = dw_kernel(oh, ow, k, s)
    ratio = r.hold("snnb_depthwise_launch", "depthwise " + why, got, ref, bound, launched, [kern], at)
    r.note(kern, "depthwise " + why, ratio)


def dense_pack(ctx, kern, bias):
    wh = vp()
    assert lib().snnb_weights_pack_dense(ctx.h, kern.shape[1], kern.shape[0], kern.ctypes.data_as(vp), bias.ctypes.data_as(vp), C.byref(wh)) == 0, \
        lib().snnb_last_error()
    return core.Weights(wh)


def restate_dense(xin, kern, bias, act, alpha, v, precision):
    """exact.conv2d of the 1x1 GEMM on the HWC-flattened input, then the soft-max over the units where asked."""
    n = xin.shape[0]
    x1 = np.asarray(xin, np.float32).reshape(n, 1, 1, -1)
    form = "simt" if v["path"] == "simt" else precision
    soft = act == "softmax"
    ref, bound = exact.conv2d(x1, kern[:, :, None, None], bias, None, 1, 0, 0, (1, 1), "" if soft else act, alpha, form=form,
                              kernel=KERNEL_OF_PATH[v["path"]])
    if soft:  # the pre-activation's bound already carries a store: an upper bound of the stored logits' error
        ref, bound = exact.softmax_rows(ref, bound)
        bound = bound + exact.store_bound(ref, False)
    return ref, bound


def run_dense(r, row, seed, sms):
    why, n, h, w, c, n_out, act = row
    rng = np.random.default_rng(seed)
    n_in = h * w * c
    x = rng.uniform(-1, 1, (n, h, w, c)).astype(np.float32)
    kern = (rng.standard_normal((n_out, n_in)) / np.sqrt(n_in)).astype(np.float32)
    bias = rng.uniform(-0.2, 0.2, n_out).astype(np.float32)
    tin, xin = r.tensor(x)
    tout = r.out(n, 1, 1, n_out)
    wobj = dense_pack(r.ctx, kern, bias)
    r.note("snnb_weights_pack_dense", why, 0.0)
    alpha = DENSE_ALPHA if act == "leakyRelu" else 0.0
    launched = r.launch("snnb_dense_launch", lib().snnb_dense_launch, r.ctx.h, wobj.h, core.ACT[act], alpha, tin.h, tout.h)
    v = r.ctx.last_conv_variant()
    q = cp.plan((1, 1, n_in), (1, 1, n_out), 1, 1, 0, 0, pad_mode=cp.PAD_NONE, may_prepad=False, row=(0, 0), n=n, precision=r.precision, sms=sms)
    assert v == plan_variant(q), (why, v)
    want = (["flatten_kernel"] if h * w > 1 else []) + [{"simt": "conv2d_simt_kernel", "igemm": "conv_umma_kernel*"}[v["path"]]] + \
        (["softmax_kernel"] if act == "softmax" else [])
    got = tout.download()
    ref, bound = restate_dense(xin, kern, bias, act, alpha, v, r.precision)
    ratio = r.hold("snnb_dense_launch", "dense " + why, got, ref, bound, launched, want)
    for key in variant_keys(v):
        r.note(key, "dense " + why, ratio)


def run_pools(r, seed):
    rng = np.random.default_rng(seed)
    for i, (n, h, w, c, k, s) in enumerate(POOL):
        x = rng.uniform(-1, 1, (n, h, w, c)).astype(np.float32)
        tin, xin = r.tensor(x)
        oh, ow = (h - 1) // s + 1, (w - 1) // s + 1
        kern = "pool_kernel<%d>" % (k if k in (2, 3) else 0)
        for avg, entry in ((False, "snnb_maxpool_launch"), (True, "snnb_avgpool_launch")):
            tout = r.out(n, oh, ow, c)
            launched = r.launch(entry, getattr(lib(), entry), r.ctx.h, k, s, tin.h, tout.h)
            ref, bound = exact.avgpool(xin, k, s, (oh, ow)) if avg else exact.maxpool(xin, k, s, (oh, ow))
            r.hold(entry, "pool n%d %dx%d c%d k%d s%d" % (n, h, w, c, k, s), tout.download(), ref, bound, launched, [kern])


def run_elementwise(r, seed):
    rng = np.random.default_rng(seed)
    ctx = r.ctx
    for i, (act, alpha) in enumerate(ACTS):
        shape = [(2, 9, 11, 20), (2, 5, 7, 3), (1, 8, 6, 13)][i % 3]
        a, b = (rng.uniform(-3, 3, shape).astype(np.float32) for _ in range(2))
        ta, av = r.tensor(a)
        tb, bv = r.tensor(b)
        to = r.out(*shape)
        launched = r.launch("snnb_add_launch", lib().snnb_add_launch, ctx.h, core.ACT[act], alpha, ta.h, tb.h, to.h)
        r.hold("snnb_add_launch", "add %s %s" % (shape, act), to.download(), *exact.add(av, bv, act, alpha), launched, ["add_kernel"])
        to = r.out(*shape)
        launched = r.launch("snnb_activation_launch", lib().snnb_activation_launch, ctx.h, core.ACT[act], alpha, ta.h, to.h)
        r.hold("snnb_activation_launch", "activation %s %s" % (shape, act), to.download(), *exact.activation(av, act, alpha), launched, ["chanwise_kernel"])
        bn = bn_params(rng, shape[3])
        wh = vp()
        assert lib().snnb_weights_pack_channels(ctx.h, shape[3], *bn_ptrs(bn), C.byref(wh)) == 0, lib().snnb_last_error()
        wb = core.Weights(wh)
        r.note("snnb_weights_pack_channels", "batchnorm", 0.0)
        to = r.out(*shape)
        launched = r.launch("snnb_batchnorm_launch", lib().snnb_batchnorm_launch, ctx.h, wb.h, core.ACT[act], alpha, ta.h, to.h)
        r.hold("snnb_batchnorm_launch", "batchnorm %s %s (var -1e-3 at channel 1)" % (shape, act), to.download(), *exact.batchnorm(av, bn, act, alpha),
               launched, ["chanwise_kernel"])
    for shape, act, alpha in (((2, 12, 9, 20), "relu", 0.0), ((1, 7, 10, 3), "leakyRelu", 0.3), ((2, 40, 33, 8), "", 0.0)):
        x = rng.uniform(-1, 1, shape).astype(np.float32)
        x[..., 0] += 100  # a large mean next to unit noise
        tx, xv = r.tensor(x)
        g, b = rng.uniform(0.5, 1.5, shape[3]).astype(np.float32), rng.uniform(-0.2, 0.2, shape[3]).astype(np.float32)
        wh = vp()
        assert lib().snnb_weights_pack_channels(ctx.h, shape[3], g.ctypes.data_as(vp), b.ctypes.data_as(vp), None, None, C.byref(wh)) == 0
        wi = core.Weights(wh)
        to = r.out(*shape)
        launched = r.launch("snnb_instancenorm_launch", lib().snnb_instancenorm_launch, ctx.h, wi.h, core.ACT[act], alpha, tx.h, to.h)
        r.hold("snnb_instancenorm_launch", "instancenorm %s %s" % (shape, act), to.download(), *exact.instancenorm(xv, g, b, act, alpha), launched,
               ["instnorm_partial_kernel", "instnorm_finalize_kernel", "instnorm_apply_kernel"])
    for shape in ((3, 2, 5, 37), (2, 1, 1, 1000)):
        x = rng.uniform(-100, 100, shape).astype(np.float32)  # only the max subtraction keeps expf finite
        tx, xv = r.tensor(x)
        to = r.out(*shape)
        launched = r.launch("snnb_softmax_launch", lib().snnb_softmax_launch, ctx.h, tx.h, to.h)
        r.hold("snnb_softmax_launch", "softmax %s logits +-100" % (shape,), to.download(), *exact.softmax(xv), launched, ["softmax_kernel"])


def run_moves(r, seed):
    rng = np.random.default_rng(seed)
    ctx = r.ctx
    for n, h, w, c, scale, bil, dh, dw in UPSAMPLE:
        tx, xv = r.tensor(rng.uniform(-1, 1, (n, h, w, c)).astype(np.float32))
        oh, ow = int(np.floor(h * scale)) + dh, int(np.floor(w * scale)) + dw
        to = r.out(n, oh, ow, c)
        launched = r.launch("snnb_upsample_launch", lib().snnb_upsample_launch, ctx.h, scale, int(bil), tx.h, to.h)
        ref, bound = exact.upsample_bilinear(xv, scale, (oh, ow)) if bil else exact.upsample_nearest(xv, (oh, ow), scale=scale)
        r.hold("snnb_upsample_launch", "upsample %s x%g %dx%d -> %dx%d" % ("bilinear" if bil else "nearest", scale, h, w, oh, ow), to.download(), ref, bound,
               launched, ["upsample_kernel"])
    for n, h, w, c, px, py, oh, ow, mode in PAD:
        tx, xv = r.tensor(rng.uniform(-1, 1, (n, h, w, c)).astype(np.float32))
        to = r.out(n, oh, ow, c)
        launched = r.launch("snnb_pad_launch", lib().snnb_pad_launch, ctx.h, px, py, core.PAD_MODE[mode], tx.h, to.h)
        ref, bound = exact.pad(xv, px, py, (oh, ow), "constant" if mode == "none" else mode)
        r.hold("snnb_pad_launch", "pad %s %dx%d pad_x %d pad_y %d -> %dx%d" % (mode, h, w, px, py, oh, ow), to.download(), ref, bound, launched, ["pad_kernel"])
    for n, h, w, ca, cb in CONCAT:
        ta, av = r.tensor(rng.uniform(-1, 1, (n, h, w, ca)).astype(np.float32))
        tb, bv = r.tensor(rng.uniform(-1, 1, (n, h, w, cb)).astype(np.float32))
        to = r.out(n, h, w, ca + cb)
        launched = r.launch("snnb_concat_launch", lib().snnb_concat_launch, ctx.h, ta.h, tb.h, to.h)
        r.hold("snnb_concat_launch", "concat %d + %d" % (ca, cb), to.download(), *exact.concat(av, bv), launched, ["concat_kernel"])
    for shape in ((2, 3, 5, 20), (2, 2, 3, 13), (3, 1, 1, 37)):
        tx, xv = r.tensor(rng.uniform(-1, 1, shape).astype(np.float32))
        to = r.out(shape[0], 1, 1, shape[1] * shape[2] * shape[3])
        launched = r.launch("snnb_flatten_launch", lib().snnb_flatten_launch, ctx.h, tx.h, to.h)
        r.hold("snnb_flatten_launch", "flatten %s" % (shape,), to.download(), *exact.flatten(xv), launched, ["flatten_kernel"])
    for n, h, w, rr in ((2, 5, 6, 2), (2, 4, 7, 3)):
        tx, xv = r.tensor(rng.uniform(-3, 3, (n, h, w, rr * rr)).astype(np.float32))
        to = r.out(n, h * rr, w * rr, 1)
        launched = r.launch("snnb_subpixel_launch", lib().snnb_subpixel_launch, ctx.h, rr, tx.h, to.h)
        r.hold("snnb_subpixel_launch", "subpixel r%d" % rr, to.download(), *exact.subpixel(xv, rr), launched, ["subpixel_kernel"])
    for n, c in ((5, 37), (3, 8)):
        x = rng.uniform(-1, 1, (n, 1, 1, c)).astype(np.float32)
        x[0, 0, 0, [3, 17 % c]] = 2.0  # a tie: the first maximum
        tx, xv = r.tensor(x)
        idx = (C.c_int * n)()
        launched = r.launch("snnb_argmax1", lib().snnb_argmax1, ctx.h, tx.h, idx)
        ref, bound = exact.argmax(xv.reshape(n, c))
        r.hold("snnb_argmax1", "argmax n%d c%d" % (n, c), np.array(list(idx), np.int64) - 1, ref.astype(np.float64), bound, launched, ["argmax_kernel"])


def c4hw4_of(x, swap=False):
    """The reference texture layout of NHWC values x: channel c at block c // 4, lane c % 4, padding lanes zero ([N, D, H, W, 4],
    D = ceil(C / 4)). swap: the two indices exchanged (block c % D, lane c // D), a misreading test_ops_exact_cpu.py shows is caught."""
    n, h, w, c = x.shape
    d = -(-c // 4)
    out = np.zeros((n, d, h, w, 4), np.float32)
    for ch in range(c):
        blk, lane = (ch % d, ch // d) if swap else (ch // 4, ch % 4)
        out[:, blk, :, :, lane] = x[..., ch]
    return out


def run_c4hw4(r, seed):
    """Round trips at C = 5, 6, 7 with N = 3: the C4HW4 download is the numpy permutation of the NHWC download, padding lanes zero, and
    a C4HW4 upload stores what an NHWC upload of the same values stores."""
    rng = np.random.default_rng(seed)
    for c in C4HW4:
        n, h, w = 3, 4, 5
        d = -(-c // 4)
        x = rng.uniform(-1, 1, (n, h, w, c)).astype(np.float32)
        t, xv = r.tensor(x)
        got = t.download_c4hw4()
        padded = np.zeros((n, h, w, 4 * d), np.float32)
        padded[..., :c] = xv
        assert np.array_equal(got, padded.reshape(n, h, w, d, 4).transpose(0, 3, 1, 2, 4)), ("download_c4hw4", c)  # the numpy permutation
        assert np.array_equal(got, c4hw4_of(xv)), ("download_c4hw4", c)
        assert not got[:, d - 1, ..., c - 4 * (d - 1):].any(), ("padding lanes", c)
        r.note("snnb_tensor_download_c4hw4", "c%d n%d" % (c, n), 0.0)
        src = rng.uniform(-1, 1, (n, d, h, w, 4)).astype(np.float32)  # the padding lanes carry values the upload must ignore
        t2 = r.out(n, h, w, c)
        t2.upload_c4hw4(src)
        nhwc = src.transpose(0, 2, 3, 1, 4).reshape(n, h, w, 4 * d)[..., :c]
        assert np.array_equal(t2.download(), exact.stored(nhwc, False)), ("upload_c4hw4", c)
        r.note("snnb_tensor_upload_c4hw4", "c%d n%d" % (c, n), 0.0)


def test_every_abi_launch_within_its_bound(ctx):
    import torch
    sms = torch.cuda.get_device_properties(ctx.device).multi_processor_count
    seen = {}
    try:
        for precision in FORMS:
            ctx.set_precision(precision)
            r = Run(ctx, precision, seen)
            for i, c in enumerate(CONV):
                run_conv(r, c, 100 + i, sms)
                r.note("snnb_weights_pack_conv2d", c.why, 0.0)
            for i, row in enumerate(DW):
                run_depthwise(r, row, 200 + i)
            for i, row in enumerate(DENSE):
                run_dense(r, row, 300 + i, sms)
            run_pools(r, 400)
            run_elementwise(r, 500)
            run_moves(r, 600)
            run_c4hw4(r, 700)
            r.keep.clear()
            run_graph(ctx, precision, sms, seen)
    finally:
        ctx.set_precision("fp32x3")
    keys = ENTRY_POINTS + expected_conv_variants() + DW_KERNELS
    for key in keys + sorted(k for k in seen if k not in keys):
        print("%-40s %s" % (key, "worst |err|/bound %.3g (%s)" % (seen[key][1], seen[key][0]) if key in seen else "NOT LAUNCHED"))
    missing = [k for k in keys if k not in seen]
    assert not missing, missing


# ---- precision switching -------------------------------------------------------------------------------------------------------
def test_precision_follows_the_context_at_each_launch(ctx):
    """One packed weight set launched under fp32x3, fp16w, fp32x3: each launch's product form is the context's at that launch."""
    import torch
    sms = torch.cuda.get_device_properties(ctx.device).multi_processor_count
    c = conv("precision switch", 2, 11, 14, 32, 48, 3, 1, 2, 0, 1, 2, act="relu", bn=True)
    x, wt, bias, bn, _ = conv_operands(c, 900)
    seen = {}
    try:
        w = None
        for precision in ("fp32x3", "fp16w", "fp32x3"):
            ctx.set_precision(precision)
            r = Run(ctx, precision, seen)
            w = w or pack_conv(ctx, c, wt, bias, bn)
            v = run_conv(r, c, 900, sms, w=w)
            assert v["path"] == "igemm" and v["terms"] == exact.TERMS[precision], (precision, v)
    finally:
        ctx.set_precision("fp32x3")


# ---- graph capture -------------------------------------------------------------------------------------------------------------
def run_graph(ctx, precision, sms, seen):
    """conv_umma with a residual -> add -> maxpool -> depthwise -> dense on a 1x1 input, captured once and replayed on two new inputs:
    every output within its bound, and bit for bit the eager launch's where the plan has no split-K or stream-K."""
    r = Run(ctx, precision, seen)
    c = conv("graph conv", 2, 6, 10, 32, 24, 3, 1, 1, 0, 2, 1, act="relu", res=True)
    rng = np.random.default_rng(800)
    _, wt, bias, bn, _ = conv_operands(c, 800)
    oh, ow = conv_out(c)
    shape_x, shape_r = (c.n, c.h, c.w, c.ic), (c.n, oh, ow, c.oc)
    tx, tr, ta = (r.out(*s) for s in (shape_x, shape_r, shape_r))
    t1, t2 = r.out(*shape_r), r.out(*shape_r)
    ph, pw = (oh - 1) // 3 + 1, (ow - 1) // 3 + 1  # maxpool k3 s3
    t3 = r.out(c.n, ph, pw, c.oc)
    # depthwise k3 s2 without top / left pads into a 1 x 1 output: the bottom / right padding is what the output size implies
    t4 = r.out(c.n, 1, 1, c.oc)
    t5 = r.out(c.n, 1, 1, 10)
    wconv = pack_conv(ctx, c, wt, bias, bn)
    dd = core.conv_desc(c.oc, c.oc, 3, 2, 0, 0, "constant", "relu6", 0.0)
    dwk = rng.standard_normal((c.oc, 3, 3)).astype(np.float32) / 3
    dbias = rng.uniform(-0.2, 0.2, c.oc).astype(np.float32)
    wh = vp()
    assert lib().snnb_weights_pack_depthwise(ctx.h, C.byref(dd), dwk.ctypes.data_as(vp), dbias.ctypes.data_as(vp), None, None, None, None, C.byref(wh)) == 0
    wdw = core.Weights(wh)
    dkern = (rng.standard_normal((10, c.oc)) / np.sqrt(c.oc)).astype(np.float32)
    dbias2 = rng.uniform(-0.2, 0.2, 10).astype(np.float32)
    wdense = dense_pack(ctx, dkern, dbias2)
    d = core.conv_desc(c.ic, c.oc, c.k, c.s, c.px, c.py, c.mode, c.act, c.alpha, c.algo)
    L = lib()

    def chain():
        rcs = [L.snnb_conv2d_launch(ctx.h, C.byref(d), wconv.h, tx.h, tr.h, t1.h),
               L.snnb_add_launch(ctx.h, core.ACT["leakyRelu"], 0.3, t1.h, ta.h, t2.h),
               L.snnb_maxpool_launch(ctx.h, 3, 3, t2.h, t3.h),
               L.snnb_depthwise_launch(ctx.h, C.byref(dd), wdw.h, t3.h, t4.h),
               L.snnb_dense_launch(ctx.h, wdense.h, core.ACT["sigmoid"], 0.0, t4.h, t5.h)]
        assert rcs == [0] * 5, (rcs, L.snnb_last_error())

    def inputs(seed):
        g = np.random.default_rng(seed)
        vals = []
        for t, s in ((tx, shape_x), (tr, shape_r), (ta, shape_r)):
            a = g.uniform(-1, 1, s).astype(np.float32)
            t.upload(a)
            vals.append(t.download())
            assert np.array_equal(vals[-1], exact.stored(a, False))
        return vals

    def outputs():
        return [t.download() for t in (t1, t2, t3, t4, t5)]

    inputs(801)
    chain()  # eagerly once: lazily created resources exist before the capture
    ctx.sync()
    v = ctx.last_conv_variant()
    assert v["path"] == "igemm" and v == plan_variant(conv_plan(c, precision, sms)), v
    dense_v = plan_variant(cp.plan((1, 1, c.oc), (1, 1, 10), 1, 1, 0, 0, pad_mode=cp.PAD_NONE, may_prepad=False, row=(0, 0), n=c.n,
                                   precision=precision, sms=sms))
    deterministic = v["ksplit"] == 1 and not v["stream_k"] and dense_v["ksplit"] == 1 and not dense_v["stream_k"]
    g = vp()
    assert L.snnb_graph_capture_begin(ctx.h) == 0, L.snnb_last_error()
    chain()
    assert L.snnb_graph_capture_end(ctx.h, C.byref(g)) == 0, L.snnb_last_error()
    try:
        for seed in (802, 803):
            xv, rv, av = inputs(seed)
            for t in (t1, t2, t3, t4, t5):  # stale results must not survive a replay
                t.upload(np.full(t.shape, np.nan, np.float32))
            assert L.snnb_graph_launch(g) == 0, L.snnb_last_error()
            ctx.sync()
            o1, o2, o3, o4, o5 = outputs()
            what = "graph replay seed %d" % seed
            r.hold("snnb_graph_launch", what + " conv", o1, *restate_conv(c, xv, wt, bias, bn, rv, v, precision), [], [])
            r.hold("snnb_graph_launch", what + " add", o2, *exact.add(o1, av, "leakyRelu", 0.3), [], [])
            r.hold("snnb_graph_launch", what + " maxpool", o3, *exact.maxpool(o2, 3, 3, (ph, pw)), [], [])
            r.hold("snnb_graph_launch", what + " depthwise", o4, *exact.depthwise(o3, dwk, dbias, None, 2, 0, 0, (1, 1), "relu6"), [], [])
            r.hold("snnb_graph_launch", what + " dense", o5, *restate_dense(o4, dkern, dbias2, "sigmoid", 0.0, dense_v, precision), [], [])
            chain()
            ctx.sync()
            eager = outputs()
            if deterministic:
                for a, b in zip((o1, o2, o3, o4, o5), eager):
                    assert np.array_equal(a, b), (what, "graph and eager launches differ")
    finally:
        L.snnb_graph_destroy(g)
    r.note("snnb_graph_capture_begin", "graph chain", 0.0)
    r.note("snnb_graph_capture_end", "graph chain", 0.0)


# ---- refusals -------------------------------------------------------------------------------------------------------------------
def refused(rc, *words):
    """A refused call: nonzero status and an error naming the cause (the callers check that the output is untouched)."""
    msg = lib().snnb_last_error().decode()
    assert rc != 0, words
    assert all(w in msg for w in words), (msg, words)


def test_refusals_leave_output_and_context_intact(ctx):
    rng = np.random.default_rng(1000)
    L = lib()

    def setup(c):
        x, wt, bias, bn, _ = conv_operands(c, 1001)
        tin = core.ImageTexture.from_numpy(ctx, x)
        tout = core.ImageTexture(ctx, c.n, *conv_out(c), c.oc)
        marker = rng.uniform(-1, 1, tout.shape).astype(np.float32)
        tout.upload(marker)
        return tin, tout, pack_conv(ctx, c, wt, bias, bn), tout.download()

    cases = [
        (conv("forced on reflect", 1, 8, 9, 32, 16, 3, 1, 1, 0, 1, 2, mode="reflect", algo="tcgen05"), ("tensor-core path", "pad_mode=3")),
        (conv("forced on IC 12", 1, 8, 9, 12, 16, 3, 1, 1, 0, 1, 2, algo="tcgen05"), ("tensor-core path", "IC=12")),
        (conv("forced on IC 8, packed for (1, 0)", 1, 8, 9, 8, 16, 3, 1, 1, 0, 1, 2, algo="tcgen05", row=(1, 0)), ("tensor-core path", "IC=8")),
        (conv("forced stream-K on stride 3", 1, 10, 11, 16, 16, 3, 3, 1, 0, 1, 2, algo="tcgen05-streamk"), ("tensor-core path", "s=3")),
    ]
    for c, words in cases:
        tin, tout, w, before = setup(c)
        d = core.conv_desc(c.ic, c.oc, c.k, c.s, c.px, c.py, c.mode, c.act, c.alpha, c.algo)
        refused(L.snnb_conv2d_launch(ctx.h, C.byref(d), w.h, tin.h, None, tout.h), *words)
        ctx.sync()
        assert np.array_equal(tout.download(), before), c.why
    x = rng.uniform(-1, 1, (2, 9, 7, 16)).astype(np.float32)
    tin = core.ImageTexture.from_numpy(ctx, x)
    tout = core.ImageTexture(ctx, 2, 9, 7, 16)
    tout.upload(rng.uniform(-1, 1, tout.shape).astype(np.float32))
    before = tout.download()
    wk = rng.standard_normal((16, 3, 3)).astype(np.float32)
    for mode in ("replicate", "reflect"):
        d = core.conv_desc(16, 16, 3, 1, 1, 1, mode)
        wh = vp()
        assert L.snnb_weights_pack_depthwise(ctx.h, C.byref(d), wk.ctypes.data_as(vp), None, None, None, None, None, C.byref(wh)) == 0
        w = core.Weights(wh)
        refused(L.snnb_depthwise_launch(ctx.h, C.byref(d), w.h, tin.h, tout.h), "snnb_depthwise_launch", "pad_mode %d" % core.PAD_MODE[mode])
        ctx.sync()
        assert np.array_equal(tout.download(), before), mode
    idx = (C.c_int * 2)(-7, -7)
    refused(L.snnb_argmax1(ctx.h, tin.h, idx), "snnb_argmax1", "9x7")
    assert list(idx) == [-7, -7]
    # the context still launches, and gets it right
    z = rng.uniform(-1, 1, (2, 1, 1, 16)).astype(np.float32)
    assert np.array_equal(core.argmax1(ctx, z) - 1, exact.argmax(exact.stored(z, False).reshape(2, 16))[0])
    c = conv("after the refusals", 2, 8, 9, 32, 16, 3, 1, 1, 0, 1, 2)
    x, wt, bias, bn, _ = conv_operands(c, 1002)
    got = core.conv2d(ctx, x, wt, bias, None, c.s, c.px, c.py, out_hw=conv_out(c))
    ref, bound = exact.conv2d(exact.stored(x, False), wt, bias, None, c.s, c.px, c.py, conv_out(c), form="fp32x3")
    assert exact.check(got, ref, bound, "conv")[1] == 0
