"""TEST INFRASTRUCTURE - float64 restatements of single layers, each with a per-element error bound.

Every function takes the layer's input tensors exactly as the engine stored them (numpy fp32, downloaded from the device: the
hi + lo pair of the split-fp16 storage is exact in fp32, an fp16 value of the half-precision storage mode is exact too) and
returns (ref, bound): ref is the layer's operation evaluated in float64 on the operands the kernel multiplies, bound[i] an upper
bound of |kernel output - ref| derived below from the operands. A kernel is right when |got - ref| <= bound everywhere. Layers
that only move data return bound = 0: their outputs must be bit-identical.

Product forms of the tensor-core convolutions (csrc/kernels_umma.cu, `TERMS`), with the folded weight wv = w * scale (pack.cpp):
  fp32x3  A_hi*B_hi + A_hi*B_lo + A_lo*B_hi, B_hi + B_lo = the fp16 pair of wv. ref uses a * (B_hi + B_lo); the dropped A_lo*B_lo
          term is bounded by sum |A_lo| |B_lo| with |A_lo| <= 2^-11 |a| (1 + 2^-10) + 2^-25 (the lo half of an fp16 pair).
  fp16w   (A_hi + A_lo) * fp16_rn(wv): ref is that product exactly.
  fp16    A_hi * fp16_rn(wv) on tensors without lo planes (a = A_hi): ref is that product exactly.
  simt    conv2d_simt_kernel: fp32 FMAs on the fp32 folded weights wv, whatever the precision.

Accumulation error of a tensor-core K block. Hopper's wgmma does not accumulate with IEEE round-to-nearest. Fasi, Higham,
Mikaitis and Pranesh, "Numerical behavior of NVIDIA tensor cores", PeerJ Comput. Sci. 7:e330 (2021), measured the fp16 -> fp32
inner products of V100, T4 and A100: the products are exact, the addends of one fused step (products and the accumulator) are
aligned to the largest of them and truncated, and the sum is normalised by truncation (round toward zero). We assume that model
on Hopper with a fused step of f >= 4 products and at most 24 significant bits kept below the leading bit of the largest addend
(keeping more bits only tightens it). A step then errs by at most (f + 1) 2^-23 max|addend| for the truncated addends plus
2^-23 |result| for the normalisation, both <= 2^-23 (|c| + sum |p|). One m64nNk16 instruction is 16 / f such steps, so it errs by
at most (16 + 2 * 16 / f) 2^-23 (|c_in| + sum|p|) <= KAPPA (|c_in| + sum|p|), KAPPA = 24 * 2^-23 (f = 4). A K block issues
TERMS instructions per K step of 16 columns into a fresh accumulator (k_blocks gives the kernels' K order: 64 channels of one tap
for conv_umma_kernel; one filter row, two taps per step, for conv_rowwin_kernel; feed_rows_per_stage filter rows, four window
pixels per step, in its feed mode). The first instruction of a step sees |c_in| = |c_prev| and the hi*hi products; the others see
at most |c_prev| + sum|p| and products 2^-11 smaller. So a step errs by at most TERMS KAPPA (|c_prev| + A_step) STEP_SLACK,
A_step = sum over the step of |a| |w|, with c_prev the exact partial sum in the kernel's K order (evaluated in float64). Block sums are added to the tile's sum with fp32 round-to-nearest adds,
and split-K / stream-K partials likewise in some order: any order of adding nb block sums errs by at most (nb - 1) u sum|block|,
u = 2^-24 (recursive summation, Higham, "Accuracy and Stability of Numerical Algorithms", 2nd ed., eq. 4.4).

conv2d_simt_kernel and the CUDA-core kernels: a chain of n fp32 FMAs / adds errs by at most gamma_n sum|terms|, gamma_n = n u / (1 - n u)
(Higham, Lemma 3.1).

Epilogue (fp32, round to nearest): + bias, + residual: one rounding each, u |value|. Activations: relu, relu6 and max(v, v alpha)
are exact apart from v * alpha (u |v alpha|); tanhf carries 2 ulp and expf 2 ulp (CUDA C++ Programming Guide, "Mathematical
Functions", single precision, default -prec-div=true); sigmoid 1 / (1 + expf(-v)) and SiLU v / (1 + expf(-v)) add two correctly
rounded operations, so all three are held to ACT_ULPS = 4 ulp of the result, ulp <= 2^-23 |y|. An error e of the activation's
argument moves the result by at most L e: L = 1 (none, relu, relu6, tanh), max(1, |alpha|) (leaky), 1/4 (sigmoid), 1.1 (SiLU).

Output storage: hi = fp16_rn(v), lo = fp16_rn(v - hi) stores v to 2^-22 |v| + 2^-25 (the half ulp of lo, also at fp16's smallest
subnormal); the fp16 storage mode stores v to 2^-11 |v| + 2^-25. Second-order terms (an error times u) are covered by SLACK.

Chosen output pixels. Every function of a layer with a spatial output takes an optional at = (n_idx, oy_idx, ox_idx), integer arrays
of equal length; with it, it returns (ref, bound) at those output pixels only, for all channels, shaped [len(at), C]. The full
restatement is the same code run at every pixel: a pixel's operands are gathered from the input by the same index arithmetic, and
its float64 operations are the same ones in the same order. The one place where the order could depend on the other pixels is a
BLAS matrix product, whose kernel (and with it the order of a dot product's additions) depends on the matrix shape; conv2d
therefore multiplies in blocks of exactly ROWS pixel rows, the last one zero-filled, so a pixel's value is the same bits whichever
pixels are evaluated with it. InstanceNorm's per-(image, channel) statistics are computed over the whole plane either way.
"""
import numpy as np

# Pixel rows per matrix product of conv2d (module docstring, "Chosen output pixels"). It cannot follow the number of pixels asked
# for, so a small restatement (a dense head of a few images, a tiny test layer) pays for a whole zero-filled block: negligible next to
# the Python overhead of its K steps. A smaller block would multiply that overhead on the large restatements instead.
ROWS = 2048
U = 2.0 ** -24          # fp32 unit roundoff
KAPPA = 24 * 2.0 ** -23  # one m64nNk16 wgmma, relative to |c_in| + sum |p| (module docstring)
ACT_ULPS = 4
SLACK = 1 + 2.0 ** -10   # second-order terms
STEP_SLACK = 1 + 2.0 ** -8  # the hi*lo / lo*hi products of a K step next to its hi*hi products (module docstring)
LIPSCHITZ = {"": 1.0, "linear": 1.0, "relu": 1.0, "relu6": 1.0, "tanh": 1.0, "sigmoid": 0.25, "SiLU": 1.1}
TERMS = {"fp32x3": 3, "fp16w": 2, "fp16": 1}


def gamma(n):
    return n * U / (1 - n * U)


def f16(x):
    """fp16 round to nearest even, back in float64 (numpy's conversion is IEEE round to nearest)."""
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float64)


def store_bound(y, half):
    """|stored - v| for an output value v ~ y: one unit of the storage format."""
    return np.abs(y) * (2.0 ** -11 if half else 2.0 ** -22) * SLACK + 2.0 ** -25


FP16_MAX = 65504.0


def sat16(v):
    """cvt.rn.satfinite.f16.f32 of fp32 values, back in float32: round to nearest even, then values past fp16's range (infinities
    included) saturate to +-65504; NaN stays NaN."""
    with np.errstate(over="ignore"):
        h = np.asarray(v, np.float32).astype(np.float16).astype(np.float32)
    return np.clip(h, np.float32(-FP16_MAX), np.float32(FP16_MAX))  # np.clip keeps NaN


def stored(v, half):
    """What the storage makes of fp32 values v: hi + lo (split-fp16) or fp16 alone, as float32. Both planes saturate
    (store8's cvt.rn.satfinite): hi holds at most +-65504, lo = sat(v - hi) as well, so split-fp16 holds at most +-131008 and fp16
    storage +-65504. NaN stays NaN."""
    v = np.asarray(v, np.float32)
    hi = sat16(v)
    if half:
        return hi
    with np.errstate(invalid="ignore"):
        return hi + sat16(v - hi)


def act64(v, act, alpha):
    if act in ("", "linear", "none", "identity"):
        return v
    if act == "relu":
        return np.maximum(v, 0.0)
    if act == "relu6":
        return np.minimum(np.maximum(v, 0.0), 6.0)
    if act in ("leakyRelu", "leaky_relu"):
        return np.maximum(v, v * float(np.float32(alpha)))
    if act == "tanh":
        return np.tanh(v)
    if act == "sigmoid":
        return 1.0 / (1.0 + np.exp(-v))
    if act == "SiLU":
        return v / (1.0 + np.exp(-v))
    raise ValueError("activation %r" % act)


def act_bound(pre, e_pre, y, act, alpha):
    """Error of act(v) computed in fp32 from v = pre +- e_pre, against act(pre) in exact arithmetic."""
    if act in ("leakyRelu", "leaky_relu"):
        a = abs(float(np.float32(alpha)))
        return max(1.0, a) * e_pre + U * a * np.abs(pre)
    if act in ("tanh", "sigmoid", "SiLU"):
        return LIPSCHITZ[act] * e_pre + ACT_ULPS * 2.0 ** -23 * np.abs(y) + 2.0 ** -149
    return LIPSCHITZ[act if act != "none" else ""] * e_pre


def fold(w_oihw, bias, bn):
    """pack.cpp:bn_fold in float32: returns (wv [oc, ic, k, k] fp32, shift [oc] fp32)."""
    w = np.asarray(w_oihw, np.float32)
    oc = w.shape[0]
    b = np.zeros(oc, np.float32) if bias is None else np.asarray(bias, np.float32)
    if bn is None:
        return w, b
    g, be, m, v = (np.asarray(bn[k], np.float32) for k in ("gamma", "beta", "mean", "var"))
    s = np.maximum(np.sqrt(v + np.float32(0.001)), np.float32(0.0001))
    scale = (g / s).astype(np.float32)
    return (w * scale[:, None, None, None]).astype(np.float32), ((b - m) * scale + be).astype(np.float32)


def weight_operand(wv, form):
    """The weights the product multiplies (float64) and, for fp32x3, the dropped lo plane |B_lo|."""
    hi = f16(wv)
    if form == "fp32x3":
        lo = f16(np.asarray(wv, np.float32) - hi.astype(np.float32))
        return hi + lo, np.abs(lo)
    if form in ("fp16w", "fp16"):
        return hi, None
    return np.asarray(wv, np.float64), None  # simt


def src_coord(s, size, mode="constant"):
    """The input coordinate an outside coordinate s reads: replicate, a single reflection, or -1 (zero) for constant padding and
    for a coordinate still outside after one reflection (src_coord in kernels_simt.cu)."""
    s = np.asarray(s)
    if mode == "replicate":
        return np.clip(s, 0, size - 1)
    if mode == "reflect":
        s = np.where(s < 0, -s, s)
        s = np.where(s >= size, 2 * size - 2 - s, s)
    return np.where((s >= 0) & (s < size), s, -1)


def pixels(at, n, oh, ow):
    """(n_idx, oy_idx, ox_idx) of the chosen output pixels, or of every pixel in NHWC order when at is None."""
    if at is None:
        return tuple(np.indices((n, oh, ow)).reshape(3, -1))
    return tuple(np.asarray(a, np.int64).reshape(-1) for a in at)


def shaped(v, at, n, oh, ow):
    """Rows of per-pixel values -> [n, oh, ow, C] for a full restatement, [len(at), C] for chosen pixels."""
    return v.reshape(n, oh, ow, -1) if at is None else v.reshape(len(at[0]), -1)


def gather(x, ni, iy, ix, mode="constant", dtype=np.float64):
    """x[ni, iy, ix, :] as [len(ni), C]; coordinates outside x read as padding mode `mode` does (src_coord)."""
    n, h, w, c = x.shape
    sy, sx = src_coord(iy, h, mode), src_coord(ix, w, mode)
    ok = (sy >= 0) & (sx >= 0)
    v = np.asarray(x[ni, np.where(ok, sy, 0), np.where(ok, sx, 0)], dtype)
    v[~ok] = 0
    return v


def row_plan_steps(k, stride, pad_x):
    """conv_rowwin_kernel's K steps of one filter row (make_row_plan, snnb_internal.h): the taps of each column parity, two per step."""
    steps = []
    for par in range(stride):
        js = [j for j in range(k) if (j - pad_x) % stride == par]
        steps += [js[q:q + 2] for q in range(0, len(js), 2)]
    return steps


def feed_rows_per_stage(k):
    """Filter rows per K block of conv_rowwin_kernel's feed mode: ceil(k / 4) groups as even as possible (launch_conv2d_rowwin)."""
    g = (k + 3) // 4
    return (k + g - 1) // g


def feed_plan_steps(k, pad_x):
    """The feed mode's K steps of one filter row (make_feed_plan): step q reads window pixels 4q .. 4q + 3, tap t sits at d + t."""
    px = (pad_x + 1) & ~1
    d = px - pad_x
    ksteps = (((d + k + 1) // 2 + 1) & ~1) // 2
    return [[t for t in range(k) if 4 * q <= d + t < 4 * q + 4] for q in range(ksteps)]


def k_blocks(kernel, k, stride, pad_x, ic):
    """The kernel's K order: a list of K blocks (one fresh accumulator each), each a list of K steps of 16 columns (TERMS wgmmas each),
    each a list of (ky, kx, channel slice) operand pieces."""
    allc = slice(0, ic)
    if kernel == "igemm":  # K block = 64 channels of one tap, taps in (ky, kx) order
        return [[[(ky, kx, slice(c1, min(c1 + 16, ic, c0 + 64)))] for c1 in range(c0, min(c0 + 64, ic), 16)]
                for ky in range(k) for kx in range(k) for c0 in range(0, ic, 64)]
    if kernel == "rowwin":  # K block = one filter row
        return [[[(ky, j, allc) for j in taps] for taps in row_plan_steps(k, stride, pad_x)] for ky in range(k)]
    if kernel == "feed":  # K block = feed_rows_per_stage filter rows
        r = feed_rows_per_stage(k)
        steps = feed_plan_steps(k, pad_x)
        return [[[(ky, t, allc) for t in taps] for ky in range(r0, min(r0 + r, k)) for taps in steps] for r0 in range(0, k, r)]
    raise ValueError(kernel)


def conv2d(x, w_oihw, bias, bn, stride, pad_x, pad_y, out_hw, act="", alpha=0.0, residual=None, form="fp32x3", kernel="igemm",
           half_out=False, pad_mode="constant", at=None):
    """Conv2D as the engine runs it: output column ox reads input column ox * stride + kx - pad_x, row oy * stride + ky - pad_y
    (the kernels' (pad_x, pad_y) = the layer's (T, L) offsets). kernel: "igemm" (conv_umma_kernel), "rowwin" / "feed"
    (conv_rowwin_kernel, regular or feed mode) or "simt". residual: [n, oh, ow, oc]. Returns (ref, bound) [n, oh, ow, oc], or
    [len(at), oc] at the output pixels `at`."""
    n, h, w, ic = np.shape(x)
    wv, shift = fold(w_oihw, bias, bn)
    oc, _, k, _ = wv.shape
    oh, ow = out_hw
    s = int(stride)
    T = TERMS.get(form, 0)
    wq, wlo = weight_operand(wv, form)
    ni, oy, ox = pixels(at, n, oh, ow)
    M = len(ni)
    y = np.zeros((M, oc))
    e_acc = np.zeros((M, oc))
    blocks = None if kernel == "simt" else k_blocks(kernel, k, s, pad_x, ic)
    for r0 in range(0, M, ROWS):  # ROWS pixel rows per product, whatever else is evaluated (module docstring)
        r1 = min(r0 + ROWS, M)
        taps = {}
        for ky in range(k):
            for kx in range(k):
                X = np.zeros((ROWS, ic))
                X[:r1 - r0] = gather(x, ni[r0:r1], oy[r0:r1] * s + ky - pad_y, ox[r0:r1] * s + kx - pad_x, pad_mode)
                taps[ky, kx] = (X, np.abs(X), wq[:, :, ky, kx].T)
        yc = np.zeros((ROWS, oc))
        ec = np.zeros((ROWS, oc))
        if kernel == "simt":
            a_all = np.zeros((ROWS, oc))
            for X, aX, W in taps.values():
                yc += X @ W
                a_all += aX @ np.abs(W)
            ec = gamma(k * k * ic) * a_all
        else:
            blocks_abs = np.zeros((ROWS, oc))
            for block in blocks:
                c = np.zeros((ROWS, oc))
                for step in block:
                    A = np.zeros((ROWS, oc))
                    P = np.zeros((ROWS, oc))
                    for ky, kx, ch in step:
                        X, aX, W = taps[ky, kx]
                        A += aX[:, ch] @ np.abs(W[ch])
                        P += X[:, ch] @ W[ch]
                    ec += T * STEP_SLACK * KAPPA * (np.abs(c) + A)
                    c += P
                yc += c
                blocks_abs += np.abs(c)
            ec += max(len(blocks) - 1, 0) * U * blocks_abs
        if wlo is not None:
            for (ky, kx), (X, aX, W) in taps.items():
                ec += (aX * (2.0 ** -11 * SLACK) + 2.0 ** -25) @ wlo[:, :, ky, kx].T
        y[r0:r1], e_acc[r0:r1] = yc[:r1 - r0], ec[:r1 - r0]
    pre = y + shift.astype(np.float64)
    e_pre = e_acc * SLACK + U * np.abs(pre)
    if residual is not None:
        pre = pre + np.asarray(residual).reshape(n, oh, ow, oc)[ni, oy, ox].astype(np.float64)
        e_pre += U * np.abs(pre)
    ref = act64(pre, act, alpha)
    bound = act_bound(pre, e_pre, ref, act, alpha) * SLACK + store_bound(ref, half_out)
    return shaped(ref, at, n, oh, ow), shaped(bound, at, n, oh, ow)


def dense(x, kernel_out_in, bias, act="", form="fp32x3", half_out=False, at=None):
    """Dense on a 1 x 1 map (or flattened HWC): a 1x1 conv_umma_kernel launch. at: output pixels (n_idx, 0, 0)."""
    n = x.shape[0]
    x1 = np.asarray(x, np.float64).reshape(n, 1, 1, -1)
    kern = np.asarray(kernel_out_in, np.float32)
    return conv2d(x1, kern[:, :, None, None], bias, None, 1, 0, 0, (1, 1), act, 0.0, form=form, half_out=half_out, at=at)


def gap_dense(x, kernel_out_in, bias, act="", alpha=0.0, softmax_out=False, half_out=False):
    """gap_dense_kernel: the fp32 channel means (summed in pixel order, then over parts, divided by H W), then fp32 FMAs on the fp32
    weights over the channels, + bias, then the activation or the soft-max over the units."""
    x = np.asarray(x, np.float64)
    n, h, w, c = x.shape
    hw = h * w
    mean = x.reshape(n, hw, c).mean(axis=1)
    e_mean = gamma(hw + 1) * np.abs(x).reshape(n, hw, c).sum(axis=1) / hw
    kern = np.asarray(kernel_out_in, np.float64)
    b = np.zeros(kern.shape[0]) if bias is None else np.asarray(bias, np.float64)
    z = mean @ kern.T
    e = gamma(c + 1) * (np.abs(mean) @ np.abs(kern.T)) + (e_mean * SLACK) @ np.abs(kern.T)
    pre = z + b
    e_pre = e * SLACK + U * np.abs(pre)
    if softmax_out:
        ref, bound = softmax_rows(pre, e_pre)
    else:
        ref = act64(pre, act, alpha)
        bound = act_bound(pre, e_pre, ref, act, alpha) * SLACK
    bound = bound + store_bound(ref, half_out)
    return ref.reshape(n, 1, 1, -1), bound.reshape(n, 1, 1, -1)


def softmax_rows(z, e_z):
    """Max-subtracted soft-max over the last axis, fp32 (softmax_kernel, gap_dense_kernel): expf at 2 ulp, a sum of C terms, one
    division. An error e of the inputs moves p by at most 2 max(e) p; the rest is (2 + 1 + C + 1) u-units relative to p, doubled for
    the ulp/u ratio of expf."""
    z = np.asarray(z, np.float64)
    m = z.max(axis=-1, keepdims=True)
    ex = np.exp(z - m)
    p = ex / ex.sum(axis=-1, keepdims=True)
    c = z.shape[-1]
    emax = np.max(np.broadcast_to(e_z, z.shape), axis=-1, keepdims=True)
    bound = p * (2 * emax * SLACK + (2 * ACT_ULPS + gamma(c) / U + 2) * U)
    return p, bound


def softmax(x, half_out=False):
    ref, bound = softmax_rows(x, 0.0)
    return ref, bound + store_bound(ref, half_out)


def depthwise(x, w_chw, bias, bn, stride, pad_x, pad_y, out_hw, act="", alpha=0.0, half_out=False, at=None):
    """Depthwise k x k on the fp32 folded weights (depthwise kernels: fp32 FMAs started from the bias, window clipped to the input)."""
    n, h, w, c = np.shape(x)
    wk = np.asarray(w_chw, np.float32)
    k = wk.shape[-1]
    wv, shift = fold(wk[:, None], bias, bn)
    wv = wv[:, 0].astype(np.float64)
    oh, ow = out_hw
    s = int(stride)
    ni, oy, ox = pixels(at, n, oh, ow)
    acc = np.zeros((len(ni), c))
    aab = np.zeros((len(ni), c))
    for ky in range(k):
        for kx in range(k):
            X = gather(x, ni, oy * s + ky - pad_y, ox * s + kx - pad_x)
            acc += X * wv[:, ky, kx]
            aab += np.abs(X * wv[:, ky, kx])
    pre = acc + shift
    e_pre = gamma(k * k) * (aab + np.abs(shift))
    ref = act64(pre, act, alpha)
    bound = act_bound(pre, e_pre, ref, act, alpha) * SLACK + store_bound(ref, half_out)
    return shaped(ref, at, n, oh, ow), shaped(bound, at, n, oh, ow)


def box_grid(n, oh, ow, box):
    """The boxes of a (tw, th, tn) tile grid laid over [n, oh, ow] from pixel (0, 0) of image 0, boxes past the edges clipped:
    (n0, y0, x0, nn, hy, wx) arrays, one entry per box, in the kernels' tile order (x fastest, then y, then images)."""
    tw, th, tn = box
    bn, by, bx = np.indices((-(-n // tn), -(-oh // th), -(-ow // tw))).reshape(3, -1)
    n0, y0, x0 = bn * tn, by * th, bx * tw
    return n0, y0, x0, np.minimum(tn, n - n0), np.minimum(th, oh - y0), np.minimum(tw, ow - x0)


def sample_pixels(n, oh, ow, boxes, seed, per_box=2):
    """Output pixels to restate for one layer: every pixel of the first and last row and column of each image, and per_box seeded
    random pixels in every box of each (tw, th, tn) grid in `boxes` (all of a box's pixels when it has fewer). The same (n, oh,
    ow, boxes, seed) give the same pixels. Returns (n_idx, oy_idx, ox_idx) in NHWC order, without repeats."""
    rng = np.random.default_rng(seed)
    lin = []
    for i in range(n):
        rows = np.concatenate([np.zeros(ow, np.int64), np.full(ow, oh - 1), np.arange(oh), np.arange(oh)])
        cols = np.concatenate([np.arange(ow), np.arange(ow), np.zeros(oh, np.int64), np.full(oh, ow - 1)])
        lin.append((i * oh + rows) * ow + cols)
    for box in boxes:
        n0, y0, x0, nn, hy, wx = box_grid(n, oh, ow, box)
        cnt = nn * hy * wx
        keys = rng.random((len(cnt), int(cnt.max())))
        keys[np.arange(keys.shape[1])[None, :] >= cnt[:, None]] = np.inf  # positions past a clipped box's pixels never win
        q = np.argsort(keys, axis=1)[:, :per_box]
        keep = np.arange(q.shape[1])[None, :] < np.minimum(cnt, per_box)[:, None]
        q, b = q[keep], np.nonzero(keep)[0]
        lin.append(((n0[b] + q // (wx[b] * hy[b])) * oh + y0[b] + (q // wx[b]) % hy[b]) * ow + x0[b] + q % wx[b])
    u = np.unique(np.concatenate(lin))
    return u // (oh * ow), (u // ow) % oh, u % ow


def elementwise_operand(x, at):
    """The operand of an elementwise layer as float64: whole, or [len(at), C] at the pixels `at`."""
    if at is None:
        return np.asarray(x, np.float64)
    ni, oy, ox = pixels(at, 0, 0, 0)
    return np.asarray(x[ni, oy, ox], np.float64)


def add(a, b, act="", alpha=0.0, half_out=False, at=None):
    pre = elementwise_operand(a, at) + elementwise_operand(b, at)
    ref = act64(pre, act, alpha)
    return ref, act_bound(pre, U * np.abs(pre), ref, act, alpha) * SLACK + store_bound(ref, half_out)


def batchnorm(x, bn, act="", alpha=0.0, half_out=False, at=None):
    """chanwise_kernel: scale * (x - mean) + beta with scale = gamma / max(sqrt(var + 1e-3), 1e-4) in fp32 (pack.cpp); three roundings."""
    g, be, m, v = (np.asarray(bn[k], np.float32) for k in ("gamma", "beta", "mean", "var"))
    scale = (g / np.maximum(np.sqrt(v + np.float32(0.001)), np.float32(0.0001))).astype(np.float64)
    x = elementwise_operand(x, at)
    d = x - m
    pre = scale * d + be
    e_pre = U * np.abs(d) * np.abs(scale) * 2 + U * np.abs(pre)
    ref = act64(pre, act, alpha)
    return ref, act_bound(pre, e_pre * SLACK, ref, act, alpha) * SLACK + store_bound(ref, half_out)


def activation(x, act, alpha=0.0, half_out=False, at=None):
    pre = elementwise_operand(x, at)
    ref = act64(pre, act, alpha)
    return ref, act_bound(pre, 0.0, ref, act, alpha) * SLACK + store_bound(ref, half_out)


def maxpool(x, k, stride, out_hw, at=None):
    """Windows start inside the input and are clipped at the bottom / right edge. A maximum is one of the stored inputs: bit-identical."""
    n, h, w, c = np.shape(x)
    oh, ow = out_hw
    ni, oy, ox = pixels(at, n, oh, ow)
    y = np.full((len(ni), c), -np.inf, np.float32)
    for ky in range(k):
        for kx in range(k):
            ys, xs = oy * stride + ky, ox * stride + kx
            inside = (ys < h) & (xs < w)
            blk = gather(x, ni, np.where(inside, ys, 0), np.where(inside, xs, 0), dtype=np.float32)
            blk[~inside] = -np.inf
            y = np.maximum(y, blk)
    return shaped(y.astype(np.float64), at, n, oh, ow), shaped(np.zeros(y.shape), at, n, oh, ow)


def avgpool(x, k, stride, out_hw, half_out=False, at=None):
    """Clipped windows averaged over the pixels inside the input (fp32 sum of at most k*k terms, one division)."""
    n, h, w, c = np.shape(x)
    oh, ow = out_hw
    ni, oy, ox = pixels(at, n, oh, ow)
    s = np.zeros((len(ni), c))
    a = np.zeros((len(ni), c))
    cnt = np.zeros((len(ni), 1))
    for ky in range(k):
        for kx in range(k):
            ys, xs = oy * stride + ky, ox * stride + kx
            inside = (ys < h) & (xs < w)
            sub = gather(x, ni[inside], ys[inside], xs[inside])
            s[inside] += sub
            a[inside] += np.abs(sub)
            cnt[inside] += 1
    ref = s / cnt
    bound = (gamma(k * k + 1) * a / cnt) * SLACK + store_bound(ref, half_out)
    return shaped(ref, at, n, oh, ow), shaped(bound, at, n, oh, ow)


def pad(x, pad_x, pad_y, out_hw, mode="constant", at=None):
    """pad_kernel: input column x lands at x + pad_x, row y at y + pad_y (the layer's (T, L) offsets, as the kernel is handed them)."""
    n = np.shape(x)[0]
    ni, oy, ox = pixels(at, n, *out_hw)
    y = gather(x, ni, oy - pad_y, ox - pad_x, mode)
    return shaped(y, at, n, *out_hw), shaped(np.zeros(y.shape), at, n, *out_hw)


def concat(a, b, at=None):
    y = np.concatenate([elementwise_operand(a, at), elementwise_operand(b, at)], axis=-1)
    return y, np.zeros(y.shape)


def flatten(x):
    x = np.asarray(x, np.float32)
    y = x.reshape(x.shape[0], 1, 1, -1)
    return y.astype(np.float64), np.zeros(y.shape)


def upsample_nearest(x, out_hw, at=None, scale=None):
    """Nearest upsampling (upsample_kernel): output column o reads input column floor(fl(o * fl(1 / scale))), the fp32 product of o
    and the fp32 reciprocal of the layer's fp32 scale, clamped to the input (rows alike). That is the index the engine promises: it is
    the reference's shader arithmetic (a float multiply by the inverse scale, then floor). At the integer scales it is floor(o / scale)
    (the reciprocals of 2 and 4 are exact; fl(1/3) rounds up, and o * fl(1/3) never drops below an integer it should reach). At other
    scales neither floor(o / scale) of the decimal scale nor that of its fp32 value is promised: at 1.7, fl(1/1.7) rounds down and
    o = 17 reads column 9, not 10; at 1.2 the kernel agrees with the decimal scale but not with fp32(1.2) = 1.20000005 (o = 6 reads
    column 5). scale None: out_hw / the input size (an integer scale)."""
    n, h, w, c = np.shape(x)
    oh, ow = out_hw
    ni, oy, ox = pixels(at, n, oh, ow)
    inv = np.float32(1) / np.float32(oh / h if scale is None else scale)
    iy = np.clip(np.floor(oy.astype(np.float32) * inv).astype(np.int64), 0, h - 1)
    ix = np.clip(np.floor(ox.astype(np.float32) * inv).astype(np.int64), 0, w - 1)
    y = gather(x, ni, iy, ix)
    return shaped(y, at, n, oh, ow), shaped(np.zeros(y.shape), at, n, oh, ow)


def bilinear_coord(o, size, scale):
    """(X, e): the exact source coordinate (o + 0.5) / scale - 0.5 of output coordinates o clamped to [0, size - 1], and a bound of
    the error of upsample_kernel's fp32 coordinate: inv = fl(1 / scale) errs by u / scale, offs = fl(0.5 - 0.5 inv) by
    0.5 u / scale + u |offs|, o inv by o u / scale before its rounding (u o inv, unless contracted into the subtraction), and the
    subtraction rounds once more (u |X|). Clamping does not increase the error."""
    s = float(np.float32(scale))
    offs = 0.5 - 0.5 / s
    o = np.asarray(o, np.float64)
    X = o / s - offs
    e = U * (2 * o / s + 0.5 / s + abs(offs) + np.abs(X)) * SLACK
    return np.clip(X, 0, size - 1), e


def upsample_bilinear(x, scale, out_hw, half_out=False, at=None):
    """Bilinear upsampling (upsample_kernel, the reference's vk_upsampling2d_bilinear): output (oy, ox) is the bilinear interpolation
    of the input at the exact source coordinate ((oy, ox) + 0.5) / scale - 0.5, each coordinate clamped to [0, size - 1], from the
    taps (floor, floor + 1) of each coordinate; a tap outside the input reads 0 (it only occurs at size - 1, with weight 0).
    The kernel evaluates the interpolant at its fp32 coordinate (bilinear_coord: error e_x, e_y). The interpolant is continuous and
    piecewise bilinear, so that moves the value by at most e_x times the largest difference of horizontal neighbours in the rows and
    the cells the coordinate may fall in (columns floor(X) - 1 .. floor(X) + 2, rows floor(Y) - 1 .. floor(Y) + 2), plus e_y likewise.
    Each weight is a product of two fp32 differences (x12 - sx is exact for sx >= 0.5, else one rounding): 3 u relative. The four
    taps are accumulated from 0 in fp32 (separate or fused multiply-adds): gamma_4 sum w |t|. Then the store."""
    n, h, w, c = np.shape(x)
    oh, ow = out_hw
    ni, oy, ox = pixels(at, n, oh, ow)
    X, ex = bilinear_coord(ox, w, scale)
    Y, ey = bilinear_coord(oy, h, scale)
    x0, y0 = np.floor(X).astype(np.int64), np.floor(Y).astype(np.int64)
    fx, fy = (X - x0)[:, None], (Y - y0)[:, None]

    def t(yy, xx):  # outside the input: 0
        return gather(x, ni, yy, xx)

    t11, t21, t22, t12 = t(y0, x0), t(y0, x0 + 1), t(y0 + 1, x0 + 1), t(y0 + 1, x0)
    w11, w21, w22, w12 = (1 - fx) * (1 - fy), fx * (1 - fy), fx * fy, (1 - fx) * fy
    ref = w11 * t11 + w21 * t21 + w22 * t22 + w12 * t12
    mag = w11 * np.abs(t11) + w21 * np.abs(t21) + w22 * np.abs(t22) + w12 * np.abs(t12)
    dx = np.zeros((len(ni), c))
    dy = np.zeros((len(ni), c))
    for r in range(-1, 3):
        for q in range(-1, 3):
            v = t(y0 + r, x0 + q)
            dx = np.maximum(dx, np.abs(t(y0 + r, x0 + q + 1) - v))
            dy = np.maximum(dy, np.abs(t(y0 + r + 1, x0 + q) - v))
    bound = (ex[:, None] * dx + ey[:, None] * dy + (3 * U + gamma(4)) * mag) * SLACK + store_bound(ref, half_out)
    return shaped(ref, at, n, oh, ow), shaped(bound, at, n, oh, ow)


def subpixel(x, r, half_out=False, at=None):
    """Depth-to-space of r*r channels into one, through tanh as the reference's subpixel shader does: output (y r + i, x r + j) =
    tanhf(input (y, x, i r + j))."""
    n, h, w, c = np.shape(x)
    ni, oy, ox = pixels(at, n, h * r, w * r)
    v = np.asarray(x[ni, oy // r, ox // r, (oy % r) * r + ox % r], np.float64)[:, None]
    ref = np.tanh(v)
    bound = act_bound(v, 0.0, ref, "tanh", 0.0) * SLACK + store_bound(ref, half_out)
    return shaped(ref, at, n, h * r, w * r), shaped(bound, at, n, h * r, w * r)


def model_input(x, half, at=None):
    """The input upload (split_f32_kernel, and the stem's feed copy): fp32 -> hi + lo, or fp16 alone. Restated exactly."""
    y = stored(elementwise_operand(np.asarray(x, np.float32), at), half)
    return y.astype(np.float64), np.zeros(y.shape)


def resize_coord(o, out, src, centre):
    """(P, e) of output texels o along an axis of `out` texels sampling `src`: P the exact source position (o + 0.5) src / out, less
    0.5 for the texel-centre convention of the linear filter (centre=True); e a bound of the error of resize_pos's fp32 position
    fl(fl((o + 0.5) / out) * src) (- 0.5): the division and the product round once each (u P each), and the subtraction rounds
    once unless the compiler contracted it with the product into an FMA (u |P - 0.5|)."""
    o = np.asarray(o, np.float64)
    p = (2 * o + 1) * src / (2.0 * out)
    if not centre:
        return p, U * 2 * p * SLACK
    return p - 0.5, U * (2 * p + np.abs(p - 0.5)) * SLACK


def resize_u8(images_u8, out_hw, mean4, norm4, linear, half):
    """ImageTexture::resize (core/inc/snn/imageTexture.h:137, the sampler of shadertemplate_vk_resize.comp) of 8-bit NHWC images to
    out_hw, then (v - mean[c & 3]) * norm[c & 3] and the store: the model input of resize_u8_kernel and frame_input_kernel (and of
    split_u8_kernel / device_input_kernel<u8> at equal size, where every position is a texel centre). Stated from the definition,
    not from the kernels' order of operations. Returns (ref, bound) [n, oh, ow, c].

    Linear: output texel o samples the source at the exact position X = (o + 0.5) src / out - 0.5 in texel-centre units, the
    bilinear interpolant of the texels clamped to the edge (continuous and piecewise bilinear). The kernel evaluates it at its fp32
    position (resize_coord: error e_x, e_y), which moves the value by at most e_x times the largest difference of horizontal
    neighbours in the rows and cells the position may fall in (columns floor(X) - 1 .. floor(X) + 2, rows floor(Y) - 1 .. floor(Y) + 2,
    clamped), plus e_y likewise: the same argument as upsample_bilinear. The weights ax = sx - floor(sx) are exact. The blend
    (two lerps along x, one along y, separate or fused multiply-adds; the tap differences of integers are exact) rounds by at most
    7 u max|tap|: 2 u M for each of top and bottom, carried through the final lerp with weights (1 - ay) and ay, plus 2 u M for its
    difference and product and u M for its sum.

    Nearest: texel floor(P), P = (o + 0.5) src / out, clamped to src - 1; no blend. Where P lies within the fp32 position's error of
    an integer k, the kernel may take k - 1 or k: ref is then the midpoint of the candidate taps' values and bound half their
    spread (nearest_candidates gives the candidates themselves, for a check that the value is one of them); everywhere else the tap
    is unique and the value must be bit-identical to its normalised fp32 value (the subtraction and the product are two roundings,
    restated exactly in float32) and its store.

    Normalisation (linear): (v - mean) * norm rounds twice, u |v - mean| |norm| + u |ref|, on top of |norm| times v's error. Then
    store_bound (nothing saturates: the values stay far inside fp16's range for 8-bit inputs and sane constants)."""
    img = np.asarray(images_u8, np.uint8)
    n, sh, sw, c = img.shape
    oh, ow = out_hw
    mean = np.array([np.float32(mean4[i & 3]) for i in range(c)], np.float32)
    norm = np.array([np.float32(norm4[i & 3]) for i in range(c)], np.float32)
    if not linear:
        vals = nearest_candidates(img, out_hw, mean, norm, half)
        lo, hi = np.minimum.reduce(vals), np.maximum.reduce(vals)
        return (lo + hi) / 2, (hi - lo) / 2
    X, ex = resize_coord(np.arange(ow), ow, sw, centre=True)
    Y, ey = resize_coord(np.arange(oh), oh, sh, centre=True)
    xf, yf = np.floor(X).astype(np.int64), np.floor(Y).astype(np.int64)
    ax, ay = (X - xf)[None, None, :, None], (Y - yf)[None, :, None, None]

    def tap(dy, dx):
        return img[:, np.clip(yf + dy, 0, sh - 1)][:, :, np.clip(xf + dx, 0, sw - 1)].astype(np.float64)
    p00, p01, p10, p11 = tap(0, 0), tap(0, 1), tap(1, 0), tap(1, 1)
    v = (1 - ay) * ((1 - ax) * p00 + ax * p01) + ay * ((1 - ax) * p10 + ax * p11)
    dx = np.zeros(v.shape)
    dy = np.zeros(v.shape)
    for r in range(-1, 3):
        for q in range(-1, 3):
            t = tap(r, q)
            dx = np.maximum(dx, np.abs(tap(r, q + 1) - t))
            dy = np.maximum(dy, np.abs(tap(r + 1, q) - t))
    mag = np.maximum.reduce([np.abs(p00), np.abs(p01), np.abs(p10), np.abs(p11)])
    e_v = (ex[None, None, :, None] * dx + ey[None, :, None, None] * dy + 7 * U * mag) * SLACK
    d = v - mean.astype(np.float64)
    ref = d * norm.astype(np.float64)
    bound = (np.abs(norm) * (e_v + U * np.abs(d)) + U * np.abs(ref)) * SLACK + store_bound(ref, half)
    return ref, bound


def nearest_candidates(images_u8, out_hw, mean, norm, half):
    """The values the nearest filter may take at each output texel (resize_u8): the normalised, stored value of texel floor(P) along
    each axis, or of k - 1 and k where P lies within the fp32 position's error of an integer k. Four arrays [n, oh, ow, c] (equal
    where the tap is unique); a nearest kernel's output must equal one of them bit for bit. mean, norm: per channel, fp32."""
    img = np.asarray(images_u8, np.uint8)
    n, sh, sw, c = img.shape

    def taps(out, src):
        p, e = resize_coord(np.arange(out), out, src, centre=False)
        k = np.floor(p + 0.5)
        lo = np.minimum(np.floor(p), src - 1)
        near = (np.abs(p - k) <= e) & (k >= 1)
        return np.where(near, np.minimum(k, src - 1), lo).astype(np.int64), np.where(near, np.minimum(k - 1, src - 1), lo).astype(np.int64)
    ys, xs = taps(out_hw[0], sh), taps(out_hw[1], sw)
    mean, norm = np.asarray(mean, np.float32), np.asarray(norm, np.float32)
    return [stored((img[:, yy][:, :, xx].astype(np.float32) - mean) * norm, half).astype(np.float64) for yy in ys for xx in xs]


def quant_u8(v, scale, offset):
    """quant_u8 (kernels_simt.cu: every 8-bit output) of stored values v: clamp(rint(v scale + offset), 0, 255), stated in float64 from
    the fp32 operands, rint rounding half to even as rintf does. The kernel forms v scale + offset in fp32 (two roundings, or one where
    the compiler contracts them into an FMA): within e = u (|v scale| + |t|) of the exact t, and exact where v scale and t are fp32
    numbers. Where t lies within e of a half-integer, the byte may be either neighbour: ref is then the midpoint of the two candidate
    bytes and bound 1/2; everywhere else bound = 0 and the byte must match. NaN gives 0: rintf(NaN) is NaN, fmaxf(NaN, 0) = 0.
    Returns (ref, bound) as float64 arrays of v's shape."""
    v = np.asarray(v, np.float32).astype(np.float64)
    s, o = float(np.float32(scale)), float(np.float32(offset))
    with np.errstate(invalid="ignore", over="ignore"):
        prod = v * s  # exact in float64: two 24-bit significands
        t = prod + o
        exact_fp32 = (np.float32(prod).astype(np.float64) == prod) & (np.float32(t).astype(np.float64) == t)
        e = np.where(exact_fp32, 0.0, U * (np.abs(prod) + np.abs(t)) * SLACK)
        k = np.floor(t)
        near = (np.abs(t - (k + 0.5)) <= e) & (e > 0)  # either neighbour of the half-integer k + 0.5
        b0 = np.clip(np.where(near, k, np.rint(t)), 0, 255)
        b1 = np.clip(np.where(near, k + 1, np.rint(t)), 0, 255)
    nan = np.isnan(v)
    b0, b1 = np.where(nan, 0.0, b0), np.where(nan, 0.0, b1)
    return (b0 + b1) / 2, (b1 - b0) / 2


def argmax(x):
    """std::max_element's index over the last axis (the reference's classes, core.cpp:230-232), per image: x[..., C] -> int64 [...].
    max_element keeps the running maximum and moves on only when it compares below a later score, so: index 0 when score 0 is NaN
    (nothing compares above a NaN) and when no score is a number; otherwise the first maximum of the scores that are numbers (a later
    NaN never compares above the running maximum). Returns (ref, bound) with bound 0: the index must match."""
    x = np.asarray(x, np.float64)
    x = x.reshape(-1, x.shape[-1]) if x.ndim > 1 else x[None]
    num = np.where(np.isnan(x), -np.inf, x)
    idx = np.argmax(num, axis=-1)  # the first maximum; a row of -inf and NaN only gives 0
    idx = np.where(np.isnan(x[:, 0]), 0, idx)
    return idx, np.zeros(idx.shape)


def check(got, ref, bound, what):
    """Returns (worst |err| / bound, number of violations); bit-identical layers (bound 0) count any difference, and a NaN or
    infinity where the reference is finite is always a violation."""
    err = np.abs(np.asarray(got, np.float64) - ref)
    bad = int(np.count_nonzero(~(err <= bound)))
    err = np.where(np.isnan(err), np.inf, err)
    ratio = float(np.max(np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0)))) if err.size else 0.0
    return ratio, bad


def instancenorm(x, gamma_c, beta_c, act="", alpha=0.0, half_out=False, at=None, eps=1e-5):
    """InstanceNorm (instnorm_*_kernel): per (image, channel) mean and biased variance over H W of d = x - x[first pixel], summed in
    fp32 (sum d with adds, sum d^2 with FMAs, any order: gamma_{HW+2}); m = S1 / HW, var = max(S2 / HW - m^2, 0), mean = x0 + m,
    rstd = 1 / sqrtf(var + 1e-5) (correctly rounded sqrt and division), y = (x - mean) * (gamma rstd) + beta, then the activation.
    ref evaluates the same formula in float64 with the exact mean and variance. The bound follows each rounding: e_m of m,
    e_var of the variance, e_r of rstd by the mean value theorem on (v + eps)^-1/2 over [v + eps - e_var, v + eps], then the
    elementwise part. The statistics always cover the whole plane; at only chooses the output pixels evaluated. eps: the kernels' is
    1e-5 (another value states a different layer, for the converter's checks)."""
    n, h, w, c = np.shape(x)
    hw = h * w
    g = np.asarray(gamma_c, np.float32).astype(np.float64)
    b = np.asarray(beta_c, np.float32).astype(np.float64)
    x0 = np.asarray(x[:, 0, 0], np.float64)
    s1, s2, sa = np.zeros((n, c)), np.zeros((n, c)), np.zeros((n, c))
    for i in range(n):  # one image at a time: a 720 x 720 plane in float64 is large enough
        d = np.asarray(x[i], np.float64).reshape(hw, c) - x0[i]
        s1[i], s2[i], sa[i] = d.sum(axis=0), (d * d).sum(axis=0), np.abs(d).sum(axis=0)
    m = s1 / hw
    mu = x0 + m
    var = s2 / hw - m * m
    e_s1 = gamma(hw + 1) * sa
    e_s2 = gamma(hw + 3) * s2
    e_m = e_s1 / hw + U * np.abs(m)
    e_mean = e_m + U * np.abs(mu)
    e_var = (e_s2 / hw + U * s2 / hw) + 2 * np.abs(m) * e_m + e_m * e_m + U * m * m + U * (np.abs(var) + 1e-30)
    v = var + eps
    r = 1.0 / np.sqrt(v)
    r_lo = 1.0 / np.sqrt(np.maximum(v - e_var * SLACK, 1e-30))
    e_r = 0.5 * r_lo ** 3 * e_var * SLACK + 2.5 * U * r_lo + U * eps * 0.5 * r_lo ** 3
    mul = g * r
    e_mul = np.abs(g) * e_r + U * np.abs(mul) * SLACK
    ni, oy, ox = pixels(at, n, h, w)
    xm = np.asarray(x[ni, oy, ox], np.float64) - mu[ni]
    e_xm = e_mean[ni] + U * (np.abs(xm) + e_mean[ni])
    pre = xm * mul[ni] + b
    e_pre = (np.abs(xm) * e_mul[ni] + np.abs(mul[ni]) * e_xm + U * np.abs(xm * mul[ni]) + U * np.abs(pre)) * SLACK
    ref = act64(pre, act, alpha)
    bound = act_bound(pre, e_pre, ref, act, alpha) * SLACK + store_bound(ref, half_out)
    return shaped(ref, at, n, h, w), shaped(bound, at, n, h, w)


# ---- YOLO decode, score order and NMS (yolo_select / yolo_rank / yolo_nms kernels; layers.cpp decodeCell, iou, nms) ------------
# Two statements of the same decode. yolo_contract is the float32 arithmetic the kernels promise (kernels_simt.cu, snnb.h): every
# + - * / one IEEE-rounded fp32 operation in the host's order, no FMA, exp = (float) exp((double) x), > against 0.35f and 0.45f,
# std::max / std::min as written, keys ordered by (score bits, -scan). The device must match it bit for bit. yolo_define is the
# mathematical decode in float64 with a bound on every value, from first-order propagation of u = 2^-24 per operation and one fp32
# ulp per exp (so glibc's expf on the host path is covered too); yolo_decisions uses it to check the contract's threshold, order and
# suppression decisions wherever the float64 margin exceeds the bound, and never decides one inside it.
YOLO_SCALE = (32, 16)
YOLO_ANCHORS = (10, 14, 23, 27, 37, 58, 81, 82, 135, 169, 344, 319)
YOLO_MASKS = (3, 4, 5, 1, 2, 3)
YOLO_CONF, YOLO_IOU = np.float32(0.35), np.float32(0.45)
FLT_MAX = np.float32(3.402823466e+38)
F32_OVERFLOW = (2.0 - 2.0 ** -24) * 2.0 ** 127  # the smallest real that rounds to +inf in fp32
EXP_REL, EXP_ABS = 2.0 ** -23, 2.0 ** -149     # one fp32 ulp of an exp: relative, and at fp32's subnormals


def yolo_cells(h0, h1, pitch=(None, None)):
    """The six values of every (cell, anchor) of two heads [N, gh, gw, C], C >= 18, in the kernels' scan order (head, gy, gx, gc).
    pitch: the channel pitch each head is read with (default its C). Returns a dict of d [N, S, 6] float32 and, per scan index, yi,
    gx, gy, gc, gw, gh (int64 [S])."""
    d, meta = [], {k: [] for k in ("yi", "gx", "gy", "gc", "gw", "gh")}
    for yi, h in enumerate((h0, h1)):
        h = np.asarray(h, np.float32)
        n, gh, gw, c = h.shape
        p = pitch[yi] or c
        cell = np.repeat(np.arange(gh * gw), 3)
        gc = np.tile(np.arange(3), gh * gw)
        flat = h.reshape(n, -1)
        d.append(flat[:, (cell * p + gc * 6)[:, None] + np.arange(6)])
        for k, v in (("yi", np.full(cell.size, yi)), ("gx", cell % gw), ("gy", cell // gw), ("gc", gc), ("gw", np.full(cell.size, gw)),
                     ("gh", np.full(cell.size, gh))):
            meta[k].append(v)
    out = {k: np.concatenate(v).astype(np.int64) for k, v in meta.items()}
    out["d"] = np.concatenate(d, axis=1)
    return out


def exp_cr(x):
    """(float) exp((double) x) of fp32 values, and a flag where exp(x) lies within 4 double ulps of an fp32 rounding midpoint: there
    numpy's float64 exp does not decide the correctly rounded result, so either neighbour is right."""
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        y = np.exp(np.asarray(x, np.float32).astype(np.float64))
        r = y.astype(np.float32)
        up, dn = np.nextafter(r, np.float32(np.inf)), np.nextafter(r, np.float32(0))
        r64 = r.astype(np.float64)
        gap = np.minimum(np.abs(y - (r64 + up.astype(np.float64)) / 2), np.where(dn != r, np.abs(y - (r64 + dn.astype(np.float64)) / 2), np.inf))
        near = np.isfinite(r) & np.isfinite(up) & (gap <= 4 * np.spacing(np.abs(y)))
    return r, near


def yolo_score32(d4, d5, exp=exp_cr):
    """prob = 1.f / ((1.f + exp(-d4) * (1.f + exp(-maxLogit)))) in fp32, maxLogit = d5 > -3.402823466e+38f ? d5 : -3.402823466e+38f.
    Returns (score, near flag of exp(-d4), near flag of exp(-maxLogit))."""
    f = np.float32
    d4, d5 = np.asarray(d4, f), np.asarray(d5, f)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        ml = np.where(d5 > -FLT_MAX, d5, -FLT_MAX)
        e4, n4 = exp(-d4)
        e5, n5 = exp(-ml)
        return (f(1) / (f(1) + e4 * (f(1) + e5))).astype(f), n4, n5


def yolo_decode32(c, exp=exp_cr):
    """decodeCell in fp32 for every cell of yolo_cells(...) c: returns cls [N, S] int64, score [N, S], box [N, S, 4] = (x, y, w, h)
    float32 (evaluated everywhere; meaningful where score > 0.35f) and near [N, S], the exp_cr flag over the exps the cell evaluates."""
    f = np.float32
    d = c["d"]
    score, n4, n5 = yolo_score32(d[..., 4], d[..., 5], exp)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        a = np.array(YOLO_ANCHORS, f)[np.array(YOLO_MASKS)[c["gc"] + 3 * c["yi"]][:, None] * 2 + np.arange(2)]
        net = (np.array(YOLO_SCALE)[c["yi"]][:, None] * np.stack([c["gw"], c["gh"]], 1)).astype(f)
        g = np.stack([c["gx"], c["gy"]], 1).astype(f)
        s0, n0 = exp(-d[..., 0:2])
        cxy = (g + f(1) / (f(1) + s0)) / np.stack([c["gw"], c["gh"]], 1).astype(f)
        e2, n2 = exp(d[..., 2:4])
        wh = e2 * a / net
        box = np.concatenate([cxy - wh / f(2), wh], axis=-1).astype(f)
    passed = score > YOLO_CONF
    near = n4 | n5 | (passed & (n0.any(-1) | n2.any(-1)))
    return np.zeros(score.shape, np.int64), score.astype(f), box, near


def yolo_iou32(a, b):
    """iou (layers.cpp) of boxes a and b [..., 4], broadcast, in fp32: std::max(p, q) = p < q ? q : p, std::min(p, q) = q < p ? q : p."""
    ax, ay, aw, ah = (a[..., k] for k in range(4))
    bx, by, bw, bh = (b[..., k] for k in range(4))
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        ix0, iy0 = np.where(ax < bx, bx, ax), np.where(ay < by, by, ay)
        ax1, bx1, ay1, by1 = ax + aw, bx + bw, ay + ah, by + bh
        ix1, iy1 = np.where(bx1 < ax1, bx1, ax1), np.where(by1 < ay1, by1, ay1)
        r = ((ix1 - ix0) * (iy1 - iy0)) / ((aw * ah + bw * bh) - (ix1 - ix0) * (iy1 - iy0))
    return np.where((ix1 < ix0) | (iy1 < iy0), np.float32(0), r).astype(np.float32)


def yolo_nms32(box, cls, max_rows):
    """Greedy NMS of a score-ordered list (yolo_greedy_nms, nms): a box is kept unless a kept box before it of the same class has
    IoU > 0.45 with it, up to max_rows kept boxes. Returns the kept positions."""
    alive = np.ones(len(box), bool)
    kept, i = [], 0
    while len(kept) < max_rows:
        nxt = np.flatnonzero(alive[i:])
        if not nxt.size:
            break
        i += int(nxt[0])
        kept.append(i)
        alive[i + 1:] &= ~((yolo_iou32(box[i], box[i + 1:]) > YOLO_IOU) & (cls[i + 1:] == cls[i]))
        i += 1
    return np.array(kept, np.int64)


def yolo_contract(h0, h1, max_rows=100):
    """The device decode of two heads [N, gh, gw, C] (C >= 18, any two grids): netW = 32 gw, netH = 32 gh on head 0 and 16 gw, 16 gh
    on head 1. Returns (rows [N, max_rows, 6] float32 {class, score, x, y, w, h} zero past the count, counts [N], near [N, S] (an exp of
    the cell within reach of an fp32 midpoint: exp_cr), paths): paths[n] = {"order": the passing scan indices stable-sorted by
    descending score, "kept": the kept positions in that order}, for yolo_decisions."""
    c = yolo_cells(h0, h1)
    cls, score, box, near = yolo_decode32(c)
    n = score.shape[0]
    rows, counts, paths = np.zeros((n, max_rows, 6), np.float32), np.zeros(n, np.int64), []
    for i in range(n):
        p = np.flatnonzero(score[i] > YOLO_CONF)
        o = p[np.argsort(-score[i, p], kind="stable")]
        kept = yolo_nms32(box[i, o], cls[i, o], max_rows)
        k = o[kept]
        rows[i, :len(k), 0], rows[i, :len(k), 1], rows[i, :len(k), 2:] = cls[i, k], score[i, k], box[i, k]
        counts[i] = len(k)
        paths.append({"order": o, "kept": kept})
    return rows, counts, near, paths


def _f32_range(v, e):
    """A float64 value v +- e as fp32 makes it: past fp32's range it rounds to +-inf, exactly when the whole interval lies past it,
    unbounded when it straddles the edge. Non-finite values are exact (what they came from was); a NaN bound is unbounded. Finite
    values gain 2^-150, the absolute error of an operation rounded into fp32's subnormals (u |v| only holds above them)."""
    a = np.abs(v)
    with np.errstate(invalid="ignore"):
        over = (a == np.inf) | (a - e >= F32_OVERFLOW)
        strad = ~over & (a + e >= F32_OVERFLOW)
    v = np.where(over, np.copysign(np.inf, v), v)
    e = np.where(np.isfinite(v), np.where(strad | np.isnan(e), np.inf, e + 2.0 ** -150), 0.0)
    return v, e


def yolo_define(h0, h1):
    """The YOLO decode in float64 for every cell of two heads: score = 1 / (1 + e^-d4 (1 + e^-d5)) (the reference's parenthesisation,
    d5 the max logit as the kernels take it: NaN gives -FLT_MAX), x = (gx + sigma(d0)) / gw - w / 2, y likewise, w = e^d2 bw / netW,
    h = e^d3 bh / netH. Returns dict of [N, S] float64 arrays score, x, y, w, h, their bounds e_score ... e_h, and the operands
    (d4, maxLogit) that decide the score. A bound covers any fp32 evaluation that rounds each operation once (u = 2^-24 |result|) and
    takes each exp within one fp32 ulp (EXP_REL |y| + EXP_ABS), to first order (SLACK); x and y carry absolute bounds, as cx - w / 2
    can cancel. Values past fp32's range are +-inf (_f32_range)."""
    c = yolo_cells(h0, h1)
    d = c["d"].astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        def ex(x):
            y = np.exp(x)
            return _f32_range(y, EXP_REL * y + EXP_ABS)

        def add1(v, e):
            return _f32_range(1.0 + v, e + U * (1.0 + v))

        def recip(v, e):
            r = 1.0 / v
            return _f32_range(r, e / (v * v) + U * np.abs(r))

        ml = np.where(d[..., 5] > -float(FLT_MAX), d[..., 5], -float(FLT_MAX))
        e4, ee4 = ex(-d[..., 4])
        p, ep = add1(*ex(-ml))
        q, eq = _f32_range(e4 * p, e4 * ep + p * ee4 + U * e4 * p)
        score, e_score = recip(*add1(q, eq))
        out = {"score": score, "e_score": e_score * SLACK, "d4": c["d"][..., 4], "maxlogit": ml}
        for k, (dv, g, gs) in enumerate(((d[..., 0], c["gx"], c["gw"]), (d[..., 1], c["gy"], c["gh"]))):
            sig, esig = recip(*add1(*ex(-dv)))
            b, eb = _f32_range(g + sig, esig + U * np.abs(g + sig))
            cen, ecen = _f32_range(b / gs, eb / gs + U * np.abs(b / gs))
            anchor = np.array(YOLO_ANCHORS, np.float64)[np.array(YOLO_MASKS)[c["gc"] + 3 * c["yi"]] * 2 + k]
            net = np.array(YOLO_SCALE)[c["yi"]] * gs
            t, et = ex(d[..., 2 + k])
            m, em = _f32_range(t * anchor, et * anchor + U * t * anchor)
            wv, ew = _f32_range(m / net, em / net + U * m / net)
            xv, exv = _f32_range(cen - wv / 2, ecen + ew / 2 + U * np.abs(cen - wv / 2))
            out["xy"[k]], out["e_" + "xy"[k]] = xv, exv * SLACK
            out["wh"[k]], out["e_" + "wh"[k]] = wv, ew * SLACK
    return out


def yolo_iou64(a, ea, b, eb):
    """iou of float64 boxes a, b [..., 4] (x, y, w, h) with per-coordinate bounds ea, eb, taking std::max / std::min as written (so a
    NaN or infinity selects as it does in fp32). Returns (iou, bound): the bound covers the boxes anywhere within their bounds and the
    fp32 evaluation's roundings; max and min move by at most the larger of their operands' errors. ref takes a negative overlap as
    empty (inter 0); the bound on inter uses the overlaps' magnitudes, so it also covers an fp32 evaluation that finds a small positive
    overlap where the float64 one is empty, or the reverse. Where an overlap is certainly negative, both return 0 and the bound is 0."""
    ax, ay, aw, ah = (a[..., k] for k in range(4))
    bx, by, bw, bh = (b[..., k] for k in range(4))
    eax, eay, eaw, eah = (ea[..., k] for k in range(4))
    ebx, eby, ebw, ebh = (eb[..., k] for k in range(4))
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        def side(p0, e0, ps, es, q0, f0, qs, fs):
            lo = np.where(p0 < q0, q0, p0)
            e_lo = np.maximum(e0, f0)
            p1, q1 = p0 + ps, q0 + qs
            e_p1, e_q1 = e0 + es + U * np.abs(p1), f0 + fs + U * np.abs(q1)
            hi = np.where(q1 < p1, q1, p1)
            e_hi = np.maximum(e_p1, e_q1)
            s = hi - lo
            return s, e_hi + e_lo + U * np.abs(s)

        iw, e_iw = side(ax, eax, aw, eaw, bx, ebx, bw, ebw)
        ih, e_ih = side(ay, eay, ah, eah, by, eby, bh, ebh)
        zero = (iw < 0) | (ih < 0)
        inter = np.where(zero, 0.0, iw * ih)
        e_inter = np.abs(iw) * e_ih + np.abs(ih) * e_iw + e_iw * e_ih + U * inter
        A, B = aw * ah, bw * bh
        eA, eB = aw * eah + ah * eaw + U * A, bw * ebh + bh * ebw + U * B
        den = A + B - inter
        e_den = eA + eB + U * np.abs(A + B) + e_inter + U * np.abs(den)
        iou = inter / den
        e = e_inter / np.abs(den) + np.abs(inter) * e_den / (den * den) + U * np.abs(iou)
        e = np.where(np.isfinite(iou), np.where(np.isnan(e), np.inf, e), 0.0)
        e = np.where((iw < -e_iw) | (ih < -e_ih), 0.0, e)  # fp32 takes the same empty branch
    return np.where(zero, 0.0, iou), e * SLACK


def yolo_decisions(h0, h1, paths, max_rows, defn=None, contract=None):
    """Every decision on the contract's path (yolo_contract's paths), classified against yolo_define: certain where the float64 margin
    exceeds its bound, inside-bound otherwise. Decisions: the threshold of every cell (a NaN score is a certain rejection), the order
    of each adjacent pair of the sorted list (two cells with the same d4 and max logit tie in any evaluation: a certain tie, broken by
    the scan) and every IoU test of a kept box against a later candidate up to where the walk stops. Returns one dict per image:
    certain / inside counts per kind, wrong (certain decisions the contract made the other way, as (kind, detail)) and first_uncertain:
    the first row whose presence or place may depend on an inside-bound decision (the count when none does)."""
    defn = yolo_define(h0, h1) if defn is None else defn
    cls, score32, box32, _ = yolo_decode32(yolo_cells(h0, h1)) if contract is None else contract
    box64 = np.stack([defn[k] for k in "xywh"], -1)
    ebox = np.stack([defn["e_" + k] for k in "xywh"], -1)
    res = []
    for n, path in enumerate(paths):
        o, kept = path["order"], path["kept"]
        r = {"certain": {"threshold": 0, "order": 0, "suppress": 0}, "inside": {"threshold": 0, "order": 0, "suppress": 0}, "wrong": []}
        kept_before = np.concatenate([[0], np.cumsum(np.isin(np.arange(len(o)), kept))])  # kept rows before sorted position p
        first = len(kept)
        s64, es = defn["score"][n], defn["e_score"][n]
        passed = score32[n] > YOLO_CONF
        margin = s64 - float(YOLO_CONF)
        nan = np.isnan(s64)
        sure = nan | (np.abs(margin) > es)
        r["certain"]["threshold"], r["inside"]["threshold"] = int(sure.sum()), int((~sure).sum())
        bad = sure & (passed != (margin > es))
        r["wrong"] += [("threshold", int(s)) for s in np.flatnonzero(bad)]
        if (~sure).any():  # where an undecided cell would sort: after every passing score above its bound
            so = score32[n, o].astype(np.float64)
            for s in np.flatnonzero(~sure):
                first = min(first, int(kept_before[int(np.sum(so > s64[s] + es[s]))]))
        if len(o) > 1:
            a, b = o[:-1], o[1:]
            m = s64[a] - s64[b]
            tie = (defn["d4"][n, a] == defn["d4"][n, b]) & (defn["maxlogit"][n, a] == defn["maxlogit"][n, b])
            sure = tie | (np.abs(m) > es[a] + es[b])
            r["certain"]["order"], r["inside"]["order"] = int(sure.sum()), int((~sure).sum())
            # no certain inversion between any two positions: s64[j] - e[j] <= min over i < j of s64[i] + e[i]
            lo = np.minimum.accumulate(s64[o] + es[o])[:-1]
            inv = (s64[b] - es[b] > lo) | (tie & (b < a)) | (sure & ~tie & (m < 0))
            r["wrong"] += [("order", int(p)) for p in np.flatnonzero(inv)]
            if (~sure).any():
                first = min(first, int(kept_before[int(np.flatnonzero(~sure)[0])]))
        stop = int(kept[-1]) + 1 if len(kept) == max_rows else len(o)
        for k in kept:
            j = np.arange(k + 1, stop)
            j = j[cls[n, o[j]] == cls[n, o[k]]]
            if not j.size:
                continue
            iou, e = yolo_iou64(box64[n, o[k]], ebox[n, o[k]], box64[n, o[j]], ebox[n, o[j]])
            got = yolo_iou32(box32[n, o[k]], box32[n, o[j]]) > YOLO_IOU
            m = iou - float(YOLO_IOU)
            sure = np.isnan(iou) | (np.abs(m) > e)
            r["certain"]["suppress"] += int(sure.sum())
            r["inside"]["suppress"] += int((~sure).sum())
            r["wrong"] += [("suppress", (int(k), int(q))) for q in j[sure & (got != (m > e))]]
            if (~sure).any():
                first = min(first, int(kept_before[int(j[~sure][0])]))
        r["first_uncertain"] = first
        res.append(r)
    return res
