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


def instancenorm(x, gamma_c, beta_c, act="", alpha=0.0, half_out=False, at=None):
    """InstanceNorm (instnorm_*_kernel): per (image, channel) mean and biased variance over H W of d = x - x[first pixel], summed in
    fp32 (sum d with adds, sum d^2 with FMAs, any order: gamma_{HW+2}); m = S1 / HW, var = max(S2 / HW - m^2, 0), mean = x0 + m,
    rstd = 1 / sqrtf(var + 1e-5) (correctly rounded sqrt and division), y = (x - mean) * (gamma rstd) + beta, then the activation.
    ref evaluates the same formula in float64 with the exact mean and variance. The bound follows each rounding: e_m of m,
    e_var of the variance, e_r of rstd by the mean value theorem on (v + eps)^-1/2 over [v + eps - e_var, v + eps], then the
    elementwise part. The statistics always cover the whole plane; at only chooses the output pixels evaluated."""
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
    v = var + 1e-5
    r = 1.0 / np.sqrt(v)
    r_lo = 1.0 / np.sqrt(np.maximum(v - e_var * SLACK, 1e-30))
    e_r = 0.5 * r_lo ** 3 * e_var * SLACK + 2.5 * U * r_lo + U * 1e-5 * 0.5 * r_lo ** 3
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
