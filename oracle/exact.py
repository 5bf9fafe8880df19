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
"""
import numpy as np

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


def stored(v, half):
    """What the storage makes of fp32 values v: hi + lo (split-fp16) or fp16 alone, as float32. Saturation at +-65504 is not
    modelled; callers keep their values inside fp16's range."""
    v = np.asarray(v, np.float32)
    hi = v.astype(np.float16).astype(np.float32)
    if half:
        return hi
    return hi + (v - hi).astype(np.float16).astype(np.float32)


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


def pad_input(x, pad_top, pad_left, need_h, need_w, mode="constant"):
    """x [n, h, w, c] -> [n, need_h, need_w, c] with x at (pad_top, pad_left): zeros, or the kernels' replicate / single reflection
    (src_coord in kernels_simt.cu; a coordinate still outside after one reflection reads zero)."""
    n, h, w, c = x.shape
    ys = np.arange(need_h) - pad_top
    xs = np.arange(need_w) - pad_left

    def src(s, size):
        if mode == "replicate":
            return np.clip(s, 0, size - 1)
        if mode == "reflect":
            s = np.where(s < 0, -s, s)
            s = np.where(s >= size, 2 * size - 2 - s, s)
        return np.where((s >= 0) & (s < size), s, -1)

    sy, sx = src(ys, h), src(xs, w)
    out = x[:, np.clip(sy, 0, h - 1)][:, :, np.clip(sx, 0, w - 1)].copy()
    out[:, sy < 0] = 0
    out[:, :, sx < 0] = 0
    return out


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
           half_out=False, pad_mode="constant"):
    """Conv2D as the engine runs it: output column ox reads input column ox * stride + kx - pad_x, row oy * stride + ky - pad_y
    (the kernels' (pad_x, pad_y) = the layer's (T, L) offsets). kernel: "igemm" (conv_umma_kernel), "rowwin" / "feed"
    (conv_rowwin_kernel, regular or feed mode) or "simt". Returns (ref, bound) [n, oh, ow, oc]."""
    x = np.asarray(x, np.float64)
    n, h, w, ic = x.shape
    wv, shift = fold(w_oihw, bias, bn)
    oc, _, k, _ = wv.shape
    oh, ow = out_hw
    s = int(stride)
    T = TERMS.get(form, 0)
    wq, wlo = weight_operand(wv, form)
    xp = pad_input(x, pad_y, pad_x, (oh - 1) * s + k, (ow - 1) * s + k, pad_mode)
    M = n * oh * ow
    taps = {}
    for ky in range(k):
        for kx in range(k):
            X = xp[:, ky:ky + (oh - 1) * s + 1:s, kx:kx + (ow - 1) * s + 1:s, :].reshape(M, ic)
            taps[ky, kx] = (X, np.abs(X), wq[:, :, ky, kx].T)
    y = np.zeros((M, oc))
    e_acc = np.zeros((M, oc))
    if kernel == "simt":
        a_all = np.zeros((M, oc))
        for X, aX, W in taps.values():
            y += X @ W
            a_all += aX @ np.abs(W)
        e_acc = gamma(k * k * ic) * a_all
    else:
        blocks_abs = np.zeros((M, oc))
        blocks = k_blocks(kernel, k, s, pad_x, ic)
        for block in blocks:
            c = np.zeros((M, oc))
            for step in block:
                A = np.zeros((M, oc))
                P = np.zeros((M, oc))
                for ky, kx, ch in step:
                    X, aX, W = taps[ky, kx]
                    A += aX[:, ch] @ np.abs(W[ch])
                    P += X[:, ch] @ W[ch]
                e_acc += T * STEP_SLACK * KAPPA * (np.abs(c) + A)
                c += P
            y += c
            blocks_abs += np.abs(c)
        e_acc += max(len(blocks) - 1, 0) * U * blocks_abs
    if wlo is not None:
        for (ky, kx), (X, aX, W) in taps.items():
            e_acc += (aX * (2.0 ** -11 * SLACK) + 2.0 ** -25) @ wlo[:, :, ky, kx].T
    pre = y + shift.astype(np.float64)
    e_pre = e_acc * SLACK + U * np.abs(pre)
    if residual is not None:
        pre = pre + np.asarray(residual, np.float64).reshape(M, oc)
        e_pre += U * np.abs(pre)
    ref = act64(pre, act, alpha)
    bound = act_bound(pre, e_pre, ref, act, alpha) * SLACK + store_bound(ref, half_out)
    return ref.reshape(n, oh, ow, oc), bound.reshape(n, oh, ow, oc)


def dense(x, kernel_out_in, bias, act="", form="fp32x3", half_out=False):
    """Dense on a 1 x 1 map (or flattened HWC): a 1x1 conv_umma_kernel launch."""
    n = x.shape[0]
    x1 = np.asarray(x, np.float64).reshape(n, 1, 1, -1)
    kern = np.asarray(kernel_out_in, np.float32)
    return conv2d(x1, kern[:, :, None, None], bias, None, 1, 0, 0, (1, 1), act, 0.0, form=form, half_out=half_out)


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


def depthwise(x, w_chw, bias, bn, stride, pad_x, pad_y, out_hw, act="", alpha=0.0, half_out=False):
    """Depthwise k x k on the fp32 folded weights (depthwise kernels: fp32 FMAs started from the bias, window clipped to the input)."""
    x = np.asarray(x, np.float64)
    n, h, w, c = x.shape
    wk = np.asarray(w_chw, np.float32)
    k = wk.shape[-1]
    wv, shift = fold(wk[:, None], bias, bn)
    wv = wv[:, 0].astype(np.float64)
    oh, ow = out_hw
    s = int(stride)
    xp = pad_input(x, pad_y, pad_x, (oh - 1) * s + k, (ow - 1) * s + k)
    acc = np.zeros((n, oh, ow, c))
    aab = np.zeros((n, oh, ow, c))
    for ky in range(k):
        for kx in range(k):
            X = xp[:, ky:ky + (oh - 1) * s + 1:s, kx:kx + (ow - 1) * s + 1:s, :]
            acc += X * wv[:, ky, kx]
            aab += np.abs(X * wv[:, ky, kx])
    pre = acc + shift
    e_pre = gamma(k * k) * (aab + np.abs(shift))
    ref = act64(pre, act, alpha)
    return ref, act_bound(pre, e_pre, ref, act, alpha) * SLACK + store_bound(ref, half_out)


def add(a, b, act="", alpha=0.0, half_out=False):
    pre = np.asarray(a, np.float64) + np.asarray(b, np.float64)
    ref = act64(pre, act, alpha)
    return ref, act_bound(pre, U * np.abs(pre), ref, act, alpha) * SLACK + store_bound(ref, half_out)


def batchnorm(x, bn, act="", alpha=0.0, half_out=False):
    """chanwise_kernel: scale * (x - mean) + beta with scale = gamma / max(sqrt(var + 1e-3), 1e-4) in fp32 (pack.cpp); three roundings."""
    g, be, m, v = (np.asarray(bn[k], np.float32) for k in ("gamma", "beta", "mean", "var"))
    scale = (g / np.maximum(np.sqrt(v + np.float32(0.001)), np.float32(0.0001))).astype(np.float64)
    x = np.asarray(x, np.float64)
    d = x - m
    pre = scale * d + be
    e_pre = U * np.abs(d) * np.abs(scale) * 2 + U * np.abs(pre)
    ref = act64(pre, act, alpha)
    return ref, act_bound(pre, e_pre * SLACK, ref, act, alpha) * SLACK + store_bound(ref, half_out)


def activation(x, act, alpha=0.0, half_out=False):
    pre = np.asarray(x, np.float64)
    ref = act64(pre, act, alpha)
    return ref, act_bound(pre, 0.0, ref, act, alpha) * SLACK + store_bound(ref, half_out)


def maxpool(x, k, stride, out_hw):
    """Windows start inside the input and are clipped at the bottom / right edge. A maximum is one of the stored inputs: bit-identical."""
    x = np.asarray(x, np.float32)
    n, h, w, c = x.shape
    oh, ow = out_hw
    y = np.full((n, oh, ow, c), -np.inf, np.float32)
    for ky in range(k):
        for kx in range(k):
            ys = np.arange(oh) * stride + ky
            xs = np.arange(ow) * stride + kx
            iy, ix = np.nonzero(ys < h)[0], np.nonzero(xs < w)[0]
            blk = np.full((n, oh, ow, c), -np.inf, np.float32)
            blk[:, iy[:, None], ix[None, :]] = x[:, ys[iy]][:, :, xs[ix]]
            y = np.maximum(y, blk)
    return y.astype(np.float64), np.zeros(y.shape)


def avgpool(x, k, stride, out_hw, half_out=False):
    """Clipped windows averaged over the pixels inside the input (fp32 sum of at most k*k terms, one division)."""
    x = np.asarray(x, np.float64)
    n, h, w, c = x.shape
    oh, ow = out_hw
    s = np.zeros((n, oh, ow, c))
    a = np.zeros((n, oh, ow, c))
    cnt = np.zeros((oh, ow))
    for ky in range(k):
        for kx in range(k):
            ys = np.arange(oh) * stride + ky
            xs = np.arange(ow) * stride + kx
            vy, vx = ys < h, xs < w
            sub = x[:, ys[vy]][:, :, xs[vx]]
            idx_y, idx_x = np.nonzero(vy)[0], np.nonzero(vx)[0]
            s[:, idx_y[:, None], idx_x[None, :]] += sub
            a[:, idx_y[:, None], idx_x[None, :]] += np.abs(sub)
            cnt[idx_y[:, None], idx_x[None, :]] += 1
    ref = s / cnt[None, :, :, None]
    bound = (gamma(k * k + 1) * a / cnt[None, :, :, None]) * SLACK + store_bound(ref, half_out)
    return ref, bound


def pad(x, pad_x, pad_y, out_hw, mode="constant"):
    """pad_kernel: input column x lands at x + pad_x, row y at y + pad_y (the layer's (T, L) offsets, as the kernel is handed them)."""
    y = pad_input(np.asarray(x, np.float32), pad_y, pad_x, out_hw[0], out_hw[1], mode)
    return y.astype(np.float64), np.zeros(y.shape)


def concat(a, b):
    y = np.concatenate([np.asarray(a, np.float32), np.asarray(b, np.float32)], axis=-1)
    return y.astype(np.float64), np.zeros(y.shape)


def flatten(x):
    x = np.asarray(x, np.float32)
    y = x.reshape(x.shape[0], 1, 1, -1)
    return y.astype(np.float64), np.zeros(y.shape)


def upsample_nearest(x, out_hw):
    """Nearest upsampling: output (y, x) reads input (floor(y h / oh), floor(x w / ow)) - for the integer scales of the zoo, y // s."""
    x = np.asarray(x, np.float32)
    n, h, w, c = x.shape
    oh, ow = out_hw
    ys = (np.arange(oh) * h) // oh
    xs = (np.arange(ow) * w) // ow
    y = x[:, ys][:, :, xs]
    return y.astype(np.float64), np.zeros(y.shape)


def subpixel(x, r, half_out=False):
    """Depth-to-space of r*r channels into one, through tanh as the reference's subpixel shader does: output (y r + i, x r + j) =
    tanhf(input (y, x, i r + j))."""
    x = np.asarray(x, np.float64)
    n, h, w, c = x.shape
    v = x.reshape(n, h, w, r, r).transpose(0, 1, 3, 2, 4).reshape(n, h * r, w * r, 1)
    ref = np.tanh(v)
    return ref, act_bound(v, 0.0, ref, "tanh", 0.0) * SLACK + store_bound(ref, half_out)


def model_input(x, half):
    """The input upload (split_f32_kernel, and the stem's feed copy): fp32 -> hi + lo, or fp16 alone. Restated exactly."""
    y = stored(np.asarray(x, np.float32), half)
    return y.astype(np.float64), np.zeros(y.shape)


def check(got, ref, bound, what):
    """Returns (worst |err| / bound, number of violations); bit-identical layers (bound 0) count any difference, and a NaN or
    infinity where the reference is finite is always a violation."""
    err = np.abs(np.asarray(got, np.float64) - ref)
    bad = int(np.count_nonzero(~(err <= bound)))
    err = np.where(np.isnan(err), np.inf, err)
    ratio = float(np.max(np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0)))) if err.size else 0.0
    return ratio, bad


def instancenorm(x, gamma_c, beta_c, act="", alpha=0.0, half_out=False):
    """InstanceNorm (instnorm_*_kernel): per (image, channel) mean and biased variance over H W of d = x - x[first pixel], summed in
    fp32 (sum d with adds, sum d^2 with FMAs, any order: gamma_{HW+2}); m = S1 / HW, var = max(S2 / HW - m^2, 0), mean = x0 + m,
    rstd = 1 / sqrtf(var + 1e-5) (correctly rounded sqrt and division), y = (x - mean) * (gamma rstd) + beta, then the activation.
    ref evaluates the same formula in float64 with the exact mean and variance. The bound follows each rounding: e_m of m,
    e_var of the variance, e_r of rstd by the mean value theorem on (v + eps)^-1/2 over [v + eps - e_var, v + eps], then the
    elementwise part."""
    x = np.asarray(x, np.float64)
    n, h, w, c = x.shape
    hw = h * w
    g = np.asarray(gamma_c, np.float32).astype(np.float64)
    b = np.asarray(beta_c, np.float32).astype(np.float64)
    xs = x.reshape(n, hw, c)
    d = xs - xs[:, :1]
    s1, s2 = d.sum(axis=1), (d * d).sum(axis=1)
    m = s1 / hw
    mu = xs[:, :1, :][:, 0] + m
    var = s2 / hw - m * m
    e_s1 = gamma(hw + 1) * np.abs(d).sum(axis=1)
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
    xm = xs - mu[:, None, :]
    e_xm = e_mean[:, None, :] + U * (np.abs(xm) + e_mean[:, None, :])
    pre = xm * mul[:, None, :] + b
    e_pre = (np.abs(xm) * e_mul[:, None, :] + np.abs(mul[:, None, :]) * e_xm + U * np.abs(xm * mul[:, None, :]) + U * np.abs(pre)) * SLACK
    ref = act64(pre, act, alpha)
    bound = act_bound(pre, e_pre, ref, act, alpha) * SLACK + store_bound(ref, half_out)
    return ref.reshape(n, h, w, c), bound.reshape(n, h, w, c)
