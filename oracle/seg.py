"""TEST INFRASTRUCTURE - numpy restatement of the label plane snnb_model_segment_frames writes: the fp32 scores of output 0 resampled
to the plane with ImageTexture::resize's taps (those of oracle.resize_normalize, applied to float scores rather than to bytes, with
every float32 + - * rounded on its own), then the arg-max over the channels or, for one channel, the threshold.
tests/test_segment_cpu.py holds it to hand-worked cases; the GPU tests hold every label byte to it."""
import numpy as np

f32 = np.float32


def taps(out_n, src_n, linear=True):
    """The taps along one axis of an out_n-sample resize of src_n samples: (i0, i1, a), a the float32 weight of i1. Output sample o is
    sampled at (o + 0.5) / out_n * src_n; linear: texel centres at i + 0.5, clamp to edge; nearest: floor (i0 == i1, a == 0)."""
    f = (np.arange(out_n, dtype=f32) + f32(0.5)) / f32(out_n) * f32(src_n)
    if not linear:
        i0 = np.minimum(f.astype(np.int64), src_n - 1)
        return i0, i0, np.zeros(out_n, f32)
    s = f - f32(0.5)
    s0 = np.floor(s)
    a = (s - s0).astype(f32)
    i0 = np.clip(s0.astype(np.int64), 0, src_n - 1)
    i1 = np.clip(s0.astype(np.int64) + 1, 0, src_n - 1)
    return i0, i1, a


def scores(t, out_hw, linear=True):
    """Scores [N, H, W, C] float32 of model output t [N, h, w, C] on an H x W label plane: t itself at equal size, else the taps of
    taps(); linear blends top = p00 + ax (p01 - p00), bot = p10 + ax (p11 - p10), top + ay (bot - top)."""
    t = np.asarray(t, f32)
    _, h, w, _ = t.shape
    oh, ow = out_hw
    if (oh, ow) == (h, w):
        return t.copy()
    x0, x1, ax = taps(ow, w, linear)
    y0, y1, ay = taps(oh, h, linear)
    p00 = t[:, y0][:, :, x0]
    if not linear:
        return p00
    p01, p10, p11 = t[:, y0][:, :, x1], t[:, y1][:, :, x0], t[:, y1][:, :, x1]
    ax_, ay_ = ax[None, None, :, None], ay[None, :, None, None]
    top = p00 + ax_ * (p01 - p00)
    bot = p10 + ax_ * (p11 - p10)
    return (top + ay_ * (bot - top)).astype(f32)


def labels(s, threshold=0.5):
    """uint8 labels [N, H, W] of scores s [N, H, W, C]. C >= 2: the smallest c whose score equals the maximum of the scores that are not
    NaN, 0 where every score is NaN. C == 1: 1 where s >= threshold (float32), else 0; NaN gives 0."""
    s = np.asarray(s, f32)
    if s.shape[-1] == 1:
        with np.errstate(invalid="ignore"):
            return (s[..., 0] >= f32(threshold)).astype(np.uint8)
    nan = np.isnan(s)
    m = np.where(nan, f32(-np.inf), s).max(-1, keepdims=True)
    hit = (s == m) & ~nan
    lab = np.argmax(hit, -1)
    lab[~hit.any(-1)] = 0
    return lab.astype(np.uint8)


def segment(t, out_hw, linear=True, threshold=0.5):
    """The label planes [N, H, W] uint8 of model output t [N, h, w, C] (the F32 output of run_frames)."""
    return labels(scores(t, out_hw, linear), threshold)
