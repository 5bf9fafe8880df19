"""TEST INFRASTRUCTURE - numpy restatement of the output side of snnb_model_transform_luma: M, the model-size 8-bit output, resized into
the Y plane, and the source frames' U and V planes each resized plane to plane, from ceil(W/2) x ceil(H/2) to ceil(Wo/2) x ceil(Ho/2),
both with ImageTexture::resize's taps and float32 blend (yuv_out.resize_rgba8 on one channel). tests/test_luma_cpu.py holds it to
hand-worked cases; the GPU tests then use it to make the frames the device must write."""
import numpy as np

from oracle import yuv, yuv_out


def resize_plane(p, out_hw, linear=True):
    """ImageTexture::resize of 8-bit planes [N, h, w] to out_hw: a copy at equal size, else the taps and float32 blend of
    oracle.resize_normalize, then rint."""
    return yuv_out.resize_rgba8(np.asarray(p, np.uint8)[..., None], out_hw, linear)[..., 0]


def chroma(fmt, c1, c2=None):
    """U and V [..., ceil(H/2), ceil(W/2)] from the chroma planes of `fmt` as yuv.planes_from_yuv lays them out."""
    if fmt == "i420":
        return np.asarray(c1), np.asarray(c2)
    if fmt not in ("nv12", "nv21"):
        raise ValueError("no chroma planes in frame format %r" % (fmt,))
    c = np.asarray(c1)
    first, second = c[..., 0::2], c[..., 1::2]
    return (first, second) if fmt == "nv12" else (second, first)


def resize_chroma(u, v, out_hw, linear=True):
    """The source chroma planes U, V [N, ch, cw] resized for frames of out_hw (H, W): each to ceil(H/2) x ceil(W/2)."""
    cshape = yuv.chroma_shape(*out_hw)
    return resize_plane(u, cshape, linear), resize_plane(v, cshape, linear)


def luma_frames(fmt, mu8, u, v, out_hw, linear=True):
    """The planes (y, c1, c2) of `fmt` that transform_luma writes from M [N, h, w] (or [N, h, w, 1]) and the source chroma U, V
    [N, ch, cw]: Y = M resized to out_hw, U and V resized plane to plane."""
    m = np.asarray(mu8, np.uint8)
    if m.ndim == 4:
        m = m[..., 0]
    y = resize_plane(m, out_hw, linear)
    uo, vo = resize_chroma(u, v, out_hw, linear)
    return yuv.planes_from_yuv(fmt, y, uo, vo)
