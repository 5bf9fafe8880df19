"""snnb_model_transform_luma without a GPU: the entry point is exported and refuses null arguments, and the numpy restatement of its
output frames (oracle/luma.py), which the GPU tests hold the kernel to, gives the values worked out by hand below (dyadic weights, so
every float32 step is exact)."""
import ctypes as C

import numpy as np

from oracle import luma, oracle, yuv
from shadernn_b200 import _lib


def test_transform_luma_is_exported_and_refuses_null_arguments(built):
    lib = _lib.lib()
    assert "snnb_model_transform_luma" in _lib.SIGNATURES
    f, o = _lib.Frames(), _lib.FramesOut()
    assert lib.snnb_model_transform_luma(None, None, None, None) != 0
    assert b"snnb_model_transform_luma: null model" in lib.snnb_last_error()
    assert lib.snnb_model_transform_luma(None, C.byref(f), C.byref(o), None) != 0
    assert b"snnb_model_transform_luma: null model" in lib.snnb_last_error()


def plane(rows):
    return np.array(rows, np.uint8)[None]


def test_equal_chroma_size_is_a_copy():
    rng = np.random.default_rng(1)
    u, v = rng.integers(0, 256, (2, 2, 9, 17), dtype=np.uint8)
    for linear in (True, False):
        uo, vo = luma.resize_chroma(u, v, (17, 33), linear)  # 17 x 33 frames: chroma 9 x 17, the source's
        assert np.array_equal(uo, u) and np.array_equal(vo, v)
        uo, vo = luma.resize_chroma(u, v, (18, 34), linear)  # even sizes with the same chroma size
        assert np.array_equal(uo, u) and np.array_equal(vo, v)


def test_one_chroma_sample_resized_to_any_size_is_constant():
    u, v = plane([[77]]), plane([[200]])
    for hw in [(1, 1), (2, 2), (3, 5), (64, 31), (1080, 1920)]:
        for linear in (True, False):
            uo, vo = luma.resize_chroma(u, v, hw, linear)
            assert uo.shape == (1,) + yuv.chroma_shape(*hw)
            assert (uo == 77).all() and (vo == 200).all()


def test_nearest_2x_duplicates_samples():
    p = plane([[1, 2, 3], [4, 5, 6]])
    want = np.repeat(np.repeat(p, 2, axis=1), 2, axis=2)
    assert np.array_equal(luma.resize_plane(p, (4, 6), linear=False), want)
    uo, vo = luma.resize_chroma(p, 255 - p, (8, 12), linear=False)  # frames 4 x 6 -> 8 x 12: chroma 2 x 3 -> 4 x 6
    assert np.array_equal(uo, want) and np.array_equal(vo, 255 - want)


def test_linear_2x_of_a_2x2_ramp():
    # source x = (ox + 0.5) / 4 * 2 - 0.5 = -0.25, 0.25, 0.75, 1.25: taps (0, 0), (0, 1), (0, 1), (1, 1), weights 0.75, 0.25, 0.75,
    # 0.25 (the first and last clamp to one texel); the same along y. Rows: 0, 25, 75, 100 and 200, 213.75, 241.25, 255.
    p = plane([[0, 100], [200, 255]])
    want_f = np.array([[0.0, 25.0, 75.0, 100.0],
                       [50.0, 72.1875, 116.5625, 138.75],
                       [150.0, 166.5625, 199.6875, 216.25],
                       [200.0, 213.75, 241.25, 255.0]], np.float32)
    got_f = oracle.resize_normalize(p[..., None], (4, 4), [0.0] * 4, [1.0] * 4, linear=True)[0, :, :, 0]
    assert got_f.dtype == np.float32 and np.array_equal(got_f, want_f)
    want = np.array([[0, 25, 75, 100], [50, 72, 117, 139], [150, 167, 200, 216], [200, 214, 241, 255]], np.uint8)
    assert np.array_equal(luma.resize_plane(p, (4, 4), linear=True)[0], want)
    uo, vo = luma.resize_chroma(p, p, (8, 8), linear=True)
    assert np.array_equal(uo[0], want) and np.array_equal(vo[0], want)


def test_odd_sizes_on_both_sides():
    # frames 4 x 4 -> 1 x 1 (chroma 2 x 2 -> 1 x 1): source position 1.0 - 0.5 = 0.5 on both axes; linear: top = 10 + 0.5 * 10 = 15,
    # bottom = 30 + 0.5 * 11 = 35.5, 15 + 0.5 * 20.5 = 25.25 -> 25; nearest: the texel at (1, 1)
    u = plane([[10, 20], [30, 41]])
    assert luma.resize_chroma(u, u, (1, 1), True)[0].tolist() == [[[25]]]
    assert luma.resize_chroma(u, u, (1, 1), False)[0].tolist() == [[[41]]]
    # frames 33 x 17 -> 66 x 34: chroma 17 x 9 -> 33 x 17; the corners clamp onto the source's corners, nearest takes source samples
    rng = np.random.default_rng(7)
    u = rng.integers(0, 256, (2, 17, 9), dtype=np.uint8)
    for linear in (True, False):
        uo, _ = luma.resize_chroma(u, u, (66, 34), linear)
        assert uo.shape == (2, 33, 17)
        assert np.array_equal(uo[:, 0, 0], u[:, 0, 0]) and np.array_equal(uo[:, -1, -1], u[:, -1, -1])
    near, _ = luma.resize_chroma(u, u, (66, 34), False)
    assert np.array_equal(near[:, ::2, ::2], u)  # output sample 2k samples source k: (2k + 0.5) * 17 / 33 and (2k + 0.5) * 9 / 17 floor to k


def test_whole_frames_keep_the_source_chroma_and_change_its_packing():
    rng = np.random.default_rng(3)
    m = rng.integers(0, 256, (2, 6, 10), dtype=np.uint8)
    u, v = rng.integers(0, 256, (2, 2, 3, 5), dtype=np.uint8)
    y, c1, c2 = luma.luma_frames("nv12", m, u, v, (6, 10))
    assert np.array_equal(y, m) and c2 is None
    assert np.array_equal(c1[..., 0::2], u) and np.array_equal(c1[..., 1::2], v)
    y, c1, c2 = luma.luma_frames("i420", m[..., None], u, v, (6, 10))
    assert np.array_equal(y, m) and np.array_equal(c1, u) and np.array_equal(c2, v)
    _, c1, _ = luma.luma_frames("nv21", m, u, v, (6, 10))
    assert np.array_equal(luma.chroma("nv21", c1)[0], u) and np.array_equal(luma.chroma("nv21", c1)[1], v)
    y, c1, _ = luma.luma_frames("nv12", m, u, v, (12, 20), linear=False)
    assert np.array_equal(y, np.repeat(np.repeat(m, 2, axis=1), 2, axis=2))
    assert np.array_equal(c1[..., 0::2], np.repeat(np.repeat(u, 2, axis=1), 2, axis=2))
