"""CPU tests of detection on regions: the C-ABI of snnb_model_detect_rois / detect_rois_list and snnb_tile_rois, the tile grid,
tests/_region_merge.py's merge_region_rows on hand-built cases with known answers, and the merge kernels' resource usage."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import _region_merge as region_merge
from shadernn_b200 import _lib, core
from shadernn_b200._lib import SnnbError

MERGE_KERNELS = ("roi_merge_gather_kernel", "roi_merge_rank_kernel", "roi_merge_nms_kernel")


def test_exports_and_roi_layout():
    lib = _lib.lib()
    for name in ("snnb_model_detect_rois", "snnb_model_detect_rois_list", "snnb_tile_rois"):
        assert hasattr(lib, name)
    a = np.zeros((2, 6), np.int32)  # snnb_roi is six ints: the int32 [k, 6] arrays of the Python layer
    assert a.strides == (24, 4)


def test_null_model_refused():
    lib = _lib.lib()
    rc = lib.snnb_model_detect_rois(None, None, 1, None, None, None, 100, None, None)
    assert rc != 0 and b"null model" in lib.snnb_last_error()
    rc = lib.snnb_model_detect_rois_list(None, None, None, None, None, 100, None, None)
    assert rc != 0 and b"null model" in lib.snnb_last_error()


def _count(nx_size, t, ov):
    return 1 if t >= nx_size else 1 + -(-(nx_size - t) // (t - ov))


@pytest.mark.parametrize("frame_hw,tile_hw,ov", [((2160, 3840), (960, 960), 96), ((1080, 1920), (640, 640), 0), ((301, 437), (100, 77), 13),
                                                 ((100, 50), (960, 960), 10), ((7, 5), (2, 3), 1), ((1, 1), (1, 1), 0), ((640, 640), (640, 320), 319)])
def test_tiles_cover_every_pixel_with_the_minimum_overlap(frame_hw, tile_hw, ov):
    H, W = frame_hw
    t = core.tile_rois(frame_hw, tile_hw, ov, frame=3)
    tw, th = min(tile_hw[1], W), min(tile_hw[0], H)
    nx, ny = _count(W, tw, ov), _count(H, th, ov)
    assert t.dtype == np.int32 and t.shape == (nx * ny, 6)
    assert (t[:, 0] == 3).all() and (t[:, 1] == np.arange(nx * ny)).all() and (t[:, 4] == tw).all() and (t[:, 5] == th).all()
    xs, ys = t[:nx, 2], t[::nx, 3]
    for j in range(ny):  # row-major: row j holds the columns in order
        assert (t[j * nx:(j + 1) * nx, 2] == xs).all() and (t[j * nx:(j + 1) * nx, 3] == ys[j]).all()
    for starts, size, tile, n in ((xs, W, tw, nx), (ys, H, th, ny)):
        assert starts[0] == 0 and starts[-1] + tile == size
        assert (starts == [i * (size - tile) // max(n - 1, 1) for i in range(n)]).all()
        if n > 1:
            assert (starts[:-1] + tile - starts[1:] >= ov).all()  # neighbours overlap by at least ov
    cover = np.zeros((H, W), np.int32)
    for _, _, x, y, w, h in t:
        cover[y:y + h, x:x + w] += 1
    assert (cover >= 1).all()


def test_tile_flagship_grid():
    t = core.tile_rois((2160, 3840), (960, 960), 96)
    assert len(t) == 15 and sorted(set(t[:, 2])) == [0, 720, 1440, 2160, 2880] and sorted(set(t[:, 3])) == [0, 600, 1200]


def test_tile_refusals():
    lib = _lib.lib()
    out = np.full((4, 6), 77, np.int32)
    count = C.c_int(-1)

    def tile(*a, cap=4, rois=out.ctypes.data_as(_lib.vp)):
        count.value = -1
        rc = lib.snnb_tile_rois(*a, rois, cap, C.byref(count))
        return rc, lib.snnb_last_error().decode()
    for args, text in (((0, 100, 100, 0, 10, 0), "tile size 0 x 10"), ((0, 100, 100, 10, -1, 0), "tile size 10 x -1"),
                       ((0, 100, 100, 10, 10, -1), "min_overlap -1"), ((0, 100, 100, 10, 10, 10), "min_overlap 10"),
                       ((0, 100, 8, 10, 10, 8), "min_overlap 8"), ((0, 0, 100, 10, 10, 0), "frame size 0 x 100")):
        rc, msg = tile(*args)
        assert rc != 0 and text in msg, (args, msg)
        assert count.value == -1 and (out == 77).all()
    rc, msg = tile(0, 100, 100, 40, 40, 0)  # 3 x 3 tiles, capacity 4: the needed count comes back and nothing is written
    assert rc != 0 and "capacity 4" in msg and count.value == 9 and (out == 77).all()
    rc, msg = tile(0, 100, 100, 40, 40, 0, cap=0, rois=None)
    assert rc != 0 and count.value == 9
    rc, _ = tile(0, 100, 100, 60, 60, 20)
    assert rc == 0 and count.value == 4 and out[3].tolist() == [0, 3, 40, 40, 60, 60]
    with pytest.raises(SnnbError):
        core.tile_rois((100, 100), (10, 10), 10)


def _rows(*rows):
    a = np.zeros((len(rows), 100, 6), np.float32)
    counts = []
    for s, rs in enumerate(rows):
        for r, row in enumerate(rs):
            a[s, r] = row
        counts.append(len(rs))
    return a, np.array(counts, np.int32)


def test_merge_maps_to_frame_coordinates():
    a, c = _rows([[2, 0.9, 0.25, 0.5, 0.5, 0.25]])
    rows, counts = region_merge.merge_region_rows(a, c, [(1, 0, 100, 40, 200, 80)], None, [(10, 10), (200, 400)], 5)
    assert counts.tolist() == [0, 1] and not rows[0].any()
    f = np.float32
    want = [2, 0.9, (f(100) + f(0.25) * f(200)) / f(400), (f(40) + f(0.5) * f(80)) / f(200), (f(0.5) * f(200)) / f(400), (f(0.25) * f(80)) / f(200)]
    assert np.array_equal(rows[1, 0], np.array(want, np.float32)) and not rows[1, 1:].any()


def test_merge_suppresses_cross_slot_duplicates_and_keeps_other_classes():
    box = [0.1, 0.1, 0.5, 0.5]
    a, c = _rows([[0, 0.9] + box], [[0, 0.8] + box, [1, 0.7] + box])
    rois = [(0, 0, 0, 0, 100, 100), (0, 1, 0, 0, 100, 100)]
    rows, counts = region_merge.merge_region_rows(a, c, rois, None, [(100, 100)], 10)
    assert counts.tolist() == [2] and rows[0, 0, 1] == np.float32(0.9) and rows[0, 1, 0] == 1


def test_merge_iou_threshold():
    # two unit boxes overlapping by o: IoU = o / (2 - o), so o = 0.62 gives 0.4493 (kept) and o = 0.63 gives 0.4599 (dropped)
    for o, kept in ((0.62, 2), (0.63, 1)):
        a, c = _rows([[0, 0.9, 0.0, 0.0, 1.0, 1.0]], [[0, 0.8, 1.0 - o, 0.0, 1.0, 1.0]])
        _, counts = region_merge.merge_region_rows(a, c, [(0, 0, 0, 0, 10, 10), (0, 1, 0, 0, 10, 10)], None, [(10, 10)], 10)
        assert counts[0] == kept, (o, region_merge.yolo_iou(a[0, 0], a[1, 0]))


def test_merge_ties_go_to_the_lower_slot_then_row():
    a, c = _rows([[3, 0.5, 0.0, 0.0, 0.1, 0.1], [4, 0.5, 0.5, 0.5, 0.1, 0.1]], [[5, 0.5, 0.2, 0.2, 0.1, 0.1]], [[6, 0.6, 0.8, 0.8, 0.1, 0.1]])
    rois = [(0, 0, 0, 0, 10, 10), (0, 1, 0, 0, 10, 10), (0, 2, 0, 0, 10, 10)]
    rows, counts = region_merge.merge_region_rows(a, c, rois, None, [(10, 10)], 10)
    assert counts[0] == 4 and rows[0, :4, 0].tolist() == [6, 3, 4, 5]
    rows, counts = region_merge.merge_region_rows(a, c, rois, None, [(10, 10)], 2)  # truncation keeps the first max_rows
    assert counts[0] == 2 and rows[0, :2, 0].tolist() == [6, 3] and rows.shape == (1, 2, 6)


def test_merge_ignores_unused_and_invalid_slots():
    a, c = _rows(*[[[s, 0.9 - 0.01 * s, 0.1 * s, 0.0, 0.05, 0.05]] for s in range(6)])
    rois = [(0, 0, 0, 0, 10, 10), (1, 1, 0, 0, 10, 10), (2, 2, 0, 0, 10, 10), (0, 3, 5, 5, 6, 5), (-1, 4, 0, 0, 1, 1), (0, 5, 0, 0, 10, 10)]
    rows, counts = region_merge.merge_region_rows(a, c, rois, 5, [(10, 10), (10, 10)], 10)  # slot 5 is past the count
    assert counts.tolist() == [1, 1] and rows[0, 0, 0] == 0 and rows[1, 0, 0] == 1
    rows, counts = region_merge.merge_region_rows(a, c, rois, 0, [(10, 10), (10, 10)], 10)
    assert counts.tolist() == [0, 0] and not rows.any()


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and os.path.exists(cand):
            return cand
    return None


def test_merge_kernels_use_no_local_memory():
    tool = _cuobjdump()
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libsnn_b200.so has not been built")
    if tool is None:
        pytest.skip("cuobjdump not found")
    r = subprocess.run([tool, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    seen, cur = {}, None
    for line in r.stdout.splitlines():
        m = re.match(r"\s*Function (_ZN4snnb(\d+)(\S+)):", line)
        if m:
            cur = m.group(3)[:int(m.group(2))] if m.group(3)[:int(m.group(2))] in MERGE_KERNELS else None
            rest = m.group(3)[int(m.group(2)):]
        elif cur is not None and "REG:" in line:
            res = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
            seen[cur + rest] = res
            cur = None
    for name in MERGE_KERNELS:
        assert any(k.startswith(name) for k in seen), "no %s in the library" % name
    assert sum(1 for k in seen if k.startswith("roi_merge_gather_kernel")) == 2  # FrameSizeV and FrameSizesV
    bad = {k: v for k, v in seen.items() if v["STACK"] or v["LOCAL"]}
    assert not bad, bad
