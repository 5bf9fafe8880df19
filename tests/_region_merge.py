"""TEST INFRASTRUCTURE - numpy float32 restatement of snnb_model_detect_rois' mapping and per-frame merge (include/snnb.h, steps 3 to 5):
each slot's detection rows mapped to its frame, one stable score sort and one greedy NMS per frame. Every float32 operation below is one
IEEE-rounded numpy operation in the order the header states, and yolo_iou follows the device's operation order, so the merge kernels
must equal it bit for bit. Used by tests/test_detect_rois_*.py and by the torch workaround of tools/device_io_bench.py --parts tiled."""
import numpy as np


def yolo_iou(a, b):
    """iou of the engine's NMS (layers.cpp / yolo_iou in kernels_simt.cu) on two {cls, score, x, y, w, h} rows, every float32
    operation in its order; std::max(p, q) = p < q ? q : p and std::min(p, q) = q < p ? q : p."""
    ax, ay, aw, ah = (np.float32(v) for v in a[2:6])
    bx, by, bw, bh = (np.float32(v) for v in b[2:6])
    ix0, iy0 = (bx if ax < bx else ax), (by if ay < by else ay)
    ax1, bx1, ay1, by1 = ax + aw, bx + bw, ay + ah, by + bh
    ix1, iy1 = (bx1 if bx1 < ax1 else ax1), (by1 if by1 < ay1 else ay1)
    if ix1 < ix0 or iy1 < iy0:
        return np.float32(0)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        inter = (ix1 - ix0) * (iy1 - iy0)
        return inter / ((aw * ah + bw * bh) - inter)


def roi_valid(roi, slot, used, frame_sizes):
    """The slot rule of snnb_model_run_rois: slot < used and the region lies inside the frame it names (frame_sizes: (H, W) each)."""
    f, _, x, y, w, h = (int(v) for v in roi)
    if not (slot < used and 0 <= f < len(frame_sizes) and w >= 1 and h >= 1 and x >= 0 and y >= 0):
        return False
    H, W = frame_sizes[f]
    return x + w <= W and y + h <= H


def merge_region_rows(slot_rows, slot_counts, rois, count, frame_sizes, max_rows):
    """snnb_model_detect_rois' steps 3 to 5 (include/snnb.h): slot_rows [B, >= slot_counts[i], 6] and slot_counts [B], each slot's
    detect_frames rows of its crop; rois [B, 6] {frame, row, x, y, width, height}; count None (every slot used) or the device count;
    frame_sizes one (H, W) per frame. Returns (rows [num_frames, max_rows, 6] float32, zero past each count, counts [num_frames] int32)."""
    slot_rows = np.asarray(slot_rows, np.float32)
    B, F = len(rois), len(frame_sizes)
    used = B if count is None else min(max(int(count), 0), B)
    lists = [[] for _ in range(F)]
    for s in range(B):
        if not roi_valid(rois[s], s, used, frame_sizes):
            continue
        f, _, rx, ry, rw, rh = (int(v) for v in rois[s])
        H, W = (np.float32(v) for v in frame_sizes[f])
        rx, ry, rw, rh = np.float32(rx), np.float32(ry), np.float32(rw), np.float32(rh)
        for r in range(int(slot_counts[s])):
            cls, score, x, y, w, h = (np.float32(v) for v in slot_rows[s, r])
            lists[f].append(np.array([cls, score, (rx + x * rw) / W, (ry + y * rh) / H, (w * rw) / W, (h * rh) / H], np.float32))
    out = np.zeros((F, max_rows, 6), np.float32)
    counts = np.zeros(F, np.int32)
    for f, rows in enumerate(lists):
        order = sorted(range(len(rows)), key=lambda i: -float(rows[i][1]))  # stable: equal scores keep slot, then row order
        kept = []
        for i in order:
            if len(kept) == max_rows:
                break
            b = rows[i]
            if not any(k[0] == b[0] and yolo_iou(k, b) > np.float32(0.45) for k in kept):
                kept.append(b)
        counts[f] = len(kept)
        if kept:
            out[f, :len(kept)] = np.stack(kept)
    return out, counts
