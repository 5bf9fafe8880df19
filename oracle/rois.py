"""TEST INFRASTRUCTURE - numpy float32 restatement of snnb_rois_from_detections (detection rows -> regions), and of the crop that
defines what snnb_model_run_rois feeds a slot. Every float32 operation below is one IEEE-rounded numpy operation, in the order snnb.h
states, so the device kernel (which uses __fmul_rn / __fadd_rn / __fsub_rn, no FMA) must equal it bit for bit."""
import numpy as np


def roi_of_row(row, frame_w, frame_h, min_score=0.0, class_id=-1, expand=0.0):
    """The region (x, y, width, height) of one {class, score, x, y, w, h} row, or None when the row is not kept."""
    cls, score, x, y, w, h = (np.float32(v) for v in np.asarray(row, np.float32))
    if not score >= np.float32(min_score):
        return None
    if class_id != -1 and cls != np.float32(class_id):
        return None
    W, H, e = np.float32(frame_w), np.float32(frame_h), np.float32(expand)
    with np.errstate(invalid="ignore", over="ignore"):
        ex, ey = e * w, e * h
        fx0, fx1 = (x - ex) * W, ((x + w) + ex) * W
        fy0, fy1 = (y - ey) * H, ((y + h) + ey) * H
    if any(np.isnan(v) for v in (fx0, fx1, fy0, fy1)):
        return None
    clamp = lambda v, hi: min(max(v, np.float32(0)), hi)  # noqa: E731  (no NaN reaches here)
    x0, x1 = int(np.floor(clamp(fx0, W))), int(np.ceil(clamp(fx1, W)))
    y0, y1 = int(np.floor(clamp(fy0, H))), int(np.ceil(clamp(fy1, H)))
    if x1 <= x0 or y1 <= y0:
        return None
    return x0, y0, x1 - x0, y1 - y0


def rois_from_detections(rows, counts, frame_hw, capacity, min_score=0.0, class_id=-1, expand=0.0):
    """rows [N, max_rows, 6] float32, counts [N] -> (rois [capacity, 6] int32 {frame, row, x, y, width, height}, zero past the count;
    count = min(kept, capacity)). Rows r < min(counts[n], max_rows) are visited frame by frame, in row order."""
    rows = np.asarray(rows, np.float32)
    n_frames, max_rows = rows.shape[:2]
    out = np.zeros((capacity, 6), np.int32)
    kept = 0
    for n in range(n_frames):
        for r in range(min(int(counts[n]), max_rows)):
            roi = roi_of_row(rows[n, r], frame_hw[1], frame_hw[0], min_score, class_id, expand)
            if roi is None:
                continue
            if kept < capacity:
                out[kept] = (n, r) + roi
            kept += 1
    return out, min(kept, capacity)


def crop_rgba(F, roi):
    """S_i of snnb_model_run_rois: region roi = {frame, row, x, y, width, height} cut out of F, libyuv's RGBA8 of the whole frames
    ([N, H, W, 4], indexed by the region's frame; or one frame [H, W, 4])."""
    frame, _, x, y, w, h = (int(v) for v in roi)
    img = F[frame] if F.ndim == 4 else F
    return np.ascontiguousarray(img[y:y + h, x:x + w])
