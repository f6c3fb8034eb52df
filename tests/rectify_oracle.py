"""CPU restatement of the rectification psm_set_rectify applies in ingest (DESIGN.md section 25): OpenCV's
remap(frame, map[0], map[1], INTER_LINEAR) with the fixed-point maps of initUndistortRectifyMap(..., CV_16SC2) and the
default BORDER_CONSTANT 0, and the reference's crop box.  golden_rectify.json pins it to cv2's own results.

The sum is integer, so its order does not matter: each output is exact."""
import numpy as np


def remap(src, xy, a):
    """u8 (SH, SW, C) frame, int16 (H, W, 2) map[0] (sx, sy), uint16 (H, W) map[1] -> u8 (H, W, C)"""
    src = np.asarray(src, np.uint8)
    if src.ndim == 2:
        return remap(src[:, :, None], xy, a)[:, :, 0]
    SH, SW = src.shape[:2]
    sx = xy[..., 0].astype(np.int64)
    sy = xy[..., 1].astype(np.int64)
    a = a.astype(np.int64) & 1023
    fx, fy = a & 31, a >> 5
    acc = np.zeros(a.shape + (src.shape[2],), np.int64)
    for dx, dy, w in ((0, 0, (32 - fx) * (32 - fy)), (1, 0, fx * (32 - fy)), (0, 1, (32 - fx) * fy), (1, 1, fx * fy)):
        X, Y = sx + dx, sy + dy
        inside = (X >= 0) & (X < SW) & (Y >= 0) & (Y < SH)   # a tap outside the frame reads 0
        v = src[np.clip(Y, 0, SH - 1), np.clip(X, 0, SW - 1)].astype(np.int64) * inside[..., None]
        acc += (w * 32)[..., None] * v
    return ((acc + 16384) >> 15).astype(np.uint8)


def crop_box(roi_left, roi_right):
    """(x, y, w, h) of the box both views' valid ROIs (stereoRectify's validPixROI1 / 2) share, as StereoMatch.cpp:474-478
    computes it"""
    tl_x = max(roi_left[0], roi_right[0])
    tl_y = max(roi_left[1], roi_right[1])
    br_x = min(roi_left[2] + roi_left[0], roi_right[2] + roi_right[0])
    br_y = min(roi_left[3] + roi_left[1], roi_right[3] + roi_right[1])
    return tl_x, tl_y, br_x - tl_x, br_y - tl_y


def crop(m, box):
    """the rows and columns of a map or image inside box (x, y, w, h)"""
    x, y, w, h = box
    return m[y:y + h, x:x + w]
