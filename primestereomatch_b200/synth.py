"""Deterministic synthetic stereo pairs (SURVEY.md section 8(d)).

Left image: per channel, a sigma=2 gaussian-blurred N(0,1) field rescaled to unit std, mixed with
white noise and quantised to 8 bits; ground-truth disparity is constant on 40-row bands,
d_gt(y) = 1 + ((y // 40) * 17) mod (D - 2); the right image is the left one shifted by d_gt(y)
(cyclically), so the left map has a known interior answer.
"""
import numpy as np

SEEDS = {(1280, 720, 64): 1280720064, (1920, 1080, 128): 19201080128, (1920, 1080, 256): 19201080256}


def _blur_rows_cols(a, sigma=2.0):
    r = int(4 * sigma + 0.5)
    k = np.exp(-0.5 * (np.arange(-r, r + 1) / sigma) ** 2)
    k /= k.sum()
    a = np.apply_along_axis(lambda v: np.convolve(np.pad(v, r, mode="reflect"), k, mode="valid"), 1, a)
    a = np.apply_along_axis(lambda v: np.convolve(np.pad(v, r, mode="reflect"), k, mode="valid"), 0, a)
    return a


def stereo_pair_u8(W, H, D, seed=None):
    """-> (left_u8[H,W,3], right_u8[H,W,3], d_gt[H]) ; BGR order is irrelevant for synthetic data."""
    if seed is None:
        seed = SEEDS.get((W, H, D), W * 1000003 + H * 1009 + D)
    rng = np.random.default_rng(seed)
    left = np.empty((H, W, 3), np.uint8)
    for c in range(3):
        tex = _blur_rows_cols(rng.standard_normal((H, W)))
        tex /= tex.std()
        v = 128.0 + 48.0 * tex + 16.0 * rng.standard_normal((H, W))
        left[:, :, c] = np.clip(np.rint(v), 0, 255).astype(np.uint8)
    d_gt = 1 + ((np.arange(H) // 40) * 17) % (D - 2)
    cols = (np.arange(W)[None, :] + d_gt[:, None]) % W
    right = np.take_along_axis(left, cols[:, :, None].repeat(3, axis=2), axis=1)
    return left, right, d_gt


def to_f32(img_u8):
    """StereoMatch.cpp:193-197: convertTo(CV_32F, 1/255.0f)."""
    return img_u8.astype(np.float32) * np.float32(1 / np.float32(255.0))


def stereo_pair_f32(W, H, D, seed=None):
    l, r, d = stereo_pair_u8(W, H, D, seed)
    return to_f32(l), to_f32(r), d


def rectify_maps(W, H, SW, SH, view=0, k1=-0.17, k2=0.027):
    """Fixed-point rectification maps of a closed-form rig, for callers without cv2: the W x H crop centred in an SW x SH
    rectified image, seen by a pinhole camera of focal length 0.5 * SW with radial distortion (k1, k2), turned by a small
    in-plane angle that differs per view.  -> (xy int16 (H, W, 2), a uint16 (H, W)), the CV_16SC2 / CV_16UC1 layout of
    initUndistortRectifyMap: each coordinate is rounded to 1/32 px, xy holds its integer part and a = fy * 32 + fx its
    fraction."""
    f, cx, cy = 0.5 * SW, (SW - 1) / 2.0, (SH - 1) / 2.0
    ang = 0.004 if view == 0 else -0.003
    x = np.arange(W, dtype=np.float64)[None, :] + (SW - W) // 2
    y = np.arange(H, dtype=np.float64)[:, None] + (SH - H) // 2
    u, v = (x - cx) / f, (y - cy) / f
    u, v = np.cos(ang) * u - np.sin(ang) * v, np.sin(ang) * u + np.cos(ang) * v
    r2 = u * u + v * v
    d = 1.0 + k1 * r2 + k2 * r2 * r2
    ix = np.rint((f * u * d + cx) * 32).astype(np.int64)
    iy = np.rint((f * v * d + cy) * 32).astype(np.int64)
    xy = np.stack([np.clip(ix >> 5, -32768, 32767), np.clip(iy >> 5, -32768, 32767)], -1).astype(np.int16)
    return xy, ((iy & 31) * 32 + (ix & 31)).astype(np.uint16)
