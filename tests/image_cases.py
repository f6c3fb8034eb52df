"""Seeded float frames outside [0, 1] for the image numerics tests (test_image_numerics.py on the CPU,
test_gpu_image_numerics.py on the device).

psm_set_images takes any float BGR frame.  Two groups of kinds:
  * FLAGGED: the ingest kernel flags the view (a negative, -0, inf, NaN or >= 2^61 channel value) and every stage after it
    runs in OpenCV's order: negative values, -0, +inf, -inf, NaN, values from 2^61 up, values near FLT_MAX (whose
    differences overflow);
  * INEXACT: finite, unflagged values outside the exact-sum domain: 1.7, 1e10, 8421505 (the first float whose product
    with 255 rounds to 2^31), subnormals and values in (0, 2^-12).
The special channel values sit on the seams where the decomposition changes hands: the border columns x < D and
x >= W - D (the fp64 border cost), the mirrored-halo columns 1..8 and W-9..W-2, columns inside a warp of the cost kernel's
interior fast path (128 columns matched inside the image at every disparity), and the strip, remainder and segment seams
of the streaming guided filter (gif_cases.seams).  The right view is the left one shifted by SHIFT columns with its own
special pixels, so that the raw volumes match real structure."""
import numpy as np

import gif_cases as GC

F32 = np.float32
FLAGGED = ("negative", "negzero", "posinf", "neginf", "nan", "huge", "fltmax")
INEXACT = ("above1", "e10", "x8421505", "subnormal", "tiny")
KINDS = FLAGGED + INEXACT
SHIFT = 3

# (W, H, D): fast-path warps exist (columns 128..255 at D = 16); below 32 columns (the separate halo pass); a single pixel
MAIN, NARROW, POINT = (320, 40, 16), (24, 20, 8), (1, 1, 3)
WIDE = (400, 16, 300)        # a 16-bit context: the arg-min of columns >= WIDE_SHIFT is WIDE_SHIFT > 255
WIDE_SHIFT = 270


def _values(kind, rng, n):
    """n special channel values of the kind"""
    if kind == "negative":
        return -np.concatenate([[1e-30, 0.5, 1.0, 3e38], rng.uniform(0, 2, n)])[:n]
    if kind == "negzero":
        return np.full(n, -0.0)
    if kind == "posinf":
        return np.full(n, np.inf)
    if kind == "neginf":
        return np.full(n, -np.inf)
    if kind == "nan":
        v = np.full(n, np.nan, F32)
        v.view(np.uint32)[1::2] = 0xFFC01234       # negative quiet NaN with a payload
        v.view(np.uint32)[2::3] = 0x7FA00001       # signalling-pattern payload
        return v
    if kind == "huge":
        return np.concatenate([[2.0 ** 61, 2.0 ** 63, 1e30], 2.0 ** rng.uniform(61, 120, n)])[:n]
    if kind == "fltmax":
        return np.concatenate([[np.finfo(F32).max, 3.0e38], rng.uniform(1.4e36, 3.4e38, n)])[:n]
    if kind == "above1":
        return np.full(n, 1.7)
    if kind == "e10":
        return np.full(n, 1e10)
    if kind == "x8421505":
        return np.full(n, 8421505.0)
    if kind == "subnormal":
        return np.concatenate([[1e-45, 2.0 ** -149 * 3, 1e-40], rng.uniform(1e-45, 1.1e-38, n)])[:n]
    if kind == "tiny":
        return np.concatenate([[2.0 ** -13, 2.0 ** -12 * 0.999], rng.uniform(1e-9, 2.0 ** -12, n)])[:n]
    raise ValueError(kind)


def columns(W, H, D):
    """the seam columns of a W x H frame at depth D"""
    cols = {0, 1, D - 1, D, W - D - 1, W - D, W - 1}          # border costs
    cols |= {1, 4, 8, W - 9, W - 5, W - 2}                      # mirrored halo
    if W >= 256 + D:
        cols |= {128, 131, 190, 255}                            # a fast-path warp
    if W > 4:
        cols |= set(GC.seams(W, H, max(D, 1))[1])               # strips, packed remainder
    return sorted(c for c in cols if 0 <= c < W)


def rows(W, H, D):
    return GC.seams(W, H, max(D, 1))[0] if H > 4 else list(range(H))


def _place(img, kind, rng, W, H, D, phase, cols=None):
    cols = columns(W, H, D) if cols is None else cols
    rs = rows(W, H, D)
    vals = _values(kind, rng, len(cols)).astype(F32)
    for i, (x, v) in enumerate(zip(cols, vals)):
        y = rs[(i + phase) % len(rs)]
        c = (i + phase) % 3
        img[y, x, c] = v
        if kind == "fltmax" and i % 2 == 0:
            img[y, x, :] = v                                    # all three channels: the colour sums overflow


def frame(kind, W, H, D, seed=0):
    """-> (left, right), float32 BGR frames with the kind's special values on the seams"""
    rng = np.random.default_rng([seed, W, H, D, KINDS.index(kind)])
    base = rng.random((H, W + SHIFT, 3), dtype=F32)
    l = np.ascontiguousarray(base[:, SHIFT:])
    r = np.ascontiguousarray(base[:, :W])
    _place(l, kind, rng, W, H, D, 0)
    _place(r, kind, rng, W, H, D, 1)
    return l, r


def wide_frame(kind, seed=0):
    """-> (left, right) at WIDE: the right view is the left one shifted by WIDE_SHIFT columns, so the left map of columns
    >= WIDE_SHIFT is WIDE_SHIFT; the special values sit in those columns and where they match in the right view"""
    W, H, D = WIDE
    rng = np.random.default_rng([seed, W, H, D, KINDS.index(kind)])
    base = rng.random((H, W + WIDE_SHIFT, 3), dtype=F32)
    l = np.ascontiguousarray(base[:, WIDE_SHIFT:])
    r = np.ascontiguousarray(base[:, :W])
    cols = [WIDE_SHIFT, WIDE_SHIFT + 1, 300, 333, W - 9, W - 2, W - 1]
    _place(l, kind, rng, W, H, D, 0, cols)
    _place(r, kind, rng, W, H, D, 1, [c - WIDE_SHIFT for c in cols] + [5, 129])
    return l, r


def posterised(img, masks=(0xC0, 0xC0, 0xC0)):
    """the frame with its in-range pixels cut to 4 levels per channel (k / 255 floats, which quantise back to k) and its
    special channel values kept: at most 64 colours plus one per special pixel, so the reference's clustering keeps
    every 6-bit colour"""
    img = np.asarray(img, F32)
    with np.errstate(invalid="ignore"):
        inside = (img >= 2.0 ** -12) & (img <= 1)
    k = np.clip(np.rint(np.where(inside, img, 0) * 255), 0, 255).astype(np.uint8) & np.array(masks, np.uint8)
    return np.where(inside, k.astype(F32) / F32(255), img).astype(F32)
