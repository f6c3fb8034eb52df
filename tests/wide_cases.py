"""Seeded inputs for the 16-bit-map tests (test_oracle_wide.py on the CPU, test_gpu_wide.py on the device, and
golden/make_golden_wide.py): arg-min volumes whose winners mostly exceed 255, and wide maps made from D = 64 maps."""
import numpy as np


def argmin_volume(W, H, D, seed, lo=256):
    """Seeded synthetic volume [D, H, W] whose arg-mins spread over [1, D) with most of them >= lo (when D > lo), and
    with exact ties (the lowest d must win) and +inf / NaN slices mixed in.  -> (vol, intended arg-min)"""
    rng = np.random.default_rng(seed)
    vol = rng.uniform(1.0, 2.0, (D, H, W)).astype(np.float32)
    want = rng.integers(max(1, min(lo, D - 1)) if D > lo else 1, D, (H, W))
    low = rng.random((H, W)) < 0.2
    want = np.where(low, rng.integers(1, D, (H, W)), want)
    yy, xx = np.mgrid[0:H, 0:W]
    vol[want, yy, xx] = 0.5
    # a tie at a higher d never wins
    hi = np.minimum(want + 1 + rng.integers(0, 7, (H, W)), D - 1)
    tie = (rng.random((H, W)) < 0.3) & (hi > want)
    vol[hi[tie], yy[tie], xx[tie]] = 0.5
    vol[0] = 0.0                                        # d = 0 is never a candidate
    vol[:, 0, 0] = np.inf                               # nothing below +inf: 0
    vol[:, 0, 1] = np.nan
    return vol, want


def widen(disp_u8, seed):
    """A wide map from a D = 64 map: 8 * d plus a seeded offset in [0, 8) that is constant on 8 x 8 blocks (values up to
    511, piecewise constant like a real disparity map)."""
    rng = np.random.default_rng(seed)
    H, W = disp_u8.shape
    off = np.repeat(np.repeat(rng.integers(0, 8, ((H + 7) // 8, (W + 7) // 8)), 8, 0), 8, 1)[:H, :W]
    return (disp_u8.astype(np.uint16) * 8 + off).astype(np.uint16)
