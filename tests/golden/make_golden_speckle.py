#!/usr/bin/env python
"""Pin the speckle-removal restatement (tests/speckle_oracle.py) to OpenCV's own cv2.filterSpeckles(m, 0, max_size,
max_diff), with its optimised (IPP) path on and off, without needing cv2 at test time.

Cases:
  - "scenes": both views of the D = 64 winner-take-all maps of Cones and Teddy (the oracle's, which equal the
    reference's, golden.json) at several (max_size, max_diff);
  - "synthetic": seeded maps, inputs in speckle_cases.npz: piecewise-constant regions with noise and zeros, u8 and
    u16 (filtered as CV_16S, values up to 4095 with neighbour differences above 255), sizes 1 x 1 to 130 x 97 with
    W or H = 1, at several (max_size, max_diff) including max_diff 0 and >= the value range.
Each entry records the sha256 of cv2's result.  The script fails unless the restatement equals cv2's plain path
everywhere, and the IPP path too wherever max_diff fits the map's type (<= 255 on u8, <= 32767 on CV_16S): IPP takes
maxDiff as a pixel value, so beyond that it compares against a wrapped threshold ("ipp_agrees" records which).

Output (committed): tests/golden/golden_speckle.json, tests/golden/speckle_cases.npz
"""
import json
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from conftest import read_png  # noqa: E402
from oracle import oracle as O  # noqa: E402
import speckle_oracle as SP  # noqa: E402

SCENE_SETTINGS = [(1, 0), (10, 0), (50, 1), (100, 1), (400, 2), (1000, 4)]
CASE_SETTINGS = [(1, 0), (2, 0), (4, 1), (20, 2), (100, 1), (400, 2), (10, 300), (50, 100000)]
SIZES = [(1, 1), (1, 57), (45, 1), (31, 33), (64, 64), (97, 130), (40, 300)]   # (H, W)


def synthetic_map(H, W, seed, wide):
    """piecewise-constant regions (a coarse random grid, upsampled), +-1 noise, small islands and zeros"""
    rng = np.random.default_rng(seed)
    top = 4096 if wide else 256
    cell = int(rng.integers(2, 9))
    coarse = rng.integers(1, top, ((H + cell - 1) // cell, (W + cell - 1) // cell))
    m = np.kron(coarse, np.ones((cell, cell), np.int64))[:H, :W]
    m = m + rng.integers(-1, 2, (H, W)) * (rng.random((H, W)) < 0.3)
    islands = rng.random((H, W)) < 0.05
    m = np.where(islands, rng.integers(1, top, (H, W)), m)
    m = np.where(rng.random((H, W)) < 0.08, 0, m)
    return np.clip(m, 0, top - 1).astype(np.uint16 if wide else np.uint8)


def cv2_speckles(m, max_size, max_diff, optimized):
    cv2.setUseOptimized(optimized)
    a = m.astype(np.int16) if m.dtype == np.uint16 else m.copy()
    cv2.filterSpeckles(a, 0, max_size, max_diff)
    return a.astype(m.dtype)


def pinned(m, settings):
    out = []
    for size, diff in settings:
        ipp, plain = cv2_speckles(m, size, diff, True), cv2_speckles(m, size, diff, False)
        mine = SP.filter_speckles(m, size, diff)
        assert np.array_equal(plain, mine), ("cv2 and the restatement differ", size, diff)
        # the IPP path takes maxDiff as a pixel value: it agrees wherever max_diff fits the map's type
        fits = diff <= (255 if m.dtype == np.uint8 else 32767)
        assert np.array_equal(ipp, plain) or not fits, ("IPP and plain cv2 differ", size, diff)
        out.append({"max_size": size, "max_diff": diff, "sha": SP.sha(plain), "ipp_agrees": bool(np.array_equal(ipp, plain)),
                    "removed": int(np.count_nonzero(m != plain))})
    return out


def main():
    gold = {"cv2": cv2.__version__, "scenes": {}, "synthetic": []}
    for scene in ("Cones", "Teddy"):
        s = scene.lower()
        l = O.u8_to_f32(read_png(os.path.join(HERE, f"{s}_im2.png")))
        r = O.u8_to_f32(read_png(os.path.join(HERE, f"{s}_im6.png")))
        _, _, lraw, rraw = O.cost_const(l, r, 64)
        ld, rd = O.disp_select(*O.cost_filter(l, r, lraw, rraw))
        gold["scenes"][scene] = {"l": pinned(ld, SCENE_SETTINGS), "r": pinned(rd, SCENE_SETTINGS)}
    cases = {}
    for k, (H, W) in enumerate(SIZES):
        for wide in (False, True):
            key = f"{'u16' if wide else 'u8'}_{H}x{W}"
            m = cases[key] = synthetic_map(H, W, seed=1000 * k + wide, wide=wide)
            gold["synthetic"].append({"key": key, "settings": pinned(m, CASE_SETTINGS)})
    np.savez_compressed(os.path.join(HERE, "speckle_cases.npz"), **cases)
    with open(os.path.join(HERE, "golden_speckle.json"), "w") as f:
        json.dump(gold, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
