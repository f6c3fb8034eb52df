#!/usr/bin/env python
"""Pin the disparity-check restatement (tests/dcheck_oracle.py) to OpenCV's own cv2.validateDisparity, without needing
cv2 at test time.

cv2 runs on m * 16 as CV_16S with the costs' int32 dense ranks (only their order matters) as CV_32S, minDisparity = 1
and numberOfDisparities = D - 1: its invalid value is then 0 and its first participating column D.  The right view is
checked as the mirror image.  Cases:
  - "scenes": both views of the D = 64 winner-take-all maps of Cones and Teddy (the oracle's, which equal the
    reference's, golden.json) with the oracle's filtered costs at each winner, at every max_diff of SCENE_DIFFS;
  - "synthetic": seeded maps and costs, inputs in dcheck_cases.npz: zeros, costs drawn from a few values so that many
    claims on one column tie exactly, -0 beside +0, -inf costs, W <= D (no participating column), W = 1, H = 1, and u16
    maps with values up to 2047 (the most m * 16 as CV_16S holds).
Each entry records the sha256 of cv2's result per view and max_diff.  The script fails unless the restatement equals
cv2 everywhere.

Output (committed): tests/golden/golden_dcheck.json, tests/golden/dcheck_cases.npz
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
import dcheck_oracle as DC  # noqa: E402
import speckle_oracle as SP  # noqa: E402

SCENE_DIFFS = [0, 1, 2, 8]
CASE_DIFFS = [0, 1, 2, 5, 64, 2047]
# (key, H, W, D, top map value + 1, u16)
SIZES = [("u8_40x120_D16", 40, 120, 16, 16, False), ("u8_10x200_D64", 10, 200, 64, 64, False),
         ("u8_30x16_D16", 30, 16, 16, 16, False), ("u8_9x10_D32", 9, 10, 32, 32, False),
         ("u8_17x1_D2", 17, 1, 2, 2, False), ("u8_1x200_D8", 1, 200, 8, 8, False), ("u8_1x1_D4", 1, 1, 4, 4, False),
         ("u8_6x300_D256", 6, 300, 256, 256, False), ("u16_3x2200_D2048", 3, 2200, 2048, 2048, True),
         ("u16_6x400_D300", 6, 400, 300, 300, True)]


def cv2_check(m, c, D, max_diff, view):
    """cv2.validateDisparity of one view -> the checked map, of m's dtype"""
    if view:
        return cv2_check(m[:, ::-1], c[:, ::-1], D, max_diff, 0)[:, ::-1].copy()
    disp = np.ascontiguousarray(m.astype(np.int16) * np.int16(16))
    cv2.validateDisparity(disp, np.ascontiguousarray(DC.dense_rank(c)), 1, D - 1, max_diff)
    assert ((disp % 16) == 0).all() and (disp >= 0).all()
    return (disp // 16).astype(m.dtype)


def pinned(m, c, D, diffs, view):
    out = []
    for diff in diffs:
        want = cv2_check(m, c, D, diff, view)
        mine = DC.check(m, c, D, diff, view)
        assert np.array_equal(want, mine), ("cv2 and the restatement differ", m.shape, D, diff, view)
        out.append({"max_diff": diff, "sha": SP.sha(want), "removed": int(np.count_nonzero(want != m))})
    return out


def synthetic(H, W, D, top, wide, seed):
    """a map of piecewise-constant runs with jumps and zeros, and costs from a few values with -0, +0 and -inf"""
    rng = np.random.default_rng(seed)
    run = int(rng.integers(3, 12))
    coarse = rng.integers(1, top, (H, (W + run - 1) // run))
    m = np.repeat(coarse, run, axis=1)[:, :W]
    m = np.where(rng.random((H, W)) < 0.25, rng.integers(1, top, (H, W)), m)
    m = np.where(rng.random((H, W)) < 0.08, 0, m).astype(np.uint16 if wide else np.uint8)
    m[0, -1] = top - 1                                       # the largest value of the range, in the last column
    values = np.array([-np.inf, -1.5, -0.0, 0.0, 0.25, 0.25, 1.0, 3.0], np.float32)
    c = values[rng.integers(0, values.size, (H, W))]
    c = np.where(rng.random((H, W)) < 0.3, rng.random((H, W)).astype(np.float32), c).astype(np.float32)
    return m, c


def main():
    gold = {"cv2": cv2.__version__, "scenes": {}, "synthetic": []}
    for scene in ("Cones", "Teddy"):
        s = scene.lower()
        l = O.u8_to_f32(read_png(os.path.join(HERE, f"{s}_im2.png")))
        r = O.u8_to_f32(read_png(os.path.join(HERE, f"{s}_im6.png")))
        _, _, lraw, rraw = O.cost_const(l, r, 64)
        lf, rf = O.cost_filter(l, r, lraw, rraw)
        ld, rd = O.disp_select(lf, rf)
        gold["scenes"][scene] = {"l": pinned(ld, DC.winner_costs(lf, ld), 64, SCENE_DIFFS, 0),
                                 "r": pinned(rd, DC.winner_costs(rf, rd), 64, SCENE_DIFFS, 1)}
    cases = {}
    for k, (key, H, W, D, top, wide) in enumerate(SIZES):
        m, c = synthetic(H, W, D, top, wide, seed=100 + k)
        cases[key + "_m"], cases[key + "_c"] = m, c
        gold["synthetic"].append({"key": key, "D": D, "l": pinned(m, c, D, CASE_DIFFS, 0),
                                  "r": pinned(m, c, D, CASE_DIFFS, 1)})
    np.savez_compressed(os.path.join(HERE, "dcheck_cases.npz"), **cases)
    with open(os.path.join(HERE, "golden_dcheck.json"), "w") as f:
        json.dump(gold, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
