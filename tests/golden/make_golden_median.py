#!/usr/bin/env python
"""Pin the median restatement (tests/median_oracle.py) to OpenCV's own cv2.medianBlur, and the uniqueness restatement
(tests/unique_oracle.py) to hashes of its result, without needing cv2 at test time.

Median cases, each at ksize 3 and 5 (cv2.medianBlur takes CV_8U and CV_16U at both):
  - "scenes": both views of the D = 64 winner-take-all maps of Cones and Teddy (the oracle's, which equal the
    reference's, golden.json), as u8 and as u16;
  - "seeded": maps drawn from numpy's default_rng(seed) (median_oracle.seeded), u8 up to 255 and u16 up to 4095, a quarter of
    the pixels 0, at the degenerate sizes 1x1, 1x7, 9x1, 2x2, 3x3, 4x5 and at 37x53 and 64x300.
Each entry records the sha256 of cv2's result; the script fails unless the restatement equals cv2 everywhere.

Uniqueness cases: cv2 has no call that takes costs, so "unique" holds the sha256 and the kept-pixel count of
unique_oracle.check on both views of the same scene maps, with the oracle's filtered costs at the winner and at the
runner-up, at every ratio of RATIOS; the script fails unless check equals check_loop there.

Output (committed): tests/golden/golden_median.json
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
import median_oracle as MD  # noqa: E402
import runner_up_cases as RU  # noqa: E402
import speckle_oracle as SP  # noqa: E402
import unique_oracle as UN  # noqa: E402

SIZES = [(1, 1), (1, 7), (9, 1), (2, 2), (3, 3), (4, 5), (37, 53), (64, 300)]   # (H, W)
RATIOS = [0, 5, 10, 15, 100]


def pinned(m):
    out = {}
    for k in MD.KSIZES:
        want = cv2.medianBlur(np.ascontiguousarray(m), k)
        assert np.array_equal(want, MD.median(m, k)), ("cv2 and the restatement differ", m.shape, m.dtype, k)
        out[str(k)] = SP.sha(want)
    return out


def scene_maps(scene):
    """((left map, left filtered volume), (right map, right volume)) of a scene at D = 64"""
    s = scene.lower()
    l = O.u8_to_f32(read_png(os.path.join(HERE, f"{s}_im2.png")))
    r = O.u8_to_f32(read_png(os.path.join(HERE, f"{s}_im6.png")))
    _, _, lraw, rraw = O.cost_const(l, r, 64)
    lf, rf = O.cost_filter(l, r, lraw, rraw)
    ld, rd = O.disp_select(lf, rf)
    return (ld, lf), (rd, rf)


def main():
    gold = {"cv2": cv2.__version__, "scenes": {}, "seeded": [], "unique": {}}
    for scene in ("Cones", "Teddy"):
        views = scene_maps(scene)
        gold["scenes"][scene] = {key: {"u8": pinned(m), "u16": pinned(m.astype(np.uint16))}
                                 for key, (m, _) in zip("lr", views)}
        un = gold["unique"][scene] = {}
        for key, (m, vol) in zip("lr", views):
            qm = np.take_along_axis(vol, m.astype(np.int64)[None], 0)[0]
            qr = RU.definition(vol, m)[1].view(np.float32)
            un[key] = []
            for ratio in RATIOS:
                got = UN.check(m, qm, qr, ratio)
                assert np.array_equal(got, UN.check_loop(m, vol, ratio)), (scene, key, ratio)
                un[key].append({"ratio": ratio, "sha": SP.sha(got), "kept": int(np.count_nonzero(got == m))})
    for k, (H, W) in enumerate(SIZES):
        for u16 in (False, True):
            seed = 200 + 2 * k + u16
            gold["seeded"].append({"H": H, "W": W, "u16": u16, "seed": seed, "sha": pinned(MD.seeded(H, W, u16, seed))})
    with open(os.path.join(HERE, "golden_median.json"), "w") as f:
        json.dump(gold, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
