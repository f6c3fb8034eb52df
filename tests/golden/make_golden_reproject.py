#!/usr/bin/env python
"""Pin the reprojection restatement (tests/reproject_oracle.py) to OpenCV's own cv2.reprojectImageTo3D, without
needing cv2 at test time.

Cases (maps and Qs in reproject_cases.npz, each with handle_missing off and on):
  - "scenes": both views of the D = 64 winner-take-all maps of Cones and Teddy (the oracle's, which equal the
    reference's, golden.json) with the stereoRectify-shaped Qs and one random Q;
  - "synthetic": seeded u8 maps and u16 maps up to 4095 (passed to cv2 as CV_16S, which cv2 takes, unlike CV_16U), each
    with and without zeros, a constant map and sizes 1 x 1, 1 x W and H x 1, with every Q:
      - cv2.stereoRectify's Q for a made-up rig, with CALIB_ZERO_DISPARITY (cx - cx' = 0) and without (cx - cx' != 0);
      - seeded random Qs whose entries span 1e-6 to 1e6;
      - a zero w row (1 / 0 = inf everywhere), +-inf and NaN entries, and all-(-0) rows (the sum starts from +0.0).
Each entry records the sha256 of cv2's result with its NaNs canonicalised (x86 cv2 gives 0xFFC00000 for 0 * inf; the
device's NaN payload may differ, so NaN positions are compared, not payloads).  The script fails unless the restatement
equals cv2 on every case.

Output (committed): tests/golden/golden_reproject.json, tests/golden/reproject_cases.npz
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
import reproject_oracle as RP  # noqa: E402

SCENE_QS = ["rectify_zero", "rectify_shift", "random0"]


def rectify_q(zero_disparity):
    K1 = np.array([[712.3456789, 0, 640.123], [0, 711.987, 360.987], [0, 0, 1]])
    K2 = np.array([[709.87654, 0, 652.321], [0, 710.123, 355.5], [0, 0, 1]])
    dist = np.array([0.01, -0.02, 0.001, 0.0005, 0.0])
    R = cv2.Rodrigues(np.array([0.002, -0.01, 0.003]))[0]
    T = np.array([-0.1201234, 0.0012, -0.0007])
    flags = cv2.CALIB_ZERO_DISPARITY if zero_disparity else 0
    return cv2.stereoRectify(K1, dist, K2, dist, (1280, 720), R, T, flags=flags)[4]


def qs():
    out = {"rectify_zero": rectify_q(True), "rectify_shift": rectify_q(False)}
    assert out["rectify_zero"][3, 3] == 0 and out["rectify_shift"][3, 3] != 0
    for k in range(4):
        rng = np.random.default_rng(50 + k)
        out[f"random{k}"] = rng.normal(size=(4, 4)) * 10.0 ** rng.uniform(-6, 6, (4, 4))
    w0 = rectify_q(True).copy()
    w0[3] = 0.0
    out["w_row_zero"] = w0
    inf = rectify_q(False).copy()
    inf[0, 0], inf[1, 3], inf[2, 2], inf[3, 1] = np.inf, -np.inf, np.inf, -np.inf
    out["inf"] = inf
    nan = rectify_q(False).copy()
    nan[0, 1], nan[2, 3], nan[3, 0] = np.nan, np.nan, np.nan
    out["nan"] = nan
    sz = np.full((4, 4), -0.0)
    sz[3, 3] = 1.0
    sz[2, 2] = 1.0
    out["signed_zero"] = sz              # X = Y = +0 (not -0); Z = d
    wz = rectify_q(True).copy()
    wz[3] = -0.0                         # h[3] = +0: r = +inf
    out["w_row_minus_zero"] = wz
    return {k: np.asarray(v, np.float64) for k, v in out.items()}


def maps():
    out = {}
    for wide in (False, True):
        top, dt, tag = (4096, np.uint16, "u16") if wide else (256, np.uint8, "u8")
        for k, (H, W) in enumerate([(37, 301), (64, 64), (1, 1), (1, 97), (53, 1)]):
            rng = np.random.default_rng(100 * k + wide)
            m = rng.integers(1, top, (H, W))
            out[f"{tag}_{H}x{W}_nozero"] = m.astype(dt)
            out[f"{tag}_{H}x{W}_zeros"] = np.where(rng.random((H, W)) < 0.1, 0, m).astype(dt)
        out[f"{tag}_const"] = np.full((19, 23), 7 if not wide else 3000, dt)
    return out


def cv2_points(m, Q, hm):
    a = m.astype(np.int16) if m.dtype == np.uint16 else m
    return cv2.reprojectImageTo3D(a, Q, handleMissingValues=bool(hm))


def pinned(m, Q, what):
    out = []
    for hm in (0, 1):
        ref = cv2_points(m, Q, hm)
        RP.assert_points_equal(RP.reproject(m, Q, hm), ref, f"{what} handle_missing {hm}: restatement vs cv2")
        out.append({"hm": hm, "sha": RP.sha(ref), "nans": int(np.isnan(ref).sum())})
    return out


def main():
    Q = qs()
    M = maps()
    gold = {"cv2": cv2.__version__, "scenes": [], "synthetic": []}
    for scene in ("Cones", "Teddy"):
        s = scene.lower()
        l = O.u8_to_f32(read_png(os.path.join(HERE, f"{s}_im2.png")))
        r = O.u8_to_f32(read_png(os.path.join(HERE, f"{s}_im6.png")))
        _, _, lraw, rraw = O.cost_const(l, r, 64)
        ld, rd = O.disp_select(*O.cost_filter(l, r, lraw, rraw))
        for view, m in (("l", ld), ("r", rd)):
            for q in SCENE_QS:
                for e in pinned(m, Q[q], f"{scene} {view} {q}"):
                    gold["scenes"].append({"scene": scene, "view": view, "q": q, **e})
    for key, m in M.items():
        for q in Q:
            for e in pinned(m, Q[q], f"{key} {q}"):
                gold["synthetic"].append({"map": key, "q": q, **e})
    np.savez_compressed(os.path.join(HERE, "reproject_cases.npz"), **{f"map_{k}": v for k, v in M.items()},
                        **{f"q_{k}": v for k, v in Q.items()})
    with open(os.path.join(HERE, "golden_reproject.json"), "w") as f:
        json.dump(gold, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
