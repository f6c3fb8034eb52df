"""Golden vectors for the matching cost at other settings than the reference's compiled ALPHA_32F = 0.9f without
truncation (include/CVC.h:18-23, src/CVC.cpp:18-39) -- TEST INFRASTRUCTURE.

The reference's truncation lines (CVC.cpp:24-25, 36-37) are commented out, so the other settings are pinned by a
call-by-call restatement driven by OpenCV: cv2.cvtColor / cv2.Sobel for CVC::preprocess, then the cost loops of
CVC.cpp with the truncation restored and float parameters in place of the constants, in numpy float32 / float64 (the
order of make_golden.py's cost4 / cost2).  The guided filter and WTA that follow are make_golden.py's, at the default
window and eps.  Reads only the fixtures in tests/golden/.

Writes tests/golden/golden_cost.json: per setting and scene the sha256 of both raw volumes and both WTA maps after the
default guided filter, and the non-occluded %BP of the left map (StereoMatch.cpp:275-311), Cones and Teddy at D = 64.
Run: python tests/golden/make_golden_cost.py"""
import hashlib
import json
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import bad_pixels, cvc_preprocess, cvf_preprocess, guided  # noqa: E402

f32 = np.float32
D = 64
INF = float("inf")
# (alpha, tau_color, tau_grad): the default, the reference's TAUs on the colour sum, wider thresholds, alpha 0 and 1,
# a zero colour threshold, and the best row of DESIGN.md section 12
CASES = [(0.9, INF, INF), (0.9, 0.028, 0.008), (0.9, 0.084, 0.008), (0.9, 0.3, 0.03), (0.5, INF, INF),
         (0.11, 0.21, 0.008), (0.0, INF, INF), (1.0, INF, INF), (0.9, 0.0, 0.03)]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def case_name(alpha, tc, tg):
    return f"a{alpha:g}_tc{tc:g}_tg{tg:g}"


def weigh(clr, grd, alpha, tc, tg):
    alpha, tc, tg = f32(alpha), f32(tc), f32(tg)
    clr = np.where(clr > tc, tc, clr)                  # CVC.cpp:24 / :36 restored
    grd = np.where(grd > tg, tg, grd)                  # CVC.cpp:25 / :37 restored
    return alpha * clr + (f32(1) - alpha) * grd        # CVC.cpp:26 / :38


def cost4(lC, rC, lG, rG, k):
    clr = (np.abs(lC[..., 0] - rC[..., 0]) + np.abs(lC[..., 1] - rC[..., 1])) + np.abs(lC[..., 2] - rC[..., 2])
    return weigh(clr, np.abs(lG - rG), *k)


def cost2(lC, lG, k):
    lc = lC.astype(np.float64)
    clr = ((np.abs(lc[..., 0] - 1.0) + np.abs(lc[..., 1] - 1.0)) + np.abs(lc[..., 2] - 1.0)).astype(f32)
    grd = np.abs(lG.astype(np.float64) - 1.0).astype(f32)
    return weigh(clr, grd, *k)


def build(l, r, lg, rg, k, right):
    H, W, _ = l.shape
    vol = np.empty((D, H, W), f32)
    for d in range(D):
        if right:   # CVC.cpp:151-179 with the caller's swapped arguments (DispEst.cpp:260)
            vol[d, :, : W - d] = cost4(l[:, : W - d], r[:, d:], lg[:, : W - d], rg[:, d:], k)
            vol[d, :, W - d:] = cost2(l[:, W - d:], lg[:, W - d:], k)
        else:       # CVC.cpp:122-149
            vol[d, :, d:] = cost4(l[:, d:], r[:, : W - d], lg[:, d:], rg[:, : W - d], k)
            vol[d, :, :d] = cost2(l[:, :d], lg[:, :d], k)
    return vol


def main():
    cv2.setNumThreads(1)
    out = {"cv2": cv2.__version__, "D": D, "cases": {}}
    scenes = {}
    for scene in ("Cones", "Teddy"):
        s = scene.lower()
        l = cv2.imread(os.path.join(HERE, f"{s}_im2.png"), cv2.IMREAD_COLOR).astype(f32) * f32(1 / f32(255.0))
        r = cv2.imread(os.path.join(HERE, f"{s}_im6.png"), cv2.IMREAD_COLOR).astype(f32) * f32(1 / f32(255.0))
        gt = cv2.imread(os.path.join(HERE, f"{s}_disp2.png"), cv2.IMREAD_GRAYSCALE)
        occl = cv2.imread(os.path.join(HERE, f"{s}_occl.png"), cv2.IMREAD_GRAYSCALE)
        scenes[scene] = (l, r, cvc_preprocess(l), cvc_preprocess(r), cvf_preprocess(l), cvf_preprocess(r), gt, occl)
    for k in CASES:
        case = {"params": {"alpha": k[0], "tau_color": k[1], "tau_grad": k[2]}}
        for scene, (l, r, lg, rg, lgd, rgd, gt, occl) in scenes.items():
            lraw = build(l, r, lg, rg, k, False)
            rraw = build(r, l, rg, lg, k, True)
            lf = np.stack([guided(*lgd, lraw[d])[0] for d in range(D)])
            rf = np.stack([guided(*rgd, rraw[d])[0] for d in range(D)])
            lDis = (np.argmin(lf[1:], axis=0) + 1).astype(np.uint8)   # DispSel.cpp:93-102
            rDis = (np.argmin(rf[1:], axis=0) + 1).astype(np.uint8)
            case[scene] = {"lRaw": sha(lraw), "rRaw": sha(rraw), "lDis": sha(lDis), "rDis": sha(rDis),
                           "bp_nonocc_left": round(bad_pixels(lDis, gt, occl, 4), 4)}
        out["cases"][case_name(*k)] = case
        print(case_name(*k), case["Cones"]["bp_nonocc_left"], case["Teddy"]["bp_nonocc_left"], flush=True)
    with open(os.path.join(HERE, "golden_cost.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
