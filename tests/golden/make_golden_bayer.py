#!/usr/bin/env python
"""Pin the demosaicing restatement (tests/bayer_oracle.py) to OpenCV's own cv2.cvtColor(..., COLOR_Bayer<PATTERN>2BGR)
and COLOR_Bayer<PATTERN>2BGR_EA, without needing cv2 at test time.

Cases, each on all eight codes (four patterns, two methods):
  - "frame": seeded frames (bayer_oracle.frame) of 1 x 1, 2 x 2, 2 x 9, 9 x 2 (below cv2's 3 x 3, all zero), 3 x 3,
    64 x 48, 130 x 38, 1922 x 6, and the two halves of the reference camera's side-by-side 2688 x 376 frame, each
    demosaiced as a frame of its own; the digest of cv2's output.  The npz keeps cv2's outputs up to 64 x 48.
  - "ties": 64 x 48 frames of values 0..2 and of 0 / 255 only, where the edge-aware rule's two differences tie often.
  - "rectify": remap(cvtColor(frame), xy, a, INTER_LINEAR) on every rectify_cases rig, the code cycling through the
    eight, on a seeded frame of the rig's source size; the digest of cv2's output.
The script fails unless the oracle (both of its forms, where the loop is affordable) equals cv2 on every case.

Output (committed): tests/golden/golden_bayer.json, tests/golden/bayer_cases.npz
"""
import hashlib
import json
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import bayer_oracle as BO  # noqa: E402
import rectify_cases  # noqa: E402
import rectify_oracle as RO  # noqa: E402

SIZES = ((1, 1), (2, 2), (2, 9), (9, 2), (3, 3), (64, 48), (130, 38), (1922, 6))
SIDE_BY_SIDE = (2688, 376)
KEEP_PIXELS = 64 * 48   # frames up to this many pixels keep cv2's output in the npz
LOOP_PIXELS = 130 * 38   # ... and are checked against the per-pixel loop too
SEED = 2800
CODES = [(p, m) for m in BO.METHODS for p in BO.PATTERNS]


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def code(pattern, method):
    return (BO.CV2_CODE_EA if method == "ea" else BO.CV2_CODE)[pattern]


def tie_frame(kind, seed):
    """a 64 x 48 frame of values 0..2 ("low") or of 0 and 255 only ("binary")"""
    f = BO.frame(seed, 64, 48, 3 if kind == "low" else 2)
    return f if kind == "low" else f * np.uint8(255)


def check(f, pattern, method, what):
    want = cv2.cvtColor(f, code(pattern, method))
    assert cv2.COLOR_BayerRGGB2BGR == BO.CV2_CODE["rggb"] and cv2.COLOR_BayerGBRG2BGR_EA == BO.CV2_CODE_EA["gbrg"]
    assert np.array_equal(BO.bgr(f, pattern, method), want), what
    if f.size <= LOOP_PIXELS:
        assert np.array_equal(BO.bgr_loop(f, pattern, method), want), what
    return want


def main():
    cases, arrays = [], {}
    for k, (w, h) in enumerate(SIZES):
        for j, (pattern, method) in enumerate(CODES):
            seed = SEED + 10 * k + j
            want = check(BO.frame(seed, w, h), pattern, method, (w, h, pattern, method))
            name = f"{pattern}_{method}_{w}x{h}"
            cases.append({"name": name, "kind": "frame", "pattern": pattern, "method": method, "size": [w, h],
                          "seed": seed, "sha256": digest(want)})
            if w * h <= KEEP_PIXELS:
                arrays[name] = want
    w, h = SIDE_BY_SIDE
    for j, (pattern, method) in enumerate(CODES):
        seed = SEED + 500 + j
        sbs = BO.frame(seed, w, h)
        for half, cols in (("left", slice(0, w // 2)), ("right", slice(w // 2, w))):
            want = check(np.ascontiguousarray(sbs[:, cols]), pattern, method, (half, pattern, method))
            cases.append({"name": f"{pattern}_{method}_sbs_{half}", "kind": "side_by_side", "half": half,
                          "pattern": pattern, "method": method, "size": [w, h], "seed": seed, "sha256": digest(want)})
    for t, kind in enumerate(("low", "binary")):
        for j, (pattern, method) in enumerate(CODES):
            seed = SEED + 600 + 10 * t + j
            want = check(tie_frame(kind, seed), pattern, method, (kind, pattern, method))
            name = f"{pattern}_{method}_ties_{kind}"
            cases.append({"name": name, "kind": "ties", "values": kind, "pattern": pattern, "method": method,
                          "seed": seed, "sha256": digest(want)})
            arrays[name] = want
    n = 0
    for name, srcs, maps, _ in rectify_cases.load():
        if not name.startswith("rig"):
            continue
        sh, sw = srcs[0].shape[:2]
        pattern, method = CODES[n % len(CODES)]
        seed = SEED + 1000 + n
        f = BO.frame(seed, sw, sh)
        xy, a = maps[0]
        want = cv2.remap(cv2.cvtColor(f, code(pattern, method)), xy, a, cv2.INTER_LINEAR)
        assert np.array_equal(RO.remap(BO.bgr(f, pattern, method), xy, a), want), name
        cases.append({"name": f"rect_{name}", "kind": "rectify", "rig": name, "pattern": pattern, "method": method,
                      "src": [sw, sh], "seed": seed, "sha256": digest(want)})
        n += 1
    np.savez_compressed(os.path.join(HERE, "bayer_cases.npz"), **arrays)
    with open(os.path.join(HERE, "golden_bayer.json"), "w") as f:
        json.dump({"cv2": cv2.__version__, "cases": cases}, f, indent=1)
    print(f"{len(cases)} cases, oracle == cv2 {cv2.__version__}")


if __name__ == "__main__":
    main()
