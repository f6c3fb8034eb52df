#!/usr/bin/env python
"""Pin the YUV-to-BGR restatement (tests/yuv_oracle.py) to OpenCV's own cv2.cvtColor(..., COLOR_YUV2BGR_<FORMAT>),
without needing cv2 at test time.

Cases:
  - "triples": every one of the 2^24 (Y, U, V) triples, as the 4096 x 4096 YUYV frame yuv_oracle.all_triples builds;
    the digest of cv2's output.
  - "frames": all seven formats on seeded frames (yuv_oracle.frame) of 2 x 2, 64 x 48, 130 x 38 (an odd number of
    chroma rows), 1922 x 6 and the reference camera's side-by-side 2688 x 376.  The digest of cv2's output; the npz
    keeps cv2's outputs of the three smallest sizes.
  - "rectify": remap(cvtColor(frame), xy, a, INTER_LINEAR) on every rectify_cases rig, the format cycling through the
    seven, on a seeded frame of the rig's source size; the digest of cv2's output.
The script fails unless the oracle equals cv2 on every case.

Output (committed): tests/golden/golden_yuv.json, tests/golden/yuv_cases.npz
"""
import hashlib
import json
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import rectify_cases  # noqa: E402
import rectify_oracle as RO  # noqa: E402
import yuv_oracle as YO  # noqa: E402

SIZES = ((2, 2), (64, 48), (130, 38), (1922, 6), (2688, 376))
KEEP = ((2, 2), (64, 48), (130, 38))   # sizes whose cv2 outputs the npz keeps
SEED = 2700


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def code(fmt):
    return getattr(cv2, f"COLOR_YUV2BGR_{fmt.upper()}")


def main():
    cases, arrays = [], {}
    got = cv2.cvtColor(YO.all_triples(), cv2.COLOR_YUV2BGR_YUYV)
    assert np.array_equal(got, YO.all_triples_bgr()), "oracle differs from cv2 on the triples"
    assert np.array_equal(got, YO.bgr(YO.all_triples(), "yuyv"))
    cases.append({"name": "triples", "kind": "triples", "sha256": digest(got)})
    for k, (w, h) in enumerate(SIZES):
        for j, fmt in enumerate(YO.FORMATS):
            seed = SEED + 10 * k + j
            f = YO.frame(seed, fmt, w, h)
            want = cv2.cvtColor(f, code(fmt))
            assert np.array_equal(YO.bgr(f, fmt), want), (fmt, w, h)
            name = f"{fmt}_{w}x{h}"
            cases.append({"name": name, "kind": "frame", "format": fmt, "size": [w, h], "seed": seed,
                          "sha256": digest(want)})
            if (w, h) in KEEP:
                arrays[name] = want
    n = 0
    for name, srcs, maps, _ in rectify_cases.load():
        if not name.startswith("rig"):
            continue
        sh, sw = srcs[0].shape[:2]
        fmt = YO.FORMATS[n % len(YO.FORMATS)]
        seed = SEED + 1000 + n
        f = YO.frame(seed, fmt, sw, sh)
        xy, a = maps[0]
        want = cv2.remap(cv2.cvtColor(f, code(fmt)), xy, a, cv2.INTER_LINEAR)
        assert np.array_equal(RO.remap(YO.bgr(f, fmt), xy, a), want), name
        cases.append({"name": f"rect_{name}", "kind": "rectify", "rig": name, "format": fmt, "src": [sw, sh],
                      "seed": seed, "sha256": digest(want)})
        n += 1
    np.savez_compressed(os.path.join(HERE, "yuv_cases.npz"), **arrays)
    with open(os.path.join(HERE, "golden_yuv.json"), "w") as f:
        json.dump({"cv2": cv2.__version__, "cases": cases}, f, indent=1)
    print(f"{len(cases)} cases, oracle == cv2 {cv2.__version__}")


if __name__ == "__main__":
    main()
