"""The rectification cases of golden_rectify.json as frame pairs: each case is
(name, (src_left, src_right), (maps_left, maps_right), (sha256_left, sha256_right)), maps = (xy, a) cropped to the
output, sha256 = the digest of cv2's rectified u8 output (None where cv2 was not run on that view).

  - rig cases: both views of a stereoRectify rig; the big rigs give one case per band of rows of the crop;
  - random cases: one map for both views, the right frame being the left one with its channels reversed."""
import json
import os

import numpy as np

import rectify_oracle as RO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def frame(seed, sw, sh):
    return np.random.default_rng(seed).integers(0, 256, (sh, sw, 3), dtype=np.uint8)


def load():
    meta = json.load(open(os.path.join(GOLDEN, "golden_rectify.json")))
    z = np.load(os.path.join(GOLDEN, "rectify_cases.npz"))
    out = []
    for c in meta["cases"]:
        name = c["name"]
        if c["kind"] == "random":
            src = z[f"{name}_src"]
            maps = (z[f"{name}_xy"], z[f"{name}_a"])
            out.append((name, (src, np.ascontiguousarray(src[..., ::-1])), (maps, maps), (c["sha256"], None)))
            continue
        sw, sh = c["src"]
        srcs = tuple(frame(c["seed"] + v, sw, sh) for v in range(2))
        if c["full_maps"]:
            maps = tuple((RO.crop(z[f"{name}_{v}_xy"], c["box"]), RO.crop(z[f"{name}_{v}_a"], c["box"])) for v in range(2))
            out.append((name, srcs, maps, tuple(view["sha256"] for view in c["views"])))
            continue
        for k in range(len(c["views"][0]["bands"])):
            maps = tuple((z[f"{name}_{v}_band{k}_xy"], z[f"{name}_{v}_band{k}_a"]) for v in range(2))
            out.append((f"{name}_band{k}", srcs, maps, tuple(view["bands"][k]["sha256"] for view in c["views"])))
    return out
