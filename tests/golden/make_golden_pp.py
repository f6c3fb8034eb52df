#!/usr/bin/env python
"""Pin the post-filter restatement (oracle.post_process, orc_wmf in oracle/stereo_oracle.c) to the reference's OWN
include/JointWMF.h at a set of psm_set_post_filter settings, without needing the reference at test time.

Needs a checkout of PRiMEStereoMatch (REF, default /root/reference) and a C++ compiler with OpenMP: ref_wmf_driver.cpp
is compiled against REF/include (JointWMF.h unmodified) and oracle/shim with the flags of oracle/Makefile's _ref build,
into a temporary directory.

Inputs: posterised Cones and Teddy (<= 256 distinct 6-bit colours, so that the reference's colour clustering is
exact, as in tests/test_pp.py), both views, starting from the D = 64 winner-take-all maps (which equal the reference's,
tests/golden/golden.json).  For every setting the golden records, per scene and view: the sha256 of the restatement's
output, the sha256 of the reference's, the number of pixels where they differ and the colour count; per setting the
sha256 of the restatement's weight table.

Output (committed): tests/golden/golden_pp.json
"""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from conftest import read_png  # noqa: E402
from oracle import oracle as O  # noqa: E402

REF = os.environ.get("REF", "/root/reference")

# (radius, sigma, iterations, weight)
SETTINGS = [
    (9, 25.5, 1, "exp"),
    (4, 25.5, 1, "exp"),
    (16, 25.5, 1, "exp"),
    (32, 25.5, 1, "exp"),
    (9, 10.0, 1, "exp"),
    (9, 80.0, 1, "exp"),
    (9, 25.5, 3, "exp"),
    (9, 25.5, 1, "iv1"),
    (9, 25.5, 1, "iv2"),
    (9, 25.5, 1, "off"),
    (20, 25.5, 2, "iv2"),
    (9, 2.0 ** -16, 1, "iv2"),
    (9, 2.0 ** -16, 1, "exp"),
    (9, 2.0 ** 16, 1, "iv1"),
    (9, 2.0 ** 16, 1, "exp"),
]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def posterise(img8, masks=(0xE0, 0xE0, 0xC0)):
    return (img8 & np.array(masks, np.uint8)).astype(np.uint8)


def key(r, sigma, it, weight):
    return f"{r}/{float(sigma).hex()}/{it}/{weight}"


def ref_lib(tmp):
    shim = os.path.join(ROOT, "oracle", "shim")
    so = os.path.join(tmp, "libref_wmf.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    obj = os.path.join(tmp, "stereo_oracle.o")
    subprocess.run(["gcc", "-O3", "-std=c11", "-fPIC", "-pthread", "-ffp-contract=off", "-fno-fast-math", "-c", "-o", obj,
                    os.path.join(ROOT, "oracle", "stereo_oracle.c")], check=True)
    subprocess.run([cxx, "-O3", "-std=c++11", "-fPIC", "-pthread", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-w",
                    "-I" + shim, "-I" + os.path.join(REF, "include"), "-shared", "-o", so,
                    os.path.join(HERE, "ref_wmf_driver.cpp"), os.path.join(shim, "opencv_shim.cpp"), obj, "-lm", "-lpthread"],
                   check=True)
    L = C.CDLL(so)
    f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
    u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")
    L.ref_wmf.argtypes = [f32p, u8p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, u8p, C.POINTER(C.c_int)]
    return L


def main():
    if not os.path.exists(os.path.join(REF, "include", "JointWMF.h")):
        raise SystemExit(f"{REF}/include/JointWMF.h not found: set REF to a PRiMEStereoMatch checkout")
    inputs = {}
    for name in ("Cones", "Teddy"):
        s = name.lower()
        l8 = read_png(os.path.join(HERE, f"{s}_im2.png"))
        r8 = read_png(os.path.join(HERE, f"{s}_im6.png"))
        res = O.pipeline(O.u8_to_f32(l8), O.u8_to_f32(r8), 64, threads=8)
        inputs[name] = {"l": (O.u8_to_f32(posterise(l8)), res["lDis"]), "r": (O.u8_to_f32(posterise(r8)), res["rDis"])}
    out = {"inputs": "posterised (0xE0, 0xE0, 0xC0) Cones / Teddy, D = 64 WTA maps", "settings": []}
    with tempfile.TemporaryDirectory() as tmp:
        L = ref_lib(tmp)
        for (r, sigma, it, weight) in SETTINGS:
            ent = {"key": key(r, sigma, it, weight), "radius": r, "sigma": float(sigma).hex(), "iterations": it,
                   "weight": weight, "table_sha": sha(O.weight_table(sigma, weight)), "scenes": {}}
            for name, views in inputs.items():
                ent["scenes"][name] = {}
                for view, (img, disp) in views.items():
                    H, W = disp.shape
                    want = np.empty((H, W), np.uint8)
                    n = C.c_int(0)
                    assert L.ref_wmf(img, np.ascontiguousarray(disp), W, H, r, sigma, it, O.WEIGHTS[weight], want,
                                     C.byref(n)) == 0
                    got = O.post_process(img, disp, r, sigma, it, weight)
                    ent["scenes"][name][view] = {"sha": sha(got), "ref_sha": sha(want), "differ": int((got != want).sum()),
                                                 "colours": n.value}
                    assert n.value <= 256
            print(ent["key"], {k: [v["differ"] for v in s.values()] for k, s in ent["scenes"].items()}, flush=True)
            out["settings"].append(ent)
    with open(os.path.join(HERE, "golden_pp.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote golden_pp.json")


if __name__ == "__main__":
    main()
