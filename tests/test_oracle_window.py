"""CPU-only: the any-window guided-filter restatement (tests/window_oracle.py).

* at (8, 1e-4f) it reproduces the existing goldens, which chains it to the reference's compiled code;
* its box equals live cv2.boxFilter at every window 1..32, on shapes smaller and larger than the window;
* at the other windows it reproduces tests/golden/golden_window.json, written by the cv2-driven make_golden_window.py.
"""
import hashlib
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
import window_oracle as WO


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def golden_window():
    with open(os.path.join(GOLDEN, "golden_window.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_default_parameters_reproduce_existing_goldens(scene, golden, scenes, oracle_scene_results):
    g, ref = golden["scenes"][scene], oracle_scene_results[scene]
    _, _, l, r = scenes[scene]
    rgb, mean, var = WO.cvf_preprocess(l, 8)
    assert sha(mean) == g["lMean"] and sha(var) == g["lVar"]
    for d in (1, 20, 63):
        q, a, b = WO.guided_filter(rgb, mean, var, ref["lraw"][d], 8, 1e-4, want_ab=True)
        assert sha(a) == g[f"l_a_d{d}"] and sha(b) == g[f"l_b_d{d}"]
    lf, rf = WO.cost_filter(l, r, ref["lraw"], ref["rraw"], 8, 1e-4)
    assert sha(lf) == g["lFilt"] and sha(rf) == g["rFilt"]
    assert sha(WO.wta(lf)) == g["lDis"] and sha(WO.wta(rf)) == g["rDis"]


def test_default_fgf_reproduces_existing_golden(scenes, oracle_scene_results):
    with open(os.path.join(GOLDEN, "golden_fgf.json")) as f:
        g = json.load(f)["scenes"]["Teddy"]
    _, _, l, r = scenes["Teddy"]
    ref = oracle_scene_results["Teddy"]
    for s in (2, 4, 8):
        lf, rf = WO.cost_filter_fgf(l, r, ref["lraw"], ref["rraw"], 8, 1e-4, s)
        assert sha(lf) == g[f"s{s}"]["lFilt"] and sha(rf) == g[f"s{s}"]["rFilt"], s


def test_box_matches_live_cv2_at_every_window():
    """The value kinds of test_box_filter_matches_cv2_on_random_shapes_and_ranges, windows 1..32, shapes below and above K."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(17)
    for K in range(1, 33):
        for kind in ("unit", "wide", "sparse", "tiny"):
            h, w = (int(x) for x in rng.integers(1, 2 * K + 20, 2))
            if kind == "unit":
                p = rng.random((h, w), dtype=np.float32)
            elif kind == "wide":
                p = (rng.standard_normal((h, w)) * np.exp(rng.uniform(-20, 10, (h, w)))).astype(np.float32)
            elif kind == "sparse":
                p = (rng.random((h, w)) * (rng.random((h, w)) < 0.2)).astype(np.float32)
            else:
                p = (rng.standard_normal((h, w)) * 1e-41).astype(np.float32)
            assert np.array_equal(WO.box(p, K), cv2.boxFilter(p, -1, (K, K))), (K, kind, h, w)
        # a shape smaller than the window in both directions
        p = rng.random((max(1, K // 2), max(1, K // 3)), dtype=np.float32)
        assert np.array_equal(WO.box(p, K), cv2.boxFilter(p, -1, (K, K))), (K, p.shape)


def test_box_direct_matches_cv2_blur():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    for K in (1, 3, 5, 9, 17, 33):
        p = (rng.standard_normal((45, 70)) * 3).astype(np.float32)
        assert np.array_equal(WO.box_direct(p, K), cv2.blur(p, (K, K))), K


def window_cases():
    with open(os.path.join(GOLDEN, "golden_window.json")) as f:
        return sorted(json.load(f)["cases"].keys())


@pytest.mark.parametrize("case", window_cases())
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_port_matches_cv2_driven_golden(scene, case, golden_window, scenes, oracle_scene_results):
    g = golden_window["cases"][case][scene]
    spec = golden_window["cases"][case]["params"]
    _, _, l, r = scenes[scene]
    ref = oracle_scene_results[scene]
    if spec["kind"] == "gif":
        K, eps = spec["window"], spec["eps"]
        _, mean, var = WO.cvf_preprocess(l, K)
        assert sha(mean) == g["lMean"] and sha(var) == g["lVar"]
        lf, rf = WO.cost_filter(l, r, ref["lraw"], ref["rraw"], K, eps)
    else:
        lf, rf = WO.cost_filter_fgf(l, r, ref["lraw"], ref["rraw"], spec["window"], spec["eps"], spec["s"])
    assert sha(lf) == g["lFilt"] and sha(rf) == g["rFilt"]
    assert sha(WO.wta(lf)) == g["lDis"] and sha(WO.wta(rf)) == g["rDis"]
