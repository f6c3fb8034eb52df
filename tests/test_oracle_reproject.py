"""CPU: the reprojection restatement (tests/reproject_oracle.py) against cv2.reprojectImageTo3D's results pinned in
golden_reproject.json, and the definition's properties."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
import reproject_oracle as RP

with open(os.path.join(GOLDEN, "golden_reproject.json")) as f:
    GOLD = json.load(f)
CASES = np.load(os.path.join(GOLDEN, "reproject_cases.npz"))
QS = sorted(k[2:] for k in CASES.files if k.startswith("q_"))


def test_synthetic_cases_equal_cv2():
    for ent in GOLD["synthetic"]:
        got = RP.reproject(CASES["map_" + ent["map"]], CASES["q_" + ent["q"]], ent["hm"])
        assert RP.sha(got) == ent["sha"], (ent["map"], ent["q"], ent["hm"])
        assert int(np.isnan(got).sum()) == ent["nans"]
    maps = {e["map"] for e in GOLD["synthetic"]}
    assert len(GOLD["synthetic"]) == len(maps) * len(QS) * 2
    assert {"u8_1x1_zeros", "u8_1x97_zeros", "u16_53x1_nozero", "u16_const"} <= maps


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_scene_maps_equal_cv2(scene, oracle_scene_results):
    ref = oracle_scene_results[scene]
    ents = [e for e in GOLD["scenes"] if e["scene"] == scene]
    assert len(ents) == 2 * 3 * 2
    for e in ents:
        got = RP.reproject(ref["ld"] if e["view"] == "l" else ref["rd"], CASES["q_" + e["q"]], e["hm"])
        assert RP.sha(got) == e["sha"], (scene, e["view"], e["q"], e["hm"])


def test_signed_zero_and_infinite_w():
    m = np.array([[0, 1, 2]], np.uint8)
    got = RP.reproject(m, CASES["q_signed_zero"])
    assert not np.signbit(got[..., :2]).any()                  # +0.0 + (-0) = +0
    assert np.array_equal(got[0, :, 2], [0, 1, 2])
    w = RP.reproject(m, CASES["q_w_row_minus_zero"])           # h[3] = +0 -> r = +inf
    assert np.isinf(w[..., 2]).all() or np.isnan(w[..., 2]).any()


def test_handle_missing_marks_the_minimum_even_without_zeros():
    m = np.array([[5, 9, 5], [7, 5, 8]], np.uint16)
    q = CASES["q_rectify_shift"]
    off, on = RP.reproject(m, q), RP.reproject(m, q, True)
    assert np.array_equal(on[..., 2] == RP.MISSING_Z, m == 5)
    assert np.array_equal(on[m != 5], off[m != 5])
    assert np.array_equal(on[..., :2], off[..., :2])


def test_comparison_ignores_nan_payloads_only():
    a = np.array([np.nan, 1.0, -0.0], np.float32)
    b = a.copy()
    b.view(np.uint32)[0] = 0xFFC00000
    RP.assert_points_equal(a.reshape(1, 1, 3), b.reshape(1, 1, 3), "payload")
    c = a.copy()
    c[2] = 0.0
    with pytest.raises(AssertionError):
        RP.assert_points_equal(a.reshape(1, 1, 3), c.reshape(1, 1, 3), "signed zero")
