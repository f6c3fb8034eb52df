"""CPU-only: the any-setting matching-cost restatement (tests/cost_oracle.py).

* at the defaults (0.9f, no truncation) it reproduces the raw-volume and map hashes of golden.json, which chains it to the
  reference's compiled code;
* at the other settings it reproduces tests/golden/golden_cost.json, written by the cv2-driven make_golden_cost.py;
* a NaN in the image survives the truncation.
"""
import hashlib
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
import cost_oracle as CO
import window_oracle as WO


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def golden_cost():
    with open(os.path.join(GOLDEN, "golden_cost.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_default_setting_reproduces_existing_goldens(scene, golden, scenes):
    g = golden["scenes"][scene]
    _, _, l, r = scenes[scene]
    assert sha(CO.preprocess(l)) == g["lGrd"] and sha(CO.preprocess(r)) == g["rGrd"]
    lraw, rraw = CO.cost_volumes(l, r, 64, *CO.DEFAULT)
    assert sha(lraw) == g["lRaw"] and sha(rraw) == g["rRaw"]
    lf, rf = WO.cost_filter(l, r, lraw, rraw)
    assert sha(WO.wta(lf)) == g["lDis"] and sha(WO.wta(rf)) == g["rDis"]


def test_gradient_matches_the_c_oracle(oracle):
    rng = np.random.default_rng(5)
    for H, W in ((37, 53), (1, 1), (3, 2), (20, 131)):
        img = rng.random((H, W, 3), dtype=np.float32)
        assert np.array_equal(CO.preprocess(img), oracle.cvc_preprocess(img)), (H, W)


@pytest.mark.parametrize("case", sorted(golden_cost()["cases"]))
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_port_matches_cv2_driven_golden(scene, case, scenes):
    spec = golden_cost()["cases"][case]
    g = spec[scene]
    k = spec["params"]
    _, _, l, r = scenes[scene]
    lraw, rraw = CO.cost_volumes(l, r, 64, k["alpha"], k["tau_color"], k["tau_grad"])
    assert sha(lraw) == g["lRaw"] and sha(rraw) == g["rRaw"]
    lf, rf = WO.cost_filter(l, r, lraw, rraw)
    assert sha(WO.wta(lf)) == g["lDis"] and sha(WO.wta(rf)) == g["rDis"]


def test_shards_are_slices_of_the_whole_volume():
    rng = np.random.default_rng(9)
    l = rng.random((11, 40, 3), dtype=np.float32)
    r = rng.random((11, 40, 3), dtype=np.float32)
    k = (0.3, 0.2, 0.01)
    lv, rv = CO.cost_volumes(l, r, 48, *k)
    ls, rs = CO.cost_volumes(l, r, 48, *k, d_begin=7, d_count=35)
    assert np.array_equal(ls, lv[7:42]) and np.array_equal(rs, rv[7:42])


def test_nan_survives_truncation():
    rng = np.random.default_rng(2)
    l = rng.random((6, 30, 3), dtype=np.float32)
    r = rng.random((6, 30, 3), dtype=np.float32)
    l[2, 12, 1] = np.nan
    for k in ((0.9, 0.028, 0.008), (0.5, 0.0, 0.0), (1.0, np.inf, 0.0)):
        lv, rv = CO.cost_volumes(l, r, 8, *k)
        assert np.isnan(lv[:, 2, 12]).all(), k         # the left pixel's own colour difference, interior and border
        assert np.isnan(rv[3, 2, 9]), k                # the right view matches it at x + d = 12
        finite = np.isfinite(lv)
        assert (lv[finite] >= 0).all() and finite.sum() > 0.9 * lv.size
