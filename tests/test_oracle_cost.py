"""CPU-only: the matching-cost restatement of the C oracle at any alpha and truncation thresholds.

* given the defaults (0.9f, no truncation) explicitly it reproduces the raw-volume and map hashes of golden.json, which chains it to the
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


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def golden_cost():
    with open(os.path.join(GOLDEN, "golden_cost.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_default_setting_reproduces_existing_goldens(scene, golden, scenes, oracle):
    g = golden["scenes"][scene]
    _, _, l, r = scenes[scene]
    lg, rg, lraw, rraw = oracle.cost_const(l, r, 64, alpha=0.9, tau_color=np.inf, tau_grad=np.inf)
    assert sha(lg) == g["lGrd"] and sha(rg) == g["rGrd"]
    assert sha(lraw) == g["lRaw"] and sha(rraw) == g["rRaw"]
    lf, rf = oracle.cost_filter(l, r, lraw, rraw)
    assert sha(oracle.wta(lf)) == g["lDis"] and sha(oracle.wta(rf)) == g["rDis"]


@pytest.mark.parametrize("case", sorted(golden_cost()["cases"]))
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_port_matches_cv2_driven_golden(scene, case, scenes, oracle):
    spec = golden_cost()["cases"][case]
    g = spec[scene]
    k = spec["params"]
    _, _, l, r = scenes[scene]
    lraw, rraw = oracle.cost_const(l, r, 64, alpha=k["alpha"], tau_color=k["tau_color"], tau_grad=k["tau_grad"])[2:]
    assert sha(lraw) == g["lRaw"] and sha(rraw) == g["rRaw"]
    lf, rf = oracle.cost_filter(l, r, lraw, rraw)
    assert sha(oracle.wta(lf)) == g["lDis"] and sha(oracle.wta(rf)) == g["rDis"]


def test_shards_are_slices_of_the_whole_volume(oracle):
    rng = np.random.default_rng(9)
    l = rng.random((11, 40, 3), dtype=np.float32)
    r = rng.random((11, 40, 3), dtype=np.float32)
    k = dict(alpha=0.3, tau_color=0.2, tau_grad=0.01)
    lv, rv = oracle.cost_const(l, r, 48, **k)[2:]
    ls, rs = oracle.cost_const(l, r, 48, **k, d_begin=7, d_count=35)[2:]
    assert np.array_equal(ls, lv[7:42]) and np.array_equal(rs, rv[7:42])


def test_nan_survives_truncation(oracle):
    rng = np.random.default_rng(2)
    l = rng.random((6, 30, 3), dtype=np.float32)
    r = rng.random((6, 30, 3), dtype=np.float32)
    l[2, 12, 1] = np.nan
    for k in ((0.9, 0.028, 0.008), (0.5, 0.0, 0.0), (1.0, np.inf, 0.0)):
        lv, rv = oracle.cost_const(l, r, 8, alpha=k[0], tau_color=k[1], tau_grad=k[2])[2:]
        assert np.isnan(lv[:, 2, 12]).all(), k         # the left pixel's own colour difference, interior and border
        assert np.isnan(rv[3, 2, 9]), k                # the right view matches it at x + d = 12
        finite = np.isfinite(lv)
        assert (lv[finite] >= 0).all() and finite.sum() > 0.9 * lv.size
