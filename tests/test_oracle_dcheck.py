"""CPU: the disparity-check restatement (tests/dcheck_oracle.py) against cv2.validateDisparity's results pinned in
golden_dcheck.json, against the literal row loop, beyond cv2's domain, and the argument checks that need no device."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
import dcheck_oracle as DC
import speckle_oracle as SP
from primestereomatch_b200 import capi

with open(os.path.join(GOLDEN, "golden_dcheck.json")) as f:
    GOLD = json.load(f)
CASES = np.load(os.path.join(GOLDEN, "dcheck_cases.npz"))


def test_synthetic_cases_equal_cv2():
    n = 0
    for ent in GOLD["synthetic"]:
        m, c = CASES[ent["key"] + "_m"], CASES[ent["key"] + "_c"]
        for view, key in ((0, "l"), (1, "r")):
            for s in ent[key]:
                got = DC.check(m, c, ent["D"], s["max_diff"], view)
                assert got.dtype == m.dtype
                assert SP.sha(got) == s["sha"], (ent["key"], view, s["max_diff"])
                assert np.array_equal(DC.check_rows(m, c, ent["D"], s["max_diff"], view), got), (ent["key"], view)
                n += 1
    assert n == len(GOLD["synthetic"]) * 2 * 6


def test_cases_cover_the_edges():
    """ties, -0 beside +0 and -inf among the participating pixels; W <= D, W = 1, H = 1; u16 values up to 2047"""
    keys = [e["key"] for e in GOLD["synthetic"]]
    shapes = {k: (CASES[k + "_m"].shape, e["D"]) for k, e in zip(keys, GOLD["synthetic"])}
    assert any(W <= D for (_, W), D in shapes.values())
    assert any(W == 1 for (_, W), _ in shapes.values()) and any(H == 1 for (H, _), _ in shapes.values())
    assert max(int(CASES[k + "_m"].max()) for k in keys if CASES[k + "_m"].dtype == np.uint16) == 2047
    c = np.concatenate([CASES[k + "_c"].ravel() for k in keys])
    assert np.isneginf(c).any() and (np.signbit(c) & (c == 0)).any() and (~np.signbit(c) & (c == 0)).any()
    m, c = CASES["u8_40x120_D16_m"], CASES["u8_40x120_D16_c"]
    x2 = np.arange(m.shape[1])[None, :] - m.astype(np.int64)
    part = (np.arange(m.shape[1]) >= 16)[None, :] & (m != 0)
    claims = {}
    for y, x in zip(*np.nonzero(part)):
        claims.setdefault((y, x2[y, x]), []).append(int(DC.order_key(c[y, x])))
    assert sum(len(v) - len(set(v)) for v in claims.values()) > 50, "too few exact ties on one claimed column"


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_scene_maps_equal_cv2(scene, oracle_scene_results):
    ref = oracle_scene_results[scene]
    for view, key, m, vol in ((0, "l", ref["ld"], ref["lf"]), (1, "r", ref["rd"], ref["rf"])):
        c = DC.winner_costs(vol, m)
        for s in GOLD["scenes"][scene][key]:
            got = DC.check(m, c, 64, s["max_diff"], view)
            assert SP.sha(got) == s["sha"], (scene, key, s["max_diff"])
            assert int(np.count_nonzero(got != m)) == s["removed"]
            # only the order of the costs matters
            assert np.array_equal(DC.check(m, DC.dense_rank(c).astype(np.float32), 64, s["max_diff"], view), got)


@pytest.mark.parametrize("seed", range(10))
def test_vectorised_equals_row_loop_beyond_cv2(seed):
    """u16 values above 2047 (m * 16 overflows CV_16S there), max_diff up to 4095, signed zeros and ties"""
    rng = np.random.default_rng(seed)
    H, W = int(rng.integers(1, 12)), int(rng.integers(1, 400))
    wide = seed % 2 == 1
    D = int(rng.integers(1, 4096 if wide else 256))
    top = max(2, min(D, int(rng.integers(2, 5000 if wide else 257))))
    m = rng.integers(0, top, (H, W)).astype(np.uint16 if wide else np.uint8)
    m = np.where(rng.random((H, W)) < 0.1, 0, m).astype(m.dtype)
    c = np.array([-0.0, 0.0, 1.0, -np.inf, 2.0], np.float32)[rng.integers(0, 5, (H, W))]
    for diff in (0, 1, 7, 300, 2048, 4095):
        for view in (0, 1):
            assert np.array_equal(DC.check(m, c, D, diff, view), DC.check_rows(m, c, D, diff, view)), (H, W, D, diff)


def test_definition_by_hand():
    # x = 4..7 claim 4 - 2 = 2, 5 - 3 = 2, 6 - 1 = 5, 7 - 2 = 5; column 2: cost 1.0 (x = 4) beats 2.0 (x = 5), so d2 = 2
    # and x = 5 (3) is off by 1; column 5: -0 (x = 6) ties +0 (x = 7), the lower x wins: d2 = 1 and x = 7 (2) is off by 1
    m = np.array([[9, 0, 1, 2, 2, 3, 1, 2]], np.uint8)
    c = np.array([[5, 5, 5, 5, 1.0, 2.0, -0.0, 0.0]], np.float32)
    assert DC.check(m, c, 4, 0).tolist() == [[9, 0, 1, 2, 2, 0, 1, 0]]
    assert DC.check(m, c, 4, 1).tolist() == m.tolist()
    assert DC.check(m, c, 8, 0).tolist() == m.tolist()                     # no column at or beyond D
    # the right view mirrors it
    assert DC.check(m[:, ::-1], c[:, ::-1], 4, 0, view=1).tolist() == [[0, 1, 0, 2, 2, 1, 0, 9]]
    # -inf is the lowest cost; a checked 0 stays 0
    c2 = np.array([[0, 0, 0, 0, 1.0, -np.inf, 0, 0]], np.float32)
    assert DC.check(m, c2, 4, 0).tolist() == [[9, 0, 1, 2, 0, 3, 1, 0]]


def test_argument_checks_without_a_device():
    m, c = np.ones((2, 3), np.uint8), np.zeros((2, 3), np.float32)
    for diff in (-1, DC.MAX_DIFF + 1):
        with pytest.raises(AssertionError):
            DC.check(m, c, 2, diff)
    with pytest.raises(AssertionError):
        DC.check(m.astype(np.int32), c, 2, 1)
    L = capi.lib()
    assert "psm_set_disparity_check" in capi.SYMBOLS
    assert (capi.PSM_DCHECK_OFF, capi.PSM_DCHECK_FIRST, capi.PSM_DCHECK_ONLY) == (0, 1, 2)
    assert L.psm_set_disparity_check(None, capi.PSM_DCHECK_FIRST, 1) == capi.PSM_EINVAL
