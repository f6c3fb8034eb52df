"""CPU: the uniqueness restatement (tests/unique_oracle.py): its runner-up form against the hashes pinned in
golden_median.json, against OpenCV's loop over every candidate (check_loop) on the scenes' volumes and on seeded edge
volumes, and the argument checks that need no device."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
import range_cases as RC
import runner_up_cases as RU
import speckle_oracle as SP
import unique_oracle as UN
from primestereomatch_b200 import capi

with open(os.path.join(GOLDEN, "golden_median.json")) as f:
    GOLD = json.load(f)["unique"]
RATIOS = (0, 1, 5, 10, 15, 50, 99, 100)


def planes(vol, lo=0):
    """the selection of a [lo, D) context over vol -> (m as u16, q(m), q(r)) as the library writes them"""
    m, costs, ru = RC.definition(vol, lo)
    return m.astype(np.uint16), costs[1].view(np.float32), ru[1].view(np.float32)


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_scene_maps_equal_the_pinned_hashes(scene, oracle_scene_results):
    ref = oracle_scene_results[scene]
    for key, m, vol in (("l", ref["ld"], ref["lf"]), ("r", ref["rd"], ref["rf"])):
        sm, qm, qr = planes(vol)
        assert np.array_equal(sm, m)
        for ent in GOLD[scene][key]:
            got = UN.check(m, qm, qr, ent["ratio"])
            assert SP.sha(got) == ent["sha"], (scene, key, ent["ratio"])
            assert int(np.count_nonzero(got == m)) == ent["kept"]
            assert np.array_equal(UN.check_loop(m, vol, ent["ratio"]), got)
        assert [e["ratio"] for e in GOLD[scene][key]] == [0, 5, 10, 15, 100]


def edge_volume(D, H, W, seed):
    """costs from a few values, so that exact ties are common, with -0 beside +0, +-inf and NaN"""
    rng = np.random.default_rng(seed)
    values = np.array([-np.inf, -2.0, -0.0, 0.0, 0.5, 0.5, 1.0, 1.05, 3.0, np.inf, np.nan], np.float32)
    vol = values[rng.integers(0, values.size, (D, H, W))]
    return np.where(rng.random((D, H, W)) < 0.3, rng.random((D, H, W)).astype(np.float32), vol).astype(np.float32)


@pytest.mark.parametrize("seed", range(12))
def test_runner_up_form_equals_the_loop_on_edge_volumes(seed):
    """D <= 3 (no runner-up can exist at D = 2 or 3 with m in the middle), range contexts with min_disp > 1, ties,
    -0, +-inf and NaN costs, ratios 0 .. 100"""
    rng = np.random.default_rng(1000 + seed)
    D = int(rng.choice([2, 3, 4, 7, 40]))
    lo = int(rng.integers(0, D)) if seed % 3 == 2 else 0
    vol = edge_volume(D, int(rng.integers(1, 9)), int(rng.integers(1, 40)), seed)
    m, qm, qr = planes(vol, lo)
    for dt in (np.uint8, np.uint16):
        for ratio in RATIOS:
            want = UN.check_loop(m.astype(dt), vol, ratio, lo)
            assert np.array_equal(UN.check(m.astype(dt), qm, qr, ratio), want), (D, lo, ratio)


def test_edge_volumes_reach_the_edges():
    seen = {"nan_qr_kept": 0, "inf_m": 0, "rejected": 0, "lo": 0}
    for seed in range(12):
        rng = np.random.default_rng(1000 + seed)
        D = int(rng.choice([2, 3, 4, 7, 40]))
        lo = int(rng.integers(0, D)) if seed % 3 == 2 else 0
        vol = edge_volume(D, int(rng.integers(1, 9)), int(rng.integers(1, 40)), seed)
        m, qm, qr = planes(vol, lo)
        seen["nan_qr_kept"] += int(np.count_nonzero((m != 0) & np.isnan(qr)))
        seen["inf_m"] += int(np.count_nonzero((m != 0) & np.isneginf(qm)))
        seen["rejected"] += int(np.count_nonzero(UN.check(m, qm, qr, 10) != m))
        seen["lo"] += lo > 1
    assert all(v > 0 for v in seen.values()), seen


def test_definition_by_hand():
    m = np.array([[3, 3, 0, 5, 7]], np.uint8)
    qm = np.array([[1.0, 1.0, 1.0, -0.0, 2.0]], np.float32)
    qr = np.array([[1.1, 1.05, 0.5, 0.0, np.nan]], np.float32)
    # ratio 10: 1.1 * 90 = 99 < 100 rejects; 1.05 * 90 = 94.5 < 100 rejects; m = 0 stays; 0 * 90 < -0 * 100 is false;
    # NaN (no runner-up) keeps
    assert UN.check(m, qm, qr, 10).tolist() == [[0, 0, 0, 5, 7]]
    # ratio 5: 1.1 * 95 = 104.5 keeps, 1.05 * 95 = 99.75 rejects
    assert UN.check(m, qm, qr, 5).tolist() == [[3, 0, 0, 5, 7]]
    # ratio 0 never rejects a runner-up at or above the winner; ratio 100 rejects every positive winner cost
    assert UN.check(m, qm, qr, 0).tolist() == m.tolist()
    assert UN.check(m, qm, qr, 100).tolist() == [[0, 0, 0, 5, 7]]


def test_matches_the_runner_up_model_brute_force(oracle_scene_results):
    """runner_up_cases.uniqueness_brute (the loop as a validity mask) agrees on the Cones volume"""
    ref = oracle_scene_results["Cones"]
    m, vol = ref["ld"], ref["lf"]
    for ratio in (5, 10, 15):
        ok = RU.uniqueness_brute(vol, m, ratio)
        got = UN.check_loop(m, vol, ratio)
        assert np.array_equal(np.where(ok, m, 0), np.where(m != 0, got, 0))


def test_argument_checks_without_a_device():
    m, q = np.ones((2, 3), np.uint8), np.zeros((2, 3), np.float32)
    for ratio in (-1, 101):
        with pytest.raises(AssertionError):
            UN.check(m, q, q, ratio)
    with pytest.raises(AssertionError):
        UN.check(m.astype(np.int32), q, q, 10)
    L = capi.lib()
    assert "psm_set_uniqueness_check" in capi.SYMBOLS
    assert (capi.PSM_UNIQUE_OFF, capi.PSM_UNIQUE_FIRST, capi.PSM_UNIQUE_ONLY) == (0, 1, 2)
    assert L.psm_set_uniqueness_check(None, capi.PSM_UNIQUE_FIRST, 10) == capi.PSM_EINVAL
