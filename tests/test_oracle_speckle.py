"""CPU: the speckle-removal restatements (tests/speckle_oracle.py) against cv2.filterSpeckles' results pinned in
golden_speckle.json, against each other, and the definition's properties."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
import speckle_oracle as SP

with open(os.path.join(GOLDEN, "golden_speckle.json")) as f:
    GOLD = json.load(f)
CASES = np.load(os.path.join(GOLDEN, "speckle_cases.npz"))


def test_synthetic_cases_equal_cv2():
    n = 0
    for ent in GOLD["synthetic"]:
        m = CASES[ent["key"]]
        for s in ent["settings"]:
            got = SP.filter_speckles(m, s["max_size"], s["max_diff"])
            assert got.dtype == m.dtype
            assert SP.sha(got) == s["sha"], (ent["key"], s["max_size"], s["max_diff"])
            n += 1
    assert n == len(GOLD["synthetic"]) * 8


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_scene_maps_equal_cv2(scene, oracle_scene_results):
    ref = oracle_scene_results[scene]
    for view, m in (("l", ref["ld"]), ("r", ref["rd"])):
        for s in GOLD["scenes"][scene][view]:
            got = SP.filter_speckles(m, s["max_size"], s["max_diff"])
            assert SP.sha(got) == s["sha"], (scene, view, s["max_size"], s["max_diff"])
            assert int(np.count_nonzero(got != m)) == s["removed"]


def random_map(H, W, seed, top=8, zeros=0.1, dtype=np.uint8):
    rng = np.random.default_rng(seed)
    m = rng.integers(1, top, (H, W))
    return np.where(rng.random((H, W)) < zeros, 0, m).astype(dtype)


@pytest.mark.parametrize("seed", range(12))
def test_components_equal_flood_fill(seed):
    rng = np.random.default_rng(seed)
    H, W = int(rng.integers(1, 40)), int(rng.integers(1, 40))
    wide = seed % 2 == 1
    m = random_map(H, W, seed, top=4096 if wide and seed % 4 == 1 else 6, dtype=np.uint16 if wide else np.uint8)
    for size in (1, 2, 5, 30, H * W):
        for diff in (0, 1, 2, 300, 5000):
            assert np.array_equal(SP.filter_speckles(m, size, diff), SP.filter_speckles_flood(m, size, diff)), \
                (H, W, size, diff)


@pytest.mark.parametrize("seed", range(6))
def test_idempotent(seed):
    m = random_map(50, 70, seed, top=5)
    for size, diff in ((1, 0), (4, 0), (20, 1), (100, 2)):
        once = SP.filter_speckles(m, size, diff)
        assert np.array_equal(SP.filter_speckles(once, size, diff), once)


@pytest.mark.parametrize("seed", range(6))
def test_larger_max_size_removes_a_superset(seed):
    m = random_map(60, 45, seed, top=7)
    for diff in (0, 1, 3):
        prev = np.zeros(m.shape, bool)
        for size in (1, 2, 3, 8, 20, 100, 10000):
            removed = SP.filter_speckles(m, size, diff) != m
            assert not (prev & ~removed).any(), (diff, size)
            prev = removed


def test_max_diff_at_the_range_joins_every_nonzero_region():
    from scipy.ndimage import label
    for seed in range(4):
        m = random_map(40, 50, seed, top=200, zeros=0.35)
        comp, n = label(m != 0)                                  # 4-connected regions of non-zero pixels
        sizes = np.bincount(comp.ravel())
        rng = int(m.max()) - int(m[m != 0].min())
        for size in (1, 3, 10, 50):
            want = np.where((comp != 0) & (sizes[comp] <= size), 0, m)
            for diff in (rng, rng + 1, 255, 10 ** 6):
                assert np.array_equal(SP.filter_speckles(m, size, diff), want), (seed, size, diff)


def test_zeros_separate_blobs_and_are_kept():
    m = np.array([[3, 3, 0, 3, 3]], np.uint8)
    assert np.array_equal(SP.filter_speckles(m, 2, 0), np.zeros_like(m))
    assert np.array_equal(SP.filter_speckles(m, 1, 0), m)                  # two blobs of 2, not one of 4
    z = np.zeros((3, 4), np.uint16)
    assert np.array_equal(SP.filter_speckles(z, 100, 5), z)
