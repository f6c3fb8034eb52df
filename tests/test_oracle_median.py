"""CPU: the median restatement (tests/median_oracle.py) against cv2.medianBlur's results pinned in golden_median.json,
the selection networks of psm_median.cuh on every 0-1 input, and the argument checks that need no device."""
import json
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
import median_oracle as MD
import speckle_oracle as SP
from primestereomatch_b200 import capi

with open(os.path.join(GOLDEN, "golden_median.json")) as f:
    GOLD = json.load(f)


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_scene_maps_equal_cv2(scene, oracle_scene_results):
    ref = oracle_scene_results[scene]
    for key, m in (("l", ref["ld"]), ("r", ref["rd"])):
        for fmt, dt in (("u8", np.uint8), ("u16", np.uint16)):
            for k in MD.KSIZES:
                got = MD.median(m.astype(dt), k)
                assert got.dtype == dt
                assert SP.sha(got) == GOLD["scenes"][scene][key][fmt][str(k)], (scene, key, fmt, k)


def test_seeded_and_degenerate_maps_equal_cv2():
    sizes = set()
    for ent in GOLD["seeded"]:
        m = MD.seeded(ent["H"], ent["W"], ent["u16"], ent["seed"])
        for k in MD.KSIZES:
            assert SP.sha(MD.median(m, k)) == ent["sha"][str(k)], (ent["H"], ent["W"], ent["u16"], k)
        sizes.add((ent["H"], ent["W"]))
        if ent["u16"]:
            assert m.max() > 255 or m.size < 8
    assert {(1, 1), (1, 7), (9, 1), (2, 2), (3, 3), (4, 5), (37, 53), (64, 300)} <= sizes


def test_definition_by_hand():
    m = np.array([[0, 9, 9], [0, 0, 9], [5, 5, 5]], np.uint8)
    # (0, 0): the 3 x 3 window with rows and columns replicated: 0 0 9 / 0 0 9 / 0 0 0 -> 0
    # (1, 1): the map itself: 0 0 0 5 5 5 9 9 9 -> 5
    got = MD.median(m, 3)
    assert got[0, 0] == 0 and got[1, 1] == 5
    assert MD.median(np.array([[7]], np.uint16), 5).tolist() == [[7]]
    # zeros are values: a lone non-zero pixel among zeros goes, a lone zero among equal values is filled
    z = np.zeros((5, 5), np.uint8)
    z[2, 2] = 40
    assert not MD.median(z, 3).any()
    assert (MD.median(np.where(z, 0, 40).astype(np.uint8), 3) == 40).all()


def _network(name):
    src = open(os.path.join(ROOT, "primestereomatch_b200", "csrc", "psm_median.cuh")).read()
    body = re.search(name + r"\(int \(&p\)\[(\d+)\]\)\s*\{(.*?)return p\[(\d+)\];", src, re.S)
    n, out = int(body.group(1)), int(body.group(3))
    return n, out, [(int(a), int(b)) for a, b in re.findall(r"cs\(p, (\d+), (\d+)\)", body.group(2))]


@pytest.mark.parametrize("name, n, count", [("median9", 9, 19), ("median25", 25, 113)])
def test_kernel_networks_select_the_median(name, n, count):
    """the 0-1 principle: a comparator network selects the k-th smallest of any input when it does so on every input of
    0s and 1s; all 2^n of them, as bit columns"""
    nn, out, ces = _network(name)
    assert (nn, out, len(ces)) == (n, n // 2, count)
    chunk = 1 << min(n, 20)
    for hi in range(1 << (n - min(n, 20))):
        idx = np.arange(chunk, dtype=np.uint64) | (np.uint64(hi) << np.uint64(min(n, 20)))
        w = [((idx >> np.uint64(i)) & np.uint64(1)).astype(bool) for i in range(n)]
        ones = sum(x.astype(np.int32) for x in w)
        for a, b in ces:
            w[a], w[b] = w[a] & w[b], w[a] | w[b]
        assert np.array_equal(w[out], ones > n // 2), (name, hi)


def test_argument_checks_without_a_device():
    with pytest.raises(AssertionError):
        MD.median(np.ones((2, 3), np.uint8), 7)
    with pytest.raises(AssertionError):
        MD.median(np.ones((2, 3), np.int32), 3)
    L = capi.lib()
    assert "psm_set_median_blur" in capi.SYMBOLS
    assert (capi.PSM_MEDIAN_OFF, capi.PSM_MEDIAN_FIRST, capi.PSM_MEDIAN_ONLY) == (0, 1, 2)
    assert L.psm_set_median_blur(None, capi.PSM_MEDIAN_FIRST, 3) == capi.PSM_EINVAL
