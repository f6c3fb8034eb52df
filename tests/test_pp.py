"""Post-processing (PP::processDM -> JointWMF::filter, reference src/PP.cpp:402-425, include/JointWMF.h).

CPU part: the C restatement (oracle.post_process: the un-clustered joint weighted median) against what the reference's
OWN JointWMF.h, compiled into oracle/_ref, returned (recorded in tests/golden by make_golden_ref.py).  The reference clusters the feature colours with cv::kmeans (RNG-seeded,
un-vendored: parity unpinned); when the image has <= 256 distinct 6-bit colours every colour is its own cluster and the
reference's result is well defined -- there the restatement must equal it EXACTLY.  On natural images the agreement with
the (stand-in-clustered) reference is reported and bounded from below.
GPU part: psm_post_process against the restatement, bit-exact."""
import hashlib
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def ref_pp():
    with open(os.path.join(GOLDEN, "ref_outputs.json")) as f:
        return json.load(f)["pp"]


def posterise(img8, masks=(0xE0, 0xE0, 0xC0)):
    return (img8 & np.array(masks, np.uint8)).astype(np.uint8)


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_port_equals_reference_jointwmf_when_clustering_is_exact(scene, scenes, oracle, oracle_scene_results, ref_pp):
    l8, r8, _, _ = scenes[scene]
    ref = oracle_scene_results[scene]
    for view, img8, disp in (("l", l8, ref["ld"]), ("r", r8, ref["rd"])):
        f = oracle.u8_to_f32(posterise(img8))
        want = ref_pp[scene][view]
        assert want["colours"] <= 256, want           # every colour is its own cluster: the reference result is RNG-free
        got = oracle.post_process(f, disp)
        assert sha(got) == want["sha"], f"{scene}: the map differs from the reference's JointWMF"
        assert int((got != disp).sum()) > 1000        # the filter really changes the map


def test_port_vs_clustered_reference_on_natural_image(scenes, oracle, oracle_scene_results, ref_pp):
    """> 256 colours: the reference approximates (JointWMF.h:70-72) through a clustering this repo can only stand in for;
    the un-clustered filter agrees with it on the large majority of pixels (measured 91-92 %)."""
    l8, _, l, _ = scenes["Teddy"]
    disp = oracle_scene_results["Teddy"]["ld"]
    want = np.load(os.path.join(GOLDEN, "ref_pp_teddy.npz"))["lpp"]
    got = oracle.post_process(l, disp)
    assert ref_pp["Teddy_natural_colours"] > 256
    assert float((got == want).mean()) > 0.85


def test_port_definition_small_cases(oracle):
    """Hand-checkable cases of the definition: uniform colour -> plain (unweighted) lower median of the clipped window."""
    H, W = 12, 14
    img = np.full((H, W, 3), 0.5, np.float32)
    rng = np.random.default_rng(1)
    disp = rng.integers(0, 64, (H, W)).astype(np.uint8)
    got = oracle.post_process(img, disp, r=2)
    for (y, x) in ((0, 0), (5, 7), (11, 13), (3, 0)):
        win = disp[max(0, y - 2):y + 3, max(0, x - 2):x + 3].ravel()
        s = np.sort(win)
        # min v with 2*#(I<=v) >= n  -> element at index ceil(n/2)-1
        assert got[y, x] == s[(len(s) + 1) // 2 - 1]


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_gpu_post_process_matches_restatement(scene, scenes, oracle, oracle_scene_results):
    from primestereomatch_b200 import DispEst
    _, _, l, r = scenes[scene]
    ref = oracle_scene_results[scene]
    with DispEst(l, r, 64) as de:
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        assert np.array_equal(de.lDisMap, ref["ld"])
        assert de.PostProcess_GPU() == 0
        lpp, rpp = de.lDisMap.copy(), de.rDisMap.copy()
    assert np.array_equal(lpp, oracle.post_process(l, ref["ld"])), "left post-processed map differs from the restatement"
    assert np.array_equal(rpp, oracle.post_process(r, ref["rd"])), "right post-processed map differs from the restatement"


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", [(37, 21), (130, 50), (19, 19), (5, 40), (300, 9)])
def test_gpu_post_process_ragged_sizes_and_u8_input(W, H, oracle):
    from primestereomatch_b200 import DispEst, capi
    rng = np.random.default_rng(W * 100 + H)
    l8 = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
    r8 = np.roll(l8, -2, axis=1).copy()
    D = 16
    with DispEst(l8, r8, D) as de:
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        ld, rd = de.lDisMap.copy(), de.rDisMap.copy()
        assert de.PostProcess_GPU() == 0
        lpp, rpp = de.lDisMap.copy(), de.rDisMap.copy()
        assert capi.lib().psm_post_process_device(de.handle) == 0     # repeatable
    assert np.array_equal(lpp, oracle.post_process(oracle.u8_to_f32(l8), ld))
    assert np.array_equal(rpp, oracle.post_process(oracle.u8_to_f32(r8), rd))


@pytest.mark.gpu
def test_gpu_post_process_stage_order():
    from primestereomatch_b200 import DispEst, capi
    l = np.zeros((32, 32, 3), np.float32)
    with DispEst(l, l, 8) as de:
        assert capi.lib().psm_post_process_device(de.handle) == capi.PSM_ESTATE
