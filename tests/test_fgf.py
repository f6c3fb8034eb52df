"""Fast Guided Filter branch (reference src/fastguidedfilter.cpp via DispEst::CostFilter_FGF, src/DispEst.cpp:281-296).
CPU: the C port against the cv2-driven golden (tests/golden/make_golden_fgf.py: the reference's code followed call by
call through the real cv2 primitives, IPP off).  GPU: psm_cost_filter_fgf against the port, bit-exact."""
import hashlib
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def golden_fgf():
    with open(os.path.join(GOLDEN, "golden_fgf.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("s", [4, 2, 8])
def test_port_matches_cv2_driven_golden(s, scenes, oracle, oracle_scene_results, golden_fgf):
    _, _, l, r = scenes["Teddy"]
    ref = oracle_scene_results["Teddy"]
    g = golden_fgf["scenes"]["Teddy"][f"s{s}"]
    lf, rf = oracle.cost_filter_fgf(l, r, ref["lraw"], ref["rraw"], s=s)
    assert sha(lf) == g["lFilt"] and sha(rf) == g["rFilt"]
    assert sha(lf[1]) == g["l_d1"] and sha(lf[20]) == g["l_d20"] and sha(lf[63]) == g["l_d63"]
    assert sha(oracle.wta(lf)) == g["lDis"] and sha(oracle.wta(rf)) == g["rDis"]


def test_port_primitives_against_live_cv2(oracle):
    """The two OpenCV primitives the FGF branch adds (K x K blur, INTER_LINEAR up-sampling) against the cv2 in this image."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    for (H, W, K) in ((67, 120, 5), (40, 33, 9), (21, 19, 3)):
        p = (rng.standard_normal((H, W)) * 3).astype(np.float32)
        assert np.array_equal(oracle.box_direct(p, K), cv2.blur(p, (K, K)))


@pytest.mark.gpu
@pytest.mark.parametrize("s", [4, 2, 8, 1])
def test_gpu_fgf_matches_port(s, scenes, oracle, oracle_scene_results):
    from primestereomatch_b200 import DispEst
    _, _, l, r = scenes["Teddy"]
    ref = oracle_scene_results["Teddy"]
    lf, rf = oracle.cost_filter_fgf(l, r, ref["lraw"], ref["rraw"], s=s)
    with DispEst(l, r, 64) as de:
        de.setSubsampleRate(s)
        de.CostConst_GPU()
        assert de.CostFilter_FGF_GPU() == 0
        gl, gr = de.read_cost_volume(0), de.read_cost_volume(1)
        de.DispSelect_GPU()
        ld, rd = de.lDisMap.copy(), de.rDisMap.copy()
    bad = np.argwhere(gl != lf)
    assert bad.size == 0, f"s={s}: {len(bad)} left voxels differ, first {bad[0].tolist()}: {gl[tuple(bad[0])]!r} vs {lf[tuple(bad[0])]!r}"
    assert np.array_equal(gr, rf)
    assert np.array_equal(ld, oracle.wta(lf)) and np.array_equal(rd, oracle.wta(rf))


@pytest.mark.gpu
@pytest.mark.parametrize("W,H,D,s", [(463, 370, 8, 4), (130, 50, 5, 2), (37, 41, 4, 8), (450, 375, 6, 4), (64, 19, 3, 4)])
def test_gpu_fgf_ragged_sizes(W, H, D, s, oracle):
    """Sizes that are not multiples of the sub-sampling rate (the Middlebury third-size scenes are 463x370 / 447x370)."""
    from primestereomatch_b200 import DispEst, capi
    rng = np.random.default_rng(W + H)
    l = rng.random((H, W, 3), dtype=np.float32)
    r = np.clip(np.roll(l, -2, axis=1) + rng.normal(0, 0.02, (H, W, 3)), 0, 1).astype(np.float32)
    _, _, lraw, rraw = oracle.cost_const(l, r, D)
    lf, rf = oracle.cost_filter_fgf(l, r, lraw, rraw, s=s)
    with DispEst(l, r, D) as de:
        de.setSubsampleRate(s)
        de.CostConst_GPU()
        de.CostFilter_FGF_GPU()
        assert np.array_equal(de.read_cost_volume(0), lf)
        assert np.array_equal(de.read_cost_volume(1), rf)
        assert capi.lib().psm_cost_filter_fgf(de.handle, s) == capi.PSM_ESTATE      # already filtered
        de.CostConst_GPU()
        assert capi.lib().psm_cost_filter_fgf(de.handle, 3) == capi.PSM_EINVAL
