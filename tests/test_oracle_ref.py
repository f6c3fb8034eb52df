"""Pins the C port (oracle/stereo_oracle.c) to the reference's OWN compiled code: the reference's
src/{CVC,CVF,DispSel}.cpp built unmodified against oracle/shim (only the five OpenCV image primitives are
stand-ins, themselves pinned against cv2 in test_oracle.py).  What that build returned for these inputs is
recorded in tests/golden/ref_outputs.json (tests/golden/make_golden_ref.py); reference == port == golden."""
import hashlib
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, read_png


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def ref_outputs():
    with open(os.path.join(GOLDEN, "ref_outputs.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_ref_equals_port_equals_golden(scene, oracle_scene_results, golden, ref_outputs):
    port = oracle_scene_results[scene]
    ref = ref_outputs["scenes"][scene]
    for k_ref, k_port in (("lGrd", "lg"), ("rGrd", "rg"), ("lRaw", "lraw"), ("rRaw", "rraw"),
                          ("lVol", "lf"), ("rVol", "rf"), ("lDis", "ld"), ("rDis", "rd")):
        assert sha(port[k_port]) == ref[k_ref], f"{scene}: reference {k_ref} != port {k_port}"
    s = scene.lower()
    assert np.array_equal(port["ld"], read_png(os.path.join(GOLDEN, f"{s}_lDis.png")))
    assert np.array_equal(port["rd"], read_png(os.path.join(GOLDEN, f"{s}_rDis.png")))
    # the cv2-driven golden hashes (tests/golden/make_golden.py) hold for the reference's compiled code as well
    g = golden["scenes"][scene]
    for gk, rk in (("lGrd", "lGrd"), ("rGrd", "rGrd"), ("lRaw", "lRaw"), ("rRaw", "rRaw"),
                   ("lFilt", "lVol"), ("rFilt", "rVol"), ("lDis", "lDis"), ("rDis", "rDis")):
        assert ref[rk] == g[gk], f"{scene}: reference {gk} differs from the cv2-driven golden hash"


def test_ref_thread_counts_and_both_code_paths(scenes, oracle, ref_outputs):
    """The reference gives the same volumes at threads = 1, 3, 8 (remainder batches, DispEst.cpp:238) and from the
    non-pthread twins buildCV_left/right (CVC.cpp:122-179) and CVSelect_thread (DispSel.cpp:53-81) -- checked when
    the record was made; the port reproduces that one result on the same crop."""
    _, _, l, r = scenes["Teddy"]
    l, r = l[:60, :128].copy(), r[:60, :128].copy()
    D = 12
    want = ref_outputs["teddy_crop_D12"]
    for t in (1, 3, 8):
        _, _, lraw, rraw = oracle.cost_const(l, r, D, threads=t)
        lf, rf = oracle.cost_filter(l, r, lraw, rraw, threads=t)
        ld, rd = oracle.disp_select(lf, rf)
        got = {"lRaw": lraw, "rRaw": rraw, "lVol": lf, "rVol": rf, "lDis": ld, "rDis": rd}
        for k, v in got.items():
            assert sha(v) == want[k], (t, k)
    assert sha(oracle.wta(lf)) == want["lDis"]


def test_ref_guided_filter_on_arbitrary_costs(oracle, ref_outputs):
    """GuidedFilter_cv compiled from the reference vs the port on signed, wide-range caller-provided costs."""
    rng = np.random.default_rng(8)
    H, W = 48, 77
    img = rng.random((H, W, 3), dtype=np.float32)
    rgb, mean, var = oracle.cvf_preprocess(img)
    for scale in (1.0, 1e-4, 300.0):
        p = (rng.normal(0, 1, (H, W)) * scale).astype(np.float32)
        assert sha(oracle.guided_filter(rgb, mean, var, p)) == ref_outputs["guided_filter_48x77"][repr(scale)], scale


def test_ref_gray_mode_switch(scenes, oracle, ref_outputs):
    _, _, l, r = scenes["Cones"]
    l, r = l[:40, :90].copy(), r[:40, :90].copy()
    for gm in (0, 1):
        want = ref_outputs["gray_mode_cones_crop_D6"][str(gm)]
        lg, rg, lraw, rraw = oracle.cost_const(l, r, 6, gray_mode=gm)
        assert sha(lg) == want["lGrd"] and sha(lraw) == want["lRaw"] and sha(rraw) == want["rRaw"], gm
