"""CPU: the guided-filter references pinned to OpenCV on the inputs of test_gpu_gif_numerics.py.

tests/golden/golden_gif.json holds sha256 values of CVF::preprocess, GuidedFilter_cv and the WTA computed call by call
with real cv2.boxFilter (tests/golden/make_golden_gif.py, IPP off), on every cost kind and image kind of gif_cases:
non-finite and 1e30 costs, a 1e15 band, wide-range, signed-zero and tied costs, a near-black float guide, its 8-bit
version and a guide with NaN / inf pixels -- inputs where OpenCV's running fp64 sums give other floats than any other
summation order.  The C oracle (orc_cvf_preprocess, orc_guided_filter, orc_wta) must reproduce every value, slice by
slice and on whole volumes, NaN at the same places whatever the payload.  The device is compared with it, so this is what
ties it to OpenCV."""
import importlib.util
import json
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")


def _generator():
    spec = importlib.util.spec_from_file_location("make_golden_gif", os.path.join(GOLDEN, "make_golden_gif.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def gen():
    pytest.importorskip("cv2")
    return _generator()


@pytest.fixture(scope="module")
def golden_gif():
    with open(os.path.join(GOLDEN, "golden_gif.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def cases(gen):
    return gen.inputs()


CASES = ["cost_posinf", "cost_neginf", "cost_nan", "cost_outlier", "cost_mixed", "cost_ties", "cost_band", "cost_wide40",
         "image_dark_f32", "image_dark_u8", "image_nan_f32"]


def test_cases_cover_every_kind(golden_gif):
    import gif_cases as GC
    assert sorted(golden_gif["cases"]) == sorted(CASES)
    assert sorted(CASES) == sorted([f"cost_{k}" for k in GC.COST_KINDS] + [f"image_{k}" for k in GC.IMAGE_KINDS])


@pytest.mark.parametrize("case", CASES)
def test_c_oracle_equals_opencv(case, cases, golden_gif, gen, oracle):
    img, vol = cases[case]
    g = golden_gif["cases"][case]
    with np.errstate(all="ignore"):
        rgb, mean, var = oracle.cvf_preprocess(img)
        q = np.stack([oracle.guided_filter(rgb, mean, var, vol[d]) for d in range(vol.shape[0])])
    assert gen.sha(mean) == g["mean"], f"{case}: orc_cvf_preprocess mean"
    assert gen.sha(var) == g["var"], f"{case}: orc_cvf_preprocess var"
    assert [gen.sha(s) for s in q] == g["slices"], f"{case}: orc_guided_filter"
    assert gen.sha(oracle.wta(q)) == g["wta"], f"{case}: orc_wta"
    assert int(np.isnan(q).sum()) == g["nan"]


@pytest.mark.parametrize("case", CASES)
def test_c_oracle_on_whole_volumes_equals_opencv(case, cases, golden_gif, gen, oracle):
    """the volume at once, window and eps given explicitly, as the device tests call the oracle"""
    img, vol = cases[case]
    g = golden_gif["cases"][case]
    rgb, mean, var = oracle.cvf_preprocess(img, window=8)
    q = oracle.guided_filter(rgb, mean, var, vol, window=8, eps=1e-4)
    assert gen.sha(mean) == g["mean"], f"{case}: orc_cvf_preprocess mean"
    assert gen.sha(var) == g["var"], f"{case}: orc_cvf_preprocess var"
    assert [gen.sha(s) for s in q] == g["slices"], f"{case}: orc_guided_filter"
    assert gen.sha(oracle.wta(q)) == g["wta"], f"{case}: orc_wta"


def test_generator_reproduces_the_golden_byte_for_byte(gen):
    with open(os.path.join(GOLDEN, "golden_gif.json")) as f:
        assert gen.golden_text() == f.read()


def test_orders_differ_on_these_inputs(cases, oracle):
    """the cases are ones where the summation order matters: direct window sums give other means than OpenCV's"""
    img, vol = cases["cost_band"]
    p = vol[1]
    assert np.count_nonzero(oracle.box(p, 8) != oracle.box_direct(p, 8)) > 1000
    img, _ = cases["image_dark_f32"]
    prod = img[..., 0] * img[..., 1]
    assert np.count_nonzero(oracle.box(prod, 8) != oracle.box_direct(prod, 8)) > 100


# ---- the carried-error bound the device test asserts on inexact sums is not vacuous ------------------------------------
@pytest.mark.parametrize("kind", ["wide40", "ties", "band"])
def test_carried_error_bound_catches_small_errors(kind, cases, oracle):
    """gif_cases.carried_error_bound is per voxel: a relative error of 1e-3 (far below any image-wide bound) lies beyond
    it at most voxels of wide-range and tied costs, and above the 1e15 band of 'band', whose rounding the running sums
    carry only below it"""
    import gif_cases as GC
    img, vol = cases[f"cost_{kind}"]
    p = vol[2]
    with np.errstate(all="ignore"):
        rgb, mean, var = oracle.cvf_preprocess(img)
        q = oracle.guided_filter(rgb, mean, var, p)
    bound = GC.carried_error_bound(img, p)
    assert not GC.beyond_bound(q, q, bound).any()
    far = GC.beyond_bound(q * np.float32(1 + 1e-3), q, bound)
    if kind == "band":
        assert far[:4].mean() > 0.9, far[:4].mean()
    else:
        assert far.mean() > 0.9, far.mean()
