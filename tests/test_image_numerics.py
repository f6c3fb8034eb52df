"""CPU: every stage that reads a float frame, pinned to OpenCV and to the reference's own compiled code on frames outside
[0, 1] (tests/image_cases.py: negative, -0, +-inf, NaN, >= 2^61 and near-FLT_MAX channel values, and the finite inexact
ones 1.7, 1e10, 8421505, subnormals and (0, 2^-12), placed on the seams of the device's decomposition).

* The post-filter's colour quantisation (`convertTo(CV_8UC3, 255)`, orc_f32_to_u8x255, which the `_ref` shim's
  Mat::convertTo calls) equals cv2's float -> u8 conversion on every value of tests/golden/golden_image.json: 0, not 255,
  where fl(v * 255) is NaN or >= 2^31 (x86 cvRound returns INT_MIN there).
* CVC::preprocess of the oracle (gray_mode 0) equals cv2.cvtColor + cv2.Sobel on every frame.
* The reference's CVC / CVF / WTA compiled against the shim equal the port on the flagged frames (the ones the device
  filters in OpenCV's order), and its JointWMF, given the frames' 8-bit colours, equals the port's post-filter of
  posterised frames with special pixels."""
import importlib.util
import json
import os

import numpy as np
import pytest

import image_cases as IC
from gif_cases import assert_same

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
SIZES = {"main": IC.MAIN, "narrow": IC.NARROW, "point": IC.POINT}


@pytest.fixture(scope="module")
def golden_image():
    with open(os.path.join(GOLDEN, "golden_image.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def ref():
    from oracle import ref as R
    if not R.available():
        pytest.skip("oracle/_ref not built (needs the reference sources)")
    return R


def frame(kind, size):
    if size == "wide":
        return IC.wide_frame(kind)
    return IC.frame(kind, *SIZES[size])


def sha(a):
    import hashlib
    a = np.array(a, copy=True)
    a[np.isnan(a)] = np.float32(np.nan)
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ---- pinned to cv2 ----------------------------------------------------------------------------------------------------
def test_quantisation_equals_opencv(golden_image, oracle):
    t = golden_image["u8x255"]
    v = np.array(t["bits"], np.uint32).view(np.float32)
    want = np.array(t["u8"], np.uint8)
    got = oracle.to_u8x255(v.reshape(1, -1, 1)).ravel()
    bad = np.flatnonzero(got != want)
    assert not len(bad), (f"{len(bad)} of {len(v)} differ, first {v[bad[0]]!r} (0x{v.view(np.uint32)[bad[0]]:08x}): "
                          f"{got[bad[0]]} vs cv2 {want[bad[0]]}")
    # the rule as DESIGN.md section 13 states it
    with np.errstate(all="ignore"):
        q = v * np.float32(255)
        rule = np.where(np.isnan(q) | (q >= 2.0 ** 31), 0, np.clip(np.rint(q), 0, 255)).astype(np.uint8)
    assert np.array_equal(rule, want)
    for x, u in ((8421504.0, 255), (8421505.0, 0), (1e10, 0), (np.inf, 0), (1.7, 255), (-0.0, 0), (0.5 / 255, 0)):
        assert oracle.to_u8x255(np.array([[[x]]], np.float32))[0, 0, 0] == u, x


def test_table_covers_the_classes(golden_image):
    v = np.array(golden_image["u8x255"]["bits"], np.uint32).view(np.float32)
    assert len(v) % golden_image["row"] == golden_image["row"] - 3
    with np.errstate(all="ignore"):
        q = v * np.float32(255)
    assert np.isnan(v).sum() >= 8 and np.isposinf(v).any() and np.isneginf(v).any()
    assert ((q >= 2.0 ** 31) & (q < 2.0 ** 63)).sum() >= 5 and ((q >= 2.0 ** 63) & np.isfinite(q)).any()
    assert (np.isinf(q) & np.isfinite(v)).any() and ((v > 0) & (v < np.finfo(np.float32).tiny)).any()
    k = np.arange(256)
    half = ((k + 0.5) / 255).astype(np.float32)
    assert set(half.view(np.uint32)) <= set(v.view(np.uint32))


@pytest.mark.parametrize("size", ["main", "narrow", "point", "wide"])
@pytest.mark.parametrize("kind", IC.KINDS)
def test_gradients_equal_opencv(kind, size, golden_image, oracle):
    l, r = frame(kind, size)
    with np.errstate(all="ignore"):
        got = [sha(oracle.cvc_preprocess(x, 0)) for x in (l, r)]
    assert got == golden_image["gradients"][f"{kind}_{size}"]


def test_generator_reproduces_the_golden_byte_for_byte():
    pytest.importorskip("cv2")
    spec = importlib.util.spec_from_file_location("make_golden_image", os.path.join(GOLDEN, "make_golden_image.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    with open(os.path.join(GOLDEN, "golden_image.json")) as f:
        assert gen.golden_text() == f.read()


# ---- the reference's compiled code on the flagged frames ------------------------------------------------------------------
@pytest.mark.parametrize("gray_mode", [0, 1])
@pytest.mark.parametrize("threads", [1, 3])
@pytest.mark.parametrize("size", ["main", "narrow"])
@pytest.mark.parametrize("kind", IC.FLAGGED)
def test_reference_pipeline_equals_port(kind, size, threads, gray_mode, ref, oracle):
    """(the 1 x 1 frame is left out: at D > W the reference's buildCV loops run past the row)"""
    l, r = frame(kind, size)
    D = SIZES[size][2]
    with np.errstate(all="ignore"):
        got = ref.pipeline(l, r, D, threads=threads, gray_mode=gray_mode, keep=True)
        lg, rg, lraw, rraw = oracle.cost_const(l, r, D, threads=threads, gray_mode=gray_mode)
        want = oracle.pipeline(l, r, D, threads=threads, gray_mode=gray_mode, keep_volumes=True)
    what = f"{kind} {size} threads {threads} gray_mode {gray_mode}"
    for k, w in (("lGrd", lg), ("rGrd", rg), ("lRaw", lraw), ("rRaw", rraw), ("lVol", want["lVol"]), ("rVol", want["rVol"]),
                 ("lDis", want["lDis"]), ("rDis", want["rDis"])):
        assert_same(got[k], w, f"{what}: {k}")


@pytest.mark.parametrize("kind", IC.KINDS)
def test_reference_post_filter_equals_port(kind, ref, oracle):
    """JointWMF compiled from the reference (its clustering keeps every colour of a frame with <= 256 6-bit colours)
    equals the port's post-filter on posterised frames whose special pixels quantise to 0 or 255.

    The reference is given the frame's 8-bit colours as k / 255 floats, which every version of the quantisation maps
    back to k: what is compared is the reference's JointWMF, not the shim's stand-in for convertTo (that step is
    orc_f32_to_u8x255, pinned to cv2 by test_quantisation_equals_opencv), so a `_ref` built from an older shim still
    measures the reference's own code.  The port is given the frame itself, special values included."""
    W, H, D = IC.MAIN
    rng = np.random.default_rng(IC.KINDS.index(kind))
    for v, img in enumerate(IC.frame(kind, W, H, D)):
        img = IC.posterised(img)
        img8 = oracle.to_u8x255(img)
        colours = (img8.astype(np.float32) / np.float32(255)).astype(np.float32)
        assert np.array_equal(oracle.to_u8x255(colours), img8)
        disp = rng.integers(1, D, (H, W)).astype(np.uint8)
        disp[:, ::7] = disp[:, :1]
        got, ncolours = ref.post_process(colours, disp)
        assert ncolours <= 256, ncolours
        assert_same(got, oracle.post_process(img, disp), f"{kind} view {v}: reference JointWMF vs the port's post-filter")


@pytest.mark.parametrize("kind", IC.KINDS)
def test_reference_buildcv_equals_port(kind, ref, oracle):
    W, H, D = IC.MAIN
    l, r = frame(kind, "main")
    with np.errstate(all="ignore"):
        lv, rv = oracle.cost_const(l, r, D)[2:]
        for d in (0, 1, 7, D - 1):
            assert_same(ref.buildcv(l, r, d), lv[d], f"{kind} buildCV_left d = {d}")
            assert_same(ref.buildcv(l, r, d, right=True), rv[d], f"{kind} buildCV_right d = {d}")
