"""CPU: the box filters of the CPU references where fp64 sums are not exact, and the two Fast Guided Filter references
against each other on the inputs of test_gpu_fgf_numerics.py.

* window_oracle.box restates cv::boxFilter in OpenCV's own order (direct row sums up to K = 5, sliding above, sliding
  column sums) and orc_box8 does so at K = 8: both equal cv2 with IPP off on data where the orders differ (values over
  50 binary orders of magnitude, 1e30 outliers, near-denormal values with O(1) spikes).
* box_direct / orc_box_k, the Fast Guided Filter's box, is defined as the direct order; it equals cv2.blur when every
  fp64 sum is exact, and the test builds data that meets that condition at every box the FGF can use.
* orc_cost_filter_fgf (C) equals window_oracle.fgf_filter_volume (numpy) on wide-range, outlier, non-finite, signed-zero
  and tied costs, so the two references the device is compared with agree with each other.
"""
import ctypes as C
import math

import numpy as np
import pytest

import fgf_cases as FC
from fgf_cases import assert_same, differ
import window_oracle as WO

F32 = np.float32
RATES = [1, 2, 4, 8]
KINDS = ["exp40", "outlier", "denormal"]


@pytest.fixture(scope="module")
def cv2():
    """cv2 with IPP off (IPP's box filter sums in its own order), restored afterwards"""
    cv2 = pytest.importorskip("cv2")
    prev = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield cv2
    cv2.ipp.setUseIPP(prev)


def image(kind, h, w, rng):
    if kind == "exp40":
        return (np.abs(rng.standard_normal((h, w))) * np.exp(rng.uniform(-40, 10, (h, w)))).astype(F32)
    if kind == "outlier":
        p = (rng.random((h, w)) + 0.5).astype(F32)
        p[rng.random((h, w)) < 0.02] = 1e30
        return p
    p = (rng.standard_normal((h, w)) * 1e-38).astype(F32)    # normal and subnormal values near the bottom of the range
    p[rng.random((h, w)) < 0.05] = 3.0
    return p


def orc_box_k(oracle, p, K):
    L = oracle.lib()
    L.orc_box_k.argtypes = [np.ctypeslib.ndpointer(np.float32, flags="C"), C.c_int, C.c_int, C.c_int,
                            np.ctypeslib.ndpointer(np.float32, flags="C")]
    p = np.ascontiguousarray(p, F32)
    out = np.empty_like(p)
    L.orc_box_k(p, p.shape[1], p.shape[0], K, out)
    return out


@pytest.mark.parametrize("K", range(1, 33))
def test_box_matches_cv2_box_filter_beyond_exact_sums(K, cv2):
    rng = np.random.default_rng(100 + K)
    for kind in KINDS:
        for h, w in ((45, 70), tuple(int(x) for x in rng.integers(1, 2 * K + 20, 2)), (max(1, K // 2), max(1, K // 3))):
            p = image(kind, h, w, rng)
            assert_same(WO.box(p, K), cv2.boxFilter(p, -1, (K, K)), f"box K={K} {kind} {h}x{w}")


def test_orc_box8_matches_cv2_box_filter_beyond_exact_sums(oracle, cv2):
    rng = np.random.default_rng(8)
    for kind in KINDS:
        for h, w in ((45, 70), (9, 13), (3, 5), (120, 31)):
            p = image(kind, h, w, rng)
            assert_same(oracle.box8(p), cv2.boxFilter(p, -1, (8, 8)), f"orc_box8 {kind} {h}x{w}")


def exact_span_image(K, h, w, rng):
    """values that are integer multiples of 2^q with magnitude below 2^Q, Q - q = 53 - ceil(log2(K*K)), with exponents
    spread over the whole span (the condition under which every fp64 sum of either order is exact); zeros included"""
    span = 53 - math.ceil(math.log2(K * K)) if K > 1 else 53
    q = int(rng.integers(-100, 60))
    m = rng.integers(-(1 << 24) + 1, 1 << 24, (h, w)).astype(np.float64)          # 24-bit integers: exact in float32
    e = rng.integers(0, span - 24 + 1, (h, w))                                       # |m * 2^e| < 2^(24 + e) <= 2^span
    e[0, 0], e[-1, -1] = 0, span - 24                                                # both ends of the span present
    p = np.ldexp(m, e + q).astype(F32)
    p[rng.random((h, w)) < 0.05] = 0
    assert np.array_equal(p.astype(np.float64), np.ldexp(m, e + q) * (p != 0))
    return p


@pytest.mark.parametrize("K", range(1, 66, 2))
def test_box_direct_equals_cv2_blur_where_sums_are_exact(K, oracle, cv2):
    """every odd box 1 .. 65 (K = 2 * (window / s) + 1 for window 1 .. 32)"""
    rng = np.random.default_rng(K)
    for h, w in ((40, 57), (K + 3, 2 * K + 1), (max(1, K // 2), max(1, K // 3 + 1))):
        p = exact_span_image(K, h, w, rng)
        direct = WO.box_direct(p, K)
        assert_same(direct, cv2.blur(p, (K, K)), f"box_direct K={K} {h}x{w}")
        assert_same(orc_box_k(oracle, p, K), direct, f"orc_box_k K={K} {h}x{w}")


def test_box_direct_is_not_cv2_blur_beyond_exact_sums(cv2):
    """the direct order is the FGF's own definition: on wide-range data cv2.blur (= box) differs from it"""
    rng = np.random.default_rng(0)
    p = image("exp40", 45, 70, rng)
    blur = cv2.blur(p, (3, 3))
    assert_same(WO.box(p, 3), blur, "box K=3")
    assert np.count_nonzero(differ(WO.box_direct(p, 3), blur)) > 0


@pytest.mark.parametrize("K", [1, 3, 5, 9, 17, 19, 33])
def test_orc_box_k_is_the_direct_order_at_any_input(K, oracle):
    rng = np.random.default_rng(K)
    for kind in KINDS + ["nonfinite"]:
        if kind == "nonfinite":
            p = rng.standard_normal((37, 50)).astype(F32)
            p[5, 7], p[20, 1], p[30, 44], p[0, 0] = np.inf, -np.inf, np.nan, -0.0
        else:
            p = image(kind, 37, 50, rng)
        with np.errstate(invalid="ignore"):
            assert_same(orc_box_k(oracle, p, K), WO.box_direct(p, K), f"K={K} {kind}")


# ---- the two FGF references agree on the GPU tests' inputs -----------------------------------------------------------
def both_references(oracle, l, lraw, s):
    c = oracle.cost_filter_fgf(l, l, lraw, lraw, s=s)[0]
    with np.errstate(all="ignore"):
        n = WO.fgf_filter_volume(l, lraw, 8, 1e-4, s)
    return c, n


@pytest.mark.parametrize("s", RATES)
@pytest.mark.parametrize("kind", FC.COST_KINDS)
def test_port_equals_restatement_on_extreme_costs(kind, s, oracle):
    l, _ = FC.dark_pair(280, 136, seed=11)
    c, n = both_references(oracle, l, FC.costs(kind, 5, 280, 136, s, seed=1), s)
    assert_same(c, n, f"{kind} s={s}")


@pytest.mark.parametrize("s", RATES)
def test_port_equals_restatement_on_dark_images(s, oracle):
    l, r = FC.dark_pair(280, 136, seed=11)
    for img in (l, oracle.u8_to_f32(FC.to_u8(l))):
        lraw = oracle.cost_const(img, np.ascontiguousarray(np.roll(img, -2, axis=1)), 6)[2]
        c, n = both_references(oracle, img, lraw, s)
        assert_same(c, n, f"dark pair s={s}")


@pytest.mark.parametrize("W,H,s", FC.GEOMETRY)
def test_port_equals_restatement_on_small_and_tile_edge_sizes(W, H, s, oracle):
    l, _ = FC.dark_pair(W, H, seed=W * 131 + H)
    c, n = both_references(oracle, l, FC.costs("outlier", 4, W, H, s, seed=W), s)
    assert_same(c, n, f"{W}x{H} s={s}")
