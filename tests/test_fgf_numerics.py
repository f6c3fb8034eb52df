"""CPU: the box filters of the C oracle where fp64 sums are not exact.

* box (orc_box) restates cv::boxFilter in OpenCV's own order (direct row sums up to K = 5, sliding above, sliding
  column sums): it equals cv2 with IPP off at every K on data where the orders differ (values over 50 binary orders of
  magnitude, 1e30 outliers, near-denormal values with O(1) spikes).
* box_direct (orc_box_k), the Fast Guided Filter's box, is defined as the direct order; it equals cv2.blur when every
  fp64 sum is exact, and the test builds data that meets that condition at every box the FGF can use.
"""
import math

import numpy as np
import pytest

from fgf_cases import assert_same, differ

F32 = np.float32
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


@pytest.mark.parametrize("K", range(1, 33))
def test_box_matches_cv2_box_filter_beyond_exact_sums(K, oracle, cv2):
    rng = np.random.default_rng(100 + K)
    for kind in KINDS:
        for h, w in ((45, 70), tuple(int(x) for x in rng.integers(1, 2 * K + 20, 2)), (max(1, K // 2), max(1, K // 3))):
            p = image(kind, h, w, rng)
            assert_same(oracle.box(p, K), cv2.boxFilter(p, -1, (K, K)), f"box K={K} {kind} {h}x{w}")


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
        assert_same(oracle.box_direct(p, K), cv2.blur(p, (K, K)), f"box_direct K={K} {h}x{w}")


def test_box_direct_is_not_cv2_blur_beyond_exact_sums(oracle, cv2):
    """the direct order is the FGF's own definition: on wide-range data cv2.blur (= box) differs from it"""
    rng = np.random.default_rng(0)
    p = image("exp40", 45, 70, rng)
    blur = cv2.blur(p, (3, 3))
    assert_same(oracle.box(p, 3), blur, "box K=3")
    assert np.count_nonzero(differ(oracle.box_direct(p, 3), blur)) > 0
