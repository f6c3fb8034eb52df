"""GPU: the full-resolution guided filter (psm_cost_filter: the tuned streaming kernel, the generic-window kernel, NAIVE,
MIXED) against its oracle where the fp64 box sums are not exact, so that OpenCV's running-sum order matters: +inf, -inf
and NaN costs, 1e30 costs, mixed signs with -0.0, ties (tests/gif_cases.py puts the special voxels on the seams of the
streaming filter's decomposition), guide images with a near-black float background and with NaN / inf pixels.

* Slices written with a negative, -0, inf, NaN or >= 2^63 cost are flagged by psm_write_cost_slice and filtered again in
  OpenCV's order; guides outside {0} U [2^-12, 1] are precomputed in OpenCV's order, and images outside the integer
  domain send the whole view through that order: there the volumes, the guide planes, a, b and both maps equal the
  oracle bit for bit (NaN at the same voxels, any payload), under every build and plan.  The cost kinds use the dark pair
  as 8-bit images as the guide, so that the slices without a special value stay in the exact-sum domain.
* Finite costs whose fp64 sums are not exact (a 1e15 band above costs near 1e-3, |N| exp(U(-40, 10)), costs under the
  near-black float guide) are filtered in the tuned kernels' order; the test prints how many voxels and map pixels differ
  from the oracle and asserts, per voxel, the bound that the fp64 rounding carried by the running sums allows
  (gif_cases.carried_error_bound)."""
import numpy as np
import pytest

from primestereomatch_b200 import DispEst, capi
from oracle import oracle as O
import gif_cases as GC
from gif_cases import assert_same, differ
import mixed_model as MM

pytestmark = pytest.mark.gpu

F32 = np.float32
D = 5


def reference(img, vol, window=8, eps=1e-4, want_ab=False):
    """filtered copy of one view's raw volume (and a, b of every slice)"""
    rgb, mean, var = O.cvf_preprocess(img, window=window)
    res = O.guided_filter(rgb, mean, var, vol, want_ab=want_ab, window=window, eps=eps)
    if want_ab:
        return res[0], list(zip(res[1], res[2]))
    return res


def run(imgs, Dn, writes=(), mode=None, variant=None, options=(), window=None, eps=1e-4, d_begin=0, map_bits=None,
        ab_slices=()):
    out = {}
    l, r = imgs
    with DispEst(l, r, Dn, d_begin=d_begin, map_bits=map_bits) as de:
        if window is not None:
            de.setGuidedFilter(window, eps)
        if mode is not None:
            de.set_option(capi.PSM_OPT_CVF_MODE, mode)
        if variant is not None:
            de.set_option(capi.PSM_OPT_VARIANT, variant)
        for k, v in options:
            de.set_option(k, v)
        de.CostConst_GPU()
        for v, d, sl in writes:
            de.write_cost_slice(v, d, sl)
        out["ab"] = {(v, d): de.read_ab_slice(v, d) for v, d in ab_slices}
        out["guide"] = [np.stack([de.read_guide_plane(v, k) for k in range(3, 12)]) for v in (0, 1)]
        assert de.CostFilter_GPU() == 0
        out["lf"], out["rf"] = de.read_cost_volume(0), de.read_cost_volume(1)
        if d_begin == 0:
            de.DispSelect_GPU()
            out["ld"], out["rd"] = de.lDisMap.copy(), de.rDisMap.copy()
    return out


def all_slices(lraw, rraw, d_begin=0):
    return [(v, d, vol[d]) for v, vol in enumerate((lraw, rraw)) for d in range(d_begin, vol.shape[0])]


def check(got, lf, rf, what, d_begin=0, map_dtype=np.uint8):
    assert_same(got["lf"], lf[d_begin:], f"{what} left volume")
    assert_same(got["rf"], rf[d_begin:], f"{what} right volume")
    if "ld" in got:
        assert_same(got["ld"], O.wta(lf, map_dtype), f"{what} left map")
        assert_same(got["rd"], O.wta(rf, map_dtype), f"{what} right map")


@pytest.fixture(scope="module")
def dark():
    return GC.dark_pair(GC.W, GC.H, seed=11)


@pytest.fixture(scope="module")
def dark8():
    """the dark pair as 8-bit images read back as floats: a guide in the u8 domain, so that only the special voxels make
    the sums inexact (the float dark pair makes the I p sums inexact in every slice, at the larger windows visibly)"""
    l, r = GC.dark_pair(GC.W, GC.H, seed=11)
    return O.u8_to_f32(GC.to_u8(l)), O.u8_to_f32(GC.to_u8(r))


def raw(kind):
    return GC.costs(kind, D, seed=1), GC.costs(kind, D, seed=2)


# ---- the tuned EXACT kernel under its builds and plans ----------------------------------------------------------------
PLANS = [("v0", 0, ()), ("v9", 9, ()), ("v11", 11, ()), ("rows24", 0, ((101, GC.FORCED_ROWS),)), ("threads64", 0, ((103, 64),)),
         ("remap", 0, ((104, 1),)), ("nopack", 0, ((105, 1),))]


@pytest.mark.parametrize("plan", PLANS, ids=[p[0] for p in PLANS])
@pytest.mark.parametrize("kind", GC.EXACT_KINDS)
def test_exact_kernel_equals_oracle(kind, plan, dark8):
    _, variant, options = plan
    l, r = dark8
    lraw, rraw = raw(kind)
    got = run(dark8, D, all_slices(lraw, rraw), variant=variant, options=options, ab_slices=[(0, 1), (1, D - 1)])
    lf, lab = reference(l, lraw, want_ab=True)
    rf, rab = reference(r, rraw, want_ab=True)
    check(got, lf, rf, f"{kind} {plan[0]}")
    for (v, d), ab in (((0, 1), lab[1]), ((1, D - 1), rab[D - 1])):
        a, b = got["ab"][(v, d)]
        assert_same(a, ab[0], f"{kind} a view {v} slice {d}"), assert_same(b, ab[1], f"{kind} b view {v} slice {d}")


@pytest.mark.parametrize("kind", GC.EXACT_KINDS)
def test_naive_equals_oracle(kind, dark):
    """NAIVE runs OpenCV's order everywhere: bit for bit even with the float dark guide, whose I p sums are not exact"""
    l, r = dark
    lraw, rraw = raw(kind)
    got = run(dark, D, all_slices(lraw, rraw), mode=capi.PSM_CVF_NAIVE)
    check(got, reference(l, lraw), reference(r, rraw), f"NAIVE {kind}")


@pytest.mark.parametrize("window,eps", [(3, 1e-4), (8, 1e-3), (16, 1e-4), (32, 1e-4)])
@pytest.mark.parametrize("kind", ["posinf", "nan", "outlier", "mixed"])
def test_generic_window_equals_oracle(kind, window, eps, dark8):
    l, r = dark8
    lraw, rraw = raw(kind)
    got = run(dark8, D, all_slices(lraw, rraw), window=window, eps=eps, ab_slices=[(1, D - 1)])
    lf = reference(l, lraw, window, eps)
    rf, ab = reference(r, rraw, window, eps, want_ab=True)
    check(got, lf, rf, f"window {window} {kind}")
    a, b = got["ab"][(1, D - 1)]
    assert_same(a, ab[D - 1][0], f"window {window} {kind} a"), assert_same(b, ab[D - 1][1], f"window {window} {kind} b")


# ---- MIXED: flagged slices take the exact reference-order pass; the rest follows mixed_model -----------------------
@pytest.mark.parametrize("kind", GC.EXACT_KINDS)
def test_mixed(kind, dark8):
    """A slice with a negative, -0, inf, NaN or >= 2^63 cost is filtered in the exact reference order; every other slice
    is MIXED's second stage (mixed_model)."""
    l, r = dark8
    lraw, rraw = raw(kind)
    got = run(dark8, D, all_slices(lraw, rraw), mode=capi.PSM_CVF_MIXED)
    nflagged = 0
    for v, (dev, img, rawv) in enumerate(((got["lf"], l, lraw), (got["rf"], r, rraw))):
        mixed, exact = MM.cost_filter_mixed(O, img, rawv), reference(img, rawv)
        for d in range(D):
            special = bool(np.any(rawv[d].view(np.uint32) >= 0x5f000000))
            nflagged += special
            assert_same(dev[d], exact[d] if special else mixed[d],
                        f"MIXED {kind} view {v} slice {d} ({'exact' if special else 'mixed model'})")
    assert nflagged == (0 if kind == "ties" else 2 * D if kind == "mixed" else 4)


# ---- guide images outside the u8 domain ----------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [capi.PSM_CVF_EXACT, capi.PSM_CVF_NAIVE])
@pytest.mark.parametrize("kind", GC.IMAGE_KINDS)
def test_images(kind, mode):
    dev, (l, r) = GC.images(kind)
    Dn = 8
    with np.errstate(all="ignore"):
        _, _, lraw, rraw = O.cost_const(l, r, Dn)
    got = run(dev, Dn, mode=mode, ab_slices=[(0, 3)])
    for v, img in enumerate((l, r)):
        with np.errstate(all="ignore"):
            _, mean, var = O.cvf_preprocess(img)
        assert_same(got["guide"][v], np.concatenate([mean, var]), f"{kind} guide planes view {v}")
    lf, ab = reference(l, lraw, want_ab=True)
    rf = reference(r, rraw)
    a, b = got["ab"][(0, 3)]
    assert_same(a, ab[3][0], f"{kind} a"), assert_same(b, ab[3][1], f"{kind} b")
    if kind == "dark_f32" and mode == capi.PSM_CVF_EXACT:
        # the guide is recomputed in OpenCV's order, but the stage-1 sums of I p (I near 1e-7, p near 1e-3) are not exact
        # and keep the tuned order: the bound applies
        check_bounded(got, (l, r), (lraw, rraw), lf, rf, f"{kind}")
    else:
        check(got, lf, rf, f"{kind} mode {mode}")


# ---- contexts: a disparity shard, 16-bit maps ---------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["posinf", "outlier"])
def test_sharded_context(kind, dark8):
    l, r = dark8
    Dn, d_begin = 9, 4
    lraw, rraw = GC.costs(kind, Dn, seed=3), GC.costs(kind, Dn, seed=4)   # special voxels at d = 1 and 8
    got = run(dark8, Dn, all_slices(lraw, rraw, d_begin), d_begin=d_begin)
    check(got, reference(l, lraw), reference(r, rraw), f"shard {kind}", d_begin=d_begin)


def test_u16_context(dark8):
    l, r = dark8
    Dn = 300
    _, _, lraw, rraw = O.cost_const(l, r, Dn)
    writes = []
    for v, vol in enumerate((lraw, rraw)):
        vol[280] = vol[5] * F32(0.5)
        vol[299] = GC.costs("nan", 5, seed=v)[1]
        vol[290] = GC.costs("outlier", 5, seed=v)[4]
        writes += [(v, d, vol[d]) for d in (280, 290, 299)]
    got = run(dark8, Dn, writes, map_bits=16)
    check(got, reference(l, lraw), reference(r, rraw), "u16 D=300", map_dtype=np.uint16)


# ---- finite costs whose fp64 sums are not exact ------------------------------------------------------------------------
def check_bounded(got, imgs, raws, lf, rf, what):
    """every voxel within gif_cases.carried_error_bound of the oracle (NaN at the same voxels); prints the counts"""
    for v, (dev, ref) in enumerate(((got["lf"], lf), (got["rf"], rf))):
        bound = np.stack([GC.carried_error_bound(imgs[v], raws[v][d]) for d in range(ref.shape[0])])
        bad, far = differ(dev, ref), GC.beyond_bound(dev, ref, bound)
        with np.errstate(all="ignore"):
            ratio = np.where(bad & np.isfinite(ref), np.abs(dev.astype(np.float64) - ref) / bound, 0)
        print(f"{what} view {v}: {int(bad.sum())} of {bad.size} voxels differ, largest error / bound {ratio.max():.3g}")
        assert not far.any(), (f"{what} view {v}: {int(far.sum())} voxels beyond the carried-error bound, first at "
                               f"{np.argwhere(far)[0].tolist()}")
    for v, (m, vol) in enumerate(((got["ld"], lf), (got["rd"], rf))):
        print(f"{what} view {v}: {int(np.count_nonzero(m != O.wta(vol)))} of {m.size} map pixels differ")


@pytest.mark.parametrize("plan", PLANS[:4], ids=[p[0] for p in PLANS[:4]])
@pytest.mark.parametrize("kind", GC.INEXACT_KINDS)
def test_inexact_costs_stay_within_the_carried_error_bound(kind, plan, dark):
    _, variant, options = plan
    l, r = dark
    lraw, rraw = raw(kind)
    got = run(dark, D, all_slices(lraw, rraw), variant=variant, options=options)
    check_bounded(got, dark, (lraw, rraw), reference(l, lraw), reference(r, rraw), f"{kind} {plan[0]}")
