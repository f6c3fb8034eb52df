"""GPU: the Fast Guided Filter (psm_cost_filter_fgf) bit for bit against the C oracle's orc_cost_filter_fgf at the
context's window and eps, where the fp64 box sums are not exact: costs
over wide ranges, a 1e30 outlier, +inf / -inf / NaN voxels, mixed signs and -0.0, exact ties between slices, a guide with
a near-black background (float and 8-bit), low-resolution sizes at and around the 32 x 16 tile edges and below half the
box, the largest box the kernel accepts, a sharded context and a 16-bit-map context at D > 256.  Filtered volumes are
compared bit for bit (NaN at the same voxels, any NaN payload), disparity maps exactly."""
import numpy as np
import pytest

from primestereomatch_b200 import DispEst, capi
from oracle import oracle as O
import fgf_cases as FC
from fgf_cases import assert_same

pytestmark = pytest.mark.gpu

F32 = np.float32
RATES = [1, 2, 4, 8]


def reference(l, r, lraw, rraw, s, window=8, eps=1e-4):
    """filtered copies of both raw volumes; float guide images"""
    return O.cost_filter_fgf(l, r, lraw, rraw, s, window=window, eps=eps)


def run(l, r, D, s, writes=(), window=None, eps=1e-4, d_begin=0, map_bits=None):
    """CostConst, then the raw slices in `writes` ((view, d, slice) triples), then the FGF and, for an unsharded context,
    the WTA -> dict of results"""
    out = {}
    with DispEst(l, r, D, d_begin=d_begin, map_bits=map_bits) as de:
        if window is not None:
            de.setGuidedFilter(window, eps)
        de.setSubsampleRate(s)
        de.CostConst_GPU()
        for v, d, sl in writes:
            de.write_cost_slice(v, d, sl)
        assert de.CostFilter_FGF_GPU() == 0
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


# ---- costs outside the bounded case ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dark():
    return FC.dark_pair(280, 136, seed=11)


@pytest.mark.parametrize("s", RATES)
@pytest.mark.parametrize("kind", FC.COST_KINDS)
def test_extreme_costs(kind, s, dark):
    """280 x 136 at full resolution: 9 low-res tiles across at s = 1, two at s = 8"""
    l, r = dark
    H, W, _ = l.shape
    D = 5
    lraw, rraw = FC.costs(kind, D, W, H, s, seed=1), FC.costs(kind, D, W, H, s, seed=2)
    got = run(l, r, D, s, all_slices(lraw, rraw))
    lf, rf = reference(l, r, lraw, rraw, s)
    check(got, lf, rf, f"{kind} s={s}")


# ---- guide images: near-black background, float and 8-bit -------------------------------------------------------------
@pytest.mark.parametrize("s", RATES)
@pytest.mark.parametrize("fmt", ["f32", "u8"])
def test_dark_background_images(fmt, s, dark):
    l, r = dark
    D = 16
    if fmt == "u8":
        l8, r8 = FC.to_u8(l), FC.to_u8(r)
        l, r = O.u8_to_f32(l8), O.u8_to_f32(r8)
        dl, dr = l8, r8
    else:
        dl, dr = l, r
    _, _, lraw, rraw = O.cost_const(l, r, D)
    got = run(dl, dr, D, s)
    lf, rf = reference(l, r, lraw, rraw, s)
    check(got, lf, rf, f"{fmt} dark pair s={s}")


# ---- geometry -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,H,s", FC.GEOMETRY)
def test_geometry(W, H, s):
    l, r = FC.dark_pair(W, H, seed=W * 131 + H)
    D = 4
    lraw, rraw = FC.costs("wide40", D, W, H, s, seed=W), FC.costs("wide40", D, W, H, s, seed=H)
    got = run(l, r, D, s, all_slices(lraw, rraw))
    lf, rf = reference(l, r, lraw, rraw, s)
    check(got, lf, rf, f"{W}x{H} s={s}")


@pytest.mark.parametrize("kind", ["wide40", "outlier", "nan", "ties"])
def test_window_giving_a_one_tap_box(kind):
    """window 3 at s = 4: K = 2 * (3 / 4) + 1 = 1, the box is the identity"""
    l, r = FC.dark_pair(150, 70, seed=5)
    D = 5
    lraw, rraw = FC.costs(kind, D, 150, 70, 4, seed=3), FC.costs(kind, D, 150, 70, 4, seed=4)
    got = run(l, r, D, 4, all_slices(lraw, rraw), window=3, eps=1e-3)
    lf, rf = reference(l, r, lraw, rraw, 4, 3, 1e-3)
    check(got, lf, rf, f"window 3 s=4 {kind}")


def test_largest_box_at_full_rate():
    """At s = 1 the box is 2 * window + 1 wide and the kernel's shared memory bounds it: find the largest window the call
    accepts (every larger one is refused with PSM_EINVAL and runs nothing), and check that one against the restatement."""
    l, r = FC.dark_pair(90, 40, seed=8)
    H, W, _ = l.shape
    D = 4
    lraw, rraw = FC.costs("outlier", D, W, H, 1, seed=6), FC.costs("wide40", D, W, H, 1, seed=7)
    L = capi.lib()
    with DispEst(l, r, D) as de:
        de.CostConst_GPU()
        for v, d, sl in all_slices(lraw, rraw):
            de.write_cost_slice(v, d, sl)
        window = 32
        while True:
            de.setGuidedFilter(window, 1e-4)
            n = de.launch_count()
            rc = L.psm_cost_filter_fgf(de.handle, 1)
            if rc == capi.PSM_OK:
                break
            assert rc == capi.PSM_EINVAL and b"shared memory" in L.psm_last_error(de.handle), window
            assert de.launch_count() == n
            window -= 1
        assert window >= 8, "the default window must run at s = 1"
        got = {"lf": de.read_cost_volume(0), "rf": de.read_cost_volume(1)}
    lf, rf = reference(l, r, lraw, rraw, 1, window, 1e-4)
    check(got, lf, rf, f"largest window {window} (K = {2 * window + 1}) at s=1")


# ---- contexts: a disparity shard, 16-bit maps at D > 256 ---------------------------------------------------------------
@pytest.mark.parametrize("s", [2, 4])
@pytest.mark.parametrize("kind", ["outlier", "posinf"])
def test_sharded_context(kind, s):
    l, r = FC.dark_pair(150, 70, seed=9)
    D, d_begin = 9, 4
    lraw, rraw = FC.costs(kind, D, 150, 70, s, seed=10), FC.costs(kind, D, 150, 70, s, seed=12)   # special voxels at d = 1, 8
    got = run(l, r, D, s, all_slices(lraw, rraw, d_begin), d_begin=d_begin)
    lf, rf = reference(l, r, lraw, rraw, s)
    check(got, lf, rf, f"shard [{d_begin}, {D}) {kind} s={s}", d_begin=d_begin)


def test_u16_context_above_256():
    l, r = FC.dark_pair(48, 24, seed=14)
    H, W, _ = l.shape
    D = 300
    _, _, lraw, rraw = O.cost_const(l, r, D)
    writes = []
    for v, vol in enumerate((lraw, rraw)):
        vol[280] = vol[5] * F32(0.5)         # the minimum lands above 255 ...
        vol[290] = vol[280]                  # ... with an exact tie further up
        vol[299] = FC.costs("wide40", 4, W, H, 4, seed=v)[1]
        writes += [(v, d, vol[d]) for d in (280, 290, 299)]
    got = run(l, r, D, 4, writes, map_bits=16)
    lf, rf = reference(l, r, lraw, rraw, 4)
    check(got, lf, rf, "u16 D=300 s=4", map_dtype=np.uint16)
    assert got["ld"].max() >= 280
