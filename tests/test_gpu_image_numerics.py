"""GPU: every stage that reads a float frame, against its oracle on frames outside [0, 1] (tests/image_cases.py), all
through the C-ABI.

* Every kind, bit for bit: the ingest planes (split channels 0-2, x-gradient 12) under both gray modes; the raw volumes of
  cvc_both_kernel (shipped build and the option-106 builds, with warps on the interior fast path) and of cvc_cost_kernel
  at two non-default matching-cost settings; the guide planes 3-11; the Fast Guided Filter at s = 1, 2, 4, 8; NAIVE.
* Flagged kinds (a negative, -0, inf, NaN or >= 2^61 channel value: the whole view runs in OpenCV's order), bit for bit:
  filtered volumes, a / b and maps under EXACT (three builds), MIXED, the generic window at 3 and 16, a 16-bit context at
  D = 300 whose arg-min exceeds 255, disparity shards reduced through keys.
* Inexact kinds (1.7, 1e10, 8421505, subnormals, (0, 2^-12)): filtered volumes within gif_cases.carried_error_bound,
  with the differing voxel and map-pixel counts printed.
* The post-filter equals the oracle on every kind (maps injected with one-hot cost slices, so the check does not depend
  on the filter's bound), u8 and u16 contexts, the default setting (tuned kernel) and (4, 10, 2, iv2) (param and
  two-level kernels): +inf, 1e10, 8421505 and >= FLT_MAX / 255 channel values quantise to 0, as OpenCV's convertTo does.
* One context switching between flagged, in-domain float and u8 frames, and the device and async upload entry points."""
import ctypes as C

import numpy as np
import pytest

import gif_cases as GC
import image_cases as IC
from gif_cases import assert_same, differ
from oracle import oracle as O
from primestereomatch_b200 import DispEst, capi
from primestereomatch_b200.sharding import shard_range

pytestmark = pytest.mark.gpu

F32 = np.float32
SIZES = {"main": IC.MAIN, "narrow": IC.NARROW, "point": IC.POINT}


def frame(kind, size):
    return IC.wide_frame(kind) if size == "wide" else IC.frame(kind, *SIZES[size])


def dims(size):
    return IC.WIDE if size == "wide" else SIZES[size]


def filtered(l, r, D):
    """the port's raw and filtered volumes (OpenCV's order)"""
    with np.errstate(all="ignore"):
        lg, rg, lraw, rraw = O.cost_const(l, r, D)
        lf, rf = O.cost_filter(l, r, lraw, rraw)
    return (lg, rg), (lraw, rraw), (lf, rf)


def check_maps(de, lf, rf, what, dtype=np.uint8):
    assert de.DispSelect_GPU() == 0
    assert_same(de.lDisMap, O.wta(lf, dtype), f"{what} left map")
    assert_same(de.rDisMap, O.wta(rf, dtype), f"{what} right map")


# ---- every kind: ingest and raw volumes ------------------------------------------------------------------------------------
@pytest.mark.parametrize("gray_mode", [0, 1])
@pytest.mark.parametrize("size", ["main", "narrow", "point"])
@pytest.mark.parametrize("kind", IC.KINDS)
def test_ingest_planes_and_raw_volumes(kind, size, gray_mode):
    l, r = frame(kind, size)
    W, H, D = dims(size)
    with np.errstate(all="ignore"):
        lg, rg, lraw, rraw = O.cost_const(l, r, D, gray_mode=gray_mode)
    builds = (0, 1, 2, 3) if size == "main" else (0,)
    for b in builds:
        with DispEst(l, r, D) as de:
            de.set_option(capi.PSM_OPT_GRAY_MODE, gray_mode)
            de.set_option(106, b)
            assert de.CostConst_GPU() == 0
            what = f"{kind} {size} gray_mode {gray_mode} CVC build {b}"
            for v, img, g in ((0, l, lg), (1, r, rg)):
                for c in range(3):
                    assert_same(de.read_guide_plane(v, c), np.ascontiguousarray(img[..., c]), f"{what} view {v} plane {c}")
                assert_same(de.read_guide_plane(v, 12), g, f"{what} view {v} x-gradient")
            assert_same(de.read_cost_volume(0), lraw, f"{what} left raw volume")
            assert_same(de.read_cost_volume(1), rraw, f"{what} right raw volume")


@pytest.mark.parametrize("setting", [(0.11, 0.21, 0.008), (1.0, 0.0, np.inf)])
@pytest.mark.parametrize("size", ["main", "narrow"])
@pytest.mark.parametrize("kind", IC.KINDS)
def test_cost_kernel_at_other_settings(kind, size, setting):
    l, r = frame(kind, size)
    W, H, D = dims(size)
    with np.errstate(all="ignore"):
        lv, rv = O.cost_const(l, r, D, alpha=setting[0], tau_color=setting[1], tau_grad=setting[2])[2:]
    with DispEst(l, r, D) as de:
        de.setMatchingCost(*setting)
        assert de.CostConst_GPU() == 0
        assert_same(de.read_cost_volume(0), lv, f"{kind} {size} {setting} left raw volume")
        assert_same(de.read_cost_volume(1), rv, f"{kind} {size} {setting} right raw volume")


@pytest.mark.parametrize("size", ["main", "narrow", "point"])
@pytest.mark.parametrize("kind", IC.KINDS)
def test_guide_planes(kind, size):
    l, r = frame(kind, size)
    W, H, D = dims(size)
    with DispEst(l, r, D) as de:
        assert de.CostConst_GPU() == 0
        for v, img in enumerate((l, r)):
            with np.errstate(all="ignore"):
                _, mean, var = O.cvf_preprocess(img)
            got = np.stack([de.read_guide_plane(v, k) for k in range(3, 12)])
            assert_same(got, np.concatenate([mean, var]), f"{kind} {size} view {v} guide planes")


@pytest.mark.parametrize("s", [1, 2, 4, 8])
@pytest.mark.parametrize("kind", IC.KINDS)
def test_fgf(kind, s):
    """DESIGN.md section 9: the FGF performs the same fp64 operations as the port at any input"""
    l, r = frame(kind, "main")
    W, H, D = IC.MAIN
    with np.errstate(all="ignore"):
        _, _, lraw, rraw = O.cost_const(l, r, D)
        lf, rf = O.cost_filter_fgf(l, r, lraw, rraw, s=s)
    with DispEst(l, r, D) as de:
        de.setSubsampleRate(s)
        assert de.CostConst_GPU() == 0 and de.CostFilter_FGF_GPU() == 0
        assert_same(de.read_cost_volume(0), lf, f"{kind} FGF s = {s} left")
        assert_same(de.read_cost_volume(1), rf, f"{kind} FGF s = {s} right")
        check_maps(de, lf, rf, f"{kind} FGF s = {s}")


@pytest.mark.parametrize("size", ["main", "narrow", "point"])
@pytest.mark.parametrize("kind", IC.KINDS)
def test_naive(kind, size):
    l, r = frame(kind, size)
    W, H, D = dims(size)
    _, _, (lf, rf) = filtered(l, r, D)
    with DispEst(l, r, D) as de:
        de.set_option(capi.PSM_OPT_CVF_MODE, capi.PSM_CVF_NAIVE)
        assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
        assert_same(de.read_cost_volume(0), lf, f"{kind} {size} NAIVE left")
        assert_same(de.read_cost_volume(1), rf, f"{kind} {size} NAIVE right")
        check_maps(de, lf, rf, f"{kind} {size} NAIVE")


# ---- flagged kinds: bit for bit ----------------------------------------------------------------------------------------------
BUILDS = [("shipped", None), ("v9", 9), ("v11", 11)]


@pytest.mark.parametrize("build", BUILDS, ids=[b[0] for b in BUILDS])
@pytest.mark.parametrize("size", ["main", "narrow", "point"])
@pytest.mark.parametrize("kind", IC.FLAGGED)
def test_flagged_exact(kind, size, build):
    l, r = frame(kind, size)
    W, H, D = dims(size)
    _, (lraw, rraw), (lf, rf) = filtered(l, r, D)
    d = min(1, D - 1)
    with np.errstate(all="ignore"):
        rgb, mean, var = O.cvf_preprocess(l)
        _, a, b = O.guided_filter(rgb, mean, var, lraw[d], want_ab=True)
    with DispEst(l, r, D) as de:
        if build[1] is not None:
            de.set_option(capi.PSM_OPT_VARIANT, build[1])
        assert de.CostConst_GPU() == 0
        what = f"{kind} {size} EXACT {build[0]}"
        ga, gb = de.read_ab_slice(0, d)          # of the raw slice: the filter works in place
        assert_same(ga, a, f"{what} a"), assert_same(gb, b, f"{what} b")
        assert de.CostFilter_GPU() == 0
        assert_same(de.read_cost_volume(0), lf, f"{what} left")
        assert_same(de.read_cost_volume(1), rf, f"{what} right")
        check_maps(de, lf, rf, what)


@pytest.mark.parametrize("kind", IC.FLAGGED)
def test_flagged_mixed_is_exact(kind):
    l, r = frame(kind, "main")
    W, H, D = IC.MAIN
    _, _, (lf, rf) = filtered(l, r, D)
    with DispEst(l, r, D) as de:
        de.set_option(capi.PSM_OPT_CVF_MODE, capi.PSM_CVF_MIXED)
        assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
        assert_same(de.read_cost_volume(0), lf, f"{kind} MIXED left")
        assert_same(de.read_cost_volume(1), rf, f"{kind} MIXED right")
        check_maps(de, lf, rf, f"{kind} MIXED")


@pytest.mark.parametrize("window", [3, 16])
@pytest.mark.parametrize("kind", IC.FLAGGED)
def test_flagged_generic_window(kind, window):
    l, r = frame(kind, "main")
    W, H, D = IC.MAIN
    eps = 1e-4
    with np.errstate(all="ignore"):
        _, _, lraw, rraw = O.cost_const(l, r, D)
        want = []
        for img, raw in ((l, lraw), (r, rraw)):
            rgb, mean, var = O.cvf_preprocess(img, window=window)
            want.append(O.guided_filter(rgb, mean, var, raw, window=window, eps=eps))
    with DispEst(l, r, D) as de:
        de.setGuidedFilter(window, eps)
        assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
        assert_same(de.read_cost_volume(0), want[0], f"{kind} window {window} left")
        assert_same(de.read_cost_volume(1), want[1], f"{kind} window {window} right")
        check_maps(de, want[0], want[1], f"{kind} window {window}")


@pytest.mark.parametrize("kind", ["posinf", "nan", "fltmax", "negative"])
def test_flagged_u16_context(kind):
    """D = 300: the left arg-min of the columns that hold the special values is 270"""
    l, r = IC.wide_frame(kind)
    W, H, D = IC.WIDE
    _, _, (lf, rf) = filtered(l, r, D)
    want = O.wta(lf, np.uint16)
    assert int(want.max()) > 255
    with DispEst(l, r, D, map_bits=16) as de:
        assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
        assert_same(de.read_cost_volume(0), lf, f"{kind} u16 left")
        assert_same(de.read_cost_volume(1), rf, f"{kind} u16 right")
        check_maps(de, lf, rf, f"{kind} u16", np.uint16)


@pytest.mark.parametrize("kind", ["posinf", "nan", "huge"])
def test_flagged_shards_reduced_through_keys(kind):
    torch = pytest.importorskip("torch")
    l, r = frame(kind, "main")
    W, H, D = IC.MAIN
    _, _, (lf, rf) = filtered(l, r, D)
    L = capi.lib()
    G = 2
    shards = [DispEst(l, r, D, d_begin=shard_range(D, G, k)[0], d_count=shard_range(D, G, k)[1]) for k in range(G)]
    try:
        keys = torch.empty((2, G, W * H), dtype=torch.int64, device="cuda")
        for k, de in enumerate(shards):
            assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
            capi.check(L.psm_disp_select_keys(de.handle, keys[0, k].data_ptr(), keys[1, k].data_ptr()), de.handle)
            de.sync()
        ld, rd = np.zeros((H, W), np.uint8), np.zeros((H, W), np.uint8)
        de = shards[0]
        capi.check(L.psm_disp_reduce_keys(de.handle, keys[0].data_ptr(), keys[1].data_ptr(), G,
                                          ld.ctypes.data_as(C.c_void_p), W, rd.ctypes.data_as(C.c_void_p), W), de.handle)
        assert_same(ld, O.wta(lf), f"{kind} {G} shards left"), assert_same(rd, O.wta(rf), f"{kind} {G} shards right")
    finally:
        for de in shards:
            de.close()


# ---- inexact kinds: within the carried-error bound --------------------------------------------------------------------------
@pytest.mark.parametrize("kind", IC.INEXACT)
def test_inexact_within_the_carried_error_bound(kind):
    l, r = frame(kind, "main")
    W, H, D = IC.MAIN
    (_, _), (lraw, rraw), (lf, rf) = filtered(l, r, D)
    with DispEst(l, r, D) as de:
        assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
        got = {"lf": de.read_cost_volume(0), "rf": de.read_cost_volume(1)}
        assert de.DispSelect_GPU() == 0
        got["ld"], got["rd"] = de.lDisMap.copy(), de.rDisMap.copy()
    for v, (dev, ref, img, raw) in enumerate(((got["lf"], lf, l, lraw), (got["rf"], rf, r, rraw))):
        with np.errstate(all="ignore"):
            bound = np.stack([GC.carried_error_bound(img, raw[d]) for d in range(D)])
        bad, far = differ(dev, ref), GC.beyond_bound(dev, ref, bound)
        print(f"{kind} view {v}: {int(bad.sum())} of {bad.size} voxels differ")
        assert not far.any(), f"{kind} view {v}: {int(far.sum())} voxels beyond the bound, first at {np.argwhere(far)[0].tolist()}"
    for v, (m, vol) in enumerate(((got["ld"], lf), (got["rd"], rf))):
        print(f"{kind} view {v}: {int(np.count_nonzero(m != O.wta(vol)))} of {m.size} map pixels differ")


# ---- the post-filter --------------------------------------------------------------------------------------------------------
def inject_maps(de, ld, rd):
    """make the context's maps exactly ld / rd with one-hot cost slices"""
    assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
    for d in range(de.maxDis):
        de.write_cost_slice(0, d, (ld != d).astype(F32))
        de.write_cost_slice(1, d, (rd != d).astype(F32))
    assert de.DispSelect_GPU() == 0
    assert_same(de.lDisMap, ld, "injected left"), assert_same(de.rDisMap, rd, "injected right")


PP_SETTINGS = [("default", None), ("r4_iv2", (4, 10.0, 2, "iv2"))]


@pytest.mark.parametrize("setting", PP_SETTINGS, ids=[s[0] for s in PP_SETTINGS])
@pytest.mark.parametrize("map_bits", [8, 16])
@pytest.mark.parametrize("kind", IC.KINDS)
def test_post_filter(kind, map_bits, setting):
    l, r = frame(kind, "main")
    W, H, _ = IC.MAIN
    D = 24 if map_bits == 8 else 300
    dtype = np.uint8 if map_bits == 8 else np.uint16
    rng = np.random.default_rng(IC.KINDS.index(kind) + map_bits)
    ld = rng.integers(1, D, (H, W)).astype(dtype)
    rd = rng.integers(1, D, (H, W)).astype(dtype)
    ld[:, 100:140] = ld[:, 100:101] // 2 + 1                     # smooth bands, so the colour weights decide
    args = () if setting[1] is None else setting[1]
    with DispEst(l, r, D, map_bits=map_bits) as de:
        if setting[1] is not None:
            de.setPostFilter(*args)
        inject_maps(de, ld, rd)
        assert de.PostProcess_GPU() == 0
        assert_same(de.lDisMap, O.post_process(l, ld, *args), f"{kind} u{map_bits} {setting[0]} left post-filtered")
        assert_same(de.rDisMap, O.post_process(r, rd, *args), f"{kind} u{map_bits} {setting[0]} right post-filtered")


# ---- one context, switching frames; the other upload entry points --------------------------------------------------------
def test_frame_switching_resets_the_flags():
    """flagged float -> in-domain float -> u8 -> flagged again in one context: each frame equals the oracle (the
    guide flags and the float-image state are reset per frame)"""
    W, H, D = IC.MAIN
    fl, fr = IC.frame("nan", W, H, D)
    rng = np.random.default_rng(5)
    il = rng.integers(0, 256, (H, W + 3, 3), dtype=np.uint8)
    u8l, u8r = np.ascontiguousarray(il[:, 3:]), np.ascontiguousarray(il[:, :W])
    in_l, in_r = O.u8_to_f32(u8l), O.u8_to_f32(u8r)       # floats in the integer domain: the tuned kernels' order
    fl2, fr2 = IC.frame("fltmax", W, H, D)
    seq = [("nan", (fl, fr), (fl, fr)), ("in-domain", (in_l, in_r), (in_l, in_r)),
           ("u8", (u8l, u8r), (O.u8_to_f32(u8l), O.u8_to_f32(u8r))), ("fltmax", (fl2, fr2), (fl2, fr2)),
           ("in-domain again", (in_l, in_r), (in_l, in_r))]
    with DispEst(fl, fr, D) as de:
        for name, dev, (l, r) in seq:
            de.setInputImages(*dev)
            _, _, (lf, rf) = filtered(l, r, D)
            assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
            assert_same(de.read_cost_volume(0), lf, f"frame {name} left")
            assert_same(de.read_cost_volume(1), rf, f"frame {name} right")
            check_maps(de, lf, rf, f"frame {name}")
            ld, rd = de.lDisMap.copy(), de.rDisMap.copy()
            assert de.PostProcess_GPU() == 0
            assert_same(de.lDisMap, O.post_process(l, ld), f"frame {name} post-filtered left")


@pytest.mark.parametrize("kind", ["posinf", "nan", "fltmax"])
def test_device_and_async_uploads(kind):
    torch = pytest.importorskip("torch")
    l, r = frame(kind, "main")
    W, H, D = IC.MAIN
    L = capi.lib()
    step = W * 3 * 4
    with DispEst(l, r, D) as de:
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        want = (de.read_cost_volume(0), de.read_cost_volume(1), de.lDisMap.copy(), de.rDisMap.copy())
        _, _, (lf, rf) = filtered(l, r, D)
        assert_same(want[0], lf, f"{kind} psm_set_images left")

        def same(what):
            capi.check(L.psm_cost_const(de.handle), de.handle)
            capi.check(L.psm_cost_filter(de.handle), de.handle)
            assert_same(de.read_cost_volume(0), want[0], f"{kind} {what} left")
            assert_same(de.read_cost_volume(1), want[1], f"{kind} {what} right")
            assert de.DispSelect_GPU() == 0
            assert_same(de.lDisMap, want[2], f"{kind} {what} left map"), assert_same(de.rDisMap, want[3], f"{kind} {what} right map")

        u8l, u8r = GC.to_u8(np.nan_to_num(np.clip(l, 0, 1))), GC.to_u8(np.nan_to_num(np.clip(r, 0, 1)))
        dl, dr = torch.from_numpy(l).cuda(), torch.from_numpy(r).cuda()
        capi.check(L.psm_set_images_u8(de.handle, u8l.ctypes.data_as(C.c_void_p), W * 3, u8r.ctypes.data_as(C.c_void_p), W * 3),
                   de.handle)
        capi.check(L.psm_set_images_device(de.handle, dl.data_ptr(), step, dr.data_ptr(), step), de.handle)
        same("psm_set_images_device")
        pl, pr = torch.from_numpy(l).pin_memory(), torch.from_numpy(r).pin_memory()
        capi.check(L.psm_set_images_u8(de.handle, u8l.ctypes.data_as(C.c_void_p), W * 3, u8r.ctypes.data_as(C.c_void_p), W * 3),
                   de.handle)
        capi.check(L.psm_set_images_async(de.handle, pl.data_ptr(), step, pr.data_ptr(), step), de.handle)
        capi.check(L.psm_set_images_commit(de.handle), de.handle)
        same("psm_set_images_async + commit")
