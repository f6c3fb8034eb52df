"""GPU: the matching cost at run-time alpha and truncation thresholds (psm_set_matching_cost), bit-exact against the
any-setting CPU restatement tests/cost_oracle.py (which reproduces the existing goldens at the defaults and the
cv2-driven golden_cost.json at the other settings).  Every comparison goes through the C-ABI."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, read_png
from primestereomatch_b200 import DispEst, capi
import cost_oracle as CO
import mixed_model as MM
import window_oracle as WO

pytestmark = pytest.mark.gpu

INF = float("inf")
SETTINGS = [(0.9, 0.028, 0.008), (0.11, 0.21, 0.008), (0.0, INF, INF), (1.0, INF, INF), (0.5, 0.0, 0.03),
            (0.9, 0.0, 0.0), (0.25, INF, 0.004), (0.75, 0.3, INF)]
BEST = (0.11, 0.21, 0.008)


def assert_same(a, b, what):
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {a.size} differ, first at {list(i)}: {a[i]!r} vs {b[i]!r}")


def run(l, r, D, cost, d_begin=0, d_count=None, window=None, filt=True):
    """CostConst at `cost` (None: never call psm_set_matching_cost) -> raw volumes, then CostFilter -> WTA."""
    out = {}
    with DispEst(l, r, D, d_begin=d_begin, d_count=d_count) as de:
        if cost is not None:
            assert de.setMatchingCost(*cost) == 0
        if window is not None:
            de.setGuidedFilter(*window)
        n = de.launch_count()
        assert de.CostConst_GPU() == 0
        out["cvc_launches"] = de.launch_count() - n
        out["lraw"], out["rraw"] = de.read_cost_volume(0), de.read_cost_volume(1)
        if filt:
            assert de.CostFilter_GPU() == 0
            out["lf"], out["rf"] = de.read_cost_volume(0), de.read_cost_volume(1)
            if d_count is None:
                de.DispSelect_GPU()
                out["ld"], out["rd"] = de.lDisMap.copy(), de.rDisMap.copy()
    return out


def check_raw(l, r, D, cost, got, what, d_begin=0, d_count=None):
    lraw, rraw = CO.cost_volumes(l, r, D, *(cost or CO.DEFAULT), d_begin=d_begin, d_count=d_count)
    assert_same(got["lraw"], lraw, f"{what} left raw volume")
    assert_same(got["rraw"], rraw, f"{what} right raw volume")
    return lraw, rraw


def bad_pixels_nonocc(ld, gt, occl):
    """StereoMatch.cpp:275-311 at D = 64 (scale 4, first 65 columns cleared, THRESH_TOZERO at 4, occlusion mask / 255)."""
    disp = np.minimum(ld.astype(np.int32) * 4, 255)
    e = np.abs(disp - gt.astype(np.int32))
    e[:, :65] = 0
    e = np.where(e > 4, e, 0)
    v = np.rint(e.astype(np.float64) * occl.astype(np.float64) / 255.0)
    return float(np.count_nonzero(v)) * 100.0 / gt.size


@pytest.fixture(scope="module")
def crops(scenes):
    """96 x 160 crops of both scenes (x from 150: the left border columns x < d are inside the crop)."""
    out = {}
    for name, (_, _, l, r) in scenes.items():
        out[name] = (np.ascontiguousarray(l[100:196, 150:310]), np.ascontiguousarray(r[100:196, 150:310]))
    return out


@pytest.mark.parametrize("cost", SETTINGS)
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_raw_volumes_on_crops(scene, cost, crops):
    l, r = crops[scene]
    got = run(l, r, 24, cost)
    lraw, rraw = check_raw(l, r, 24, cost, got, f"{scene} crop {cost}")
    lf, rf = WO.cost_filter(l, r, lraw, rraw)
    assert_same(got["lf"], lf, f"{scene} crop {cost} left filtered")
    assert_same(got["rf"], rf, f"{scene} crop {cost} right filtered")
    assert_same(got["ld"], WO.wta(lf), f"{scene} crop {cost} left map")
    assert_same(got["rd"], WO.wta(rf), f"{scene} crop {cost} right map")


@pytest.mark.parametrize("W,H,D", [(1, 1, 3), (2, 3, 4), (5, 40, 5), (17, 23, 7), (31, 9, 40), (32, 6, 33), (33, 5, 40),
                                   (113, 40, 9), (451, 20, 21)])
def test_ragged_sizes(W, H, D):
    rng = np.random.default_rng(W * 1000 + H)
    l = rng.random((H, W, 3), dtype=np.float32)
    r = np.clip(np.roll(l, -1, axis=1) + rng.normal(0, 0.03, (H, W, 3)), 0, 1).astype(np.float32)
    cost = (0.3, 0.12, 0.01)
    got = run(l, r, D, cost)
    lraw, rraw = check_raw(l, r, D, cost, got, f"{W}x{H}x{D}")
    lf, rf = WO.cost_filter(l, r, lraw, rraw)   # W < 32: the mirrored halo comes from the separate pass
    assert_same(got["lf"], lf, f"{W}x{H}x{D} left filtered")
    assert_same(got["rf"], rf, f"{W}x{H}x{D} right filtered")


@pytest.mark.parametrize("W,H,D,d_begin,d_count", [(130, 24, 40, 7, 9), (130, 24, 40, 8, 13), (1280, 9, 64, 33, 31),
                                                   (253, 12, 256, 128, 128), (253, 12, 256, 0, 256), (66, 10, 7, 4, 3),
                                                   (37, 16, 48, 5, 43)])
def test_shards_and_depth_256(W, H, D, d_begin, d_count):
    rng = np.random.default_rng(W + 31 * D + d_begin)
    l = rng.random((H, W, 3), dtype=np.float32)
    r = np.clip(np.roll(l, -5, axis=1) + rng.normal(0, 0.05, (H, W, 3)), 0, 1).astype(np.float32)
    for cost in ((0.11, 0.21, 0.008), (0.0, 0.5, 0.02)):
        got = run(l, r, D, cost, d_begin=d_begin, d_count=d_count, filt=False)
        check_raw(l, r, D, cost, got, f"{W}x{H}x{D} shard [{d_begin}, +{d_count}) {cost}", d_begin, d_count)


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_full_scene_maps_and_bad_pixels_at_best_setting(scene, scenes):
    with open(os.path.join(GOLDEN, "golden_cost.json")) as f:
        golden = json.load(f)
    name = "a{:g}_tc{:g}_tg{:g}".format(*BEST)
    g = golden["cases"][name][scene]
    _, _, l, r = scenes[scene]
    got = run(l, r, 64, BEST)
    lraw, rraw = check_raw(l, r, 64, BEST, got, f"{scene} {BEST}")
    lf, rf = WO.cost_filter(l, r, lraw, rraw)
    assert_same(got["ld"], WO.wta(lf), f"{scene} left map")
    assert_same(got["rd"], WO.wta(rf), f"{scene} right map")
    s = scene.lower()
    gt, occl = read_png(os.path.join(GOLDEN, f"{s}_disp2.png"), True), read_png(os.path.join(GOLDEN, f"{s}_occl.png"), True)
    assert abs(bad_pixels_nonocc(got["ld"], gt, occl) - g["bp_nonocc_left"]) < 1e-3


def test_non_default_setting_with_default_values_runs_the_new_kernel(crops):
    """alpha 0.9f with tau 1e30 is not the default setting: the parameterised kernel runs and, since no difference of images
    in [0, 1] exceeds 1e30, yields the default volumes bit for bit, with the same number of launches."""
    torch = pytest.importorskip("torch")
    from torch.profiler import ProfilerActivity, profile
    l, r = crops["Cones"]
    base = run(l, r, 24, None, filt=False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        got = run(l, r, 24, (0.9, 1e30, 1e30), filt=False)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert any("cvc_cost_kernel" in n for n in names), "the parameterised CVC kernel did not run"
    assert not any("cvc_both_kernel" in n for n in names)
    assert_same(got["lraw"], base["lraw"], "left raw volume at (0.9, 1e30, 1e30)")
    assert_same(got["rraw"], base["rraw"], "right raw volume at (0.9, 1e30, 1e30)")
    assert got["cvc_launches"] == base["cvc_launches"]


def test_with_window_16(crops):
    l, r = crops["Teddy"]
    got = run(l, r, 24, BEST, window=(16, 1e-4))
    lraw, rraw = check_raw(l, r, 24, BEST, got, "window 16")
    lf, rf = WO.cost_filter(l, r, lraw, rraw, 16, 1e-4)
    assert_same(got["lf"], lf, "window 16 left filtered")
    assert_same(got["rf"], rf, "window 16 right filtered")


def test_with_fgf(scenes):
    _, _, l, r = scenes["Teddy"]
    lraw, rraw = CO.cost_volumes(l, r, 64, *BEST)
    lf, rf = WO.cost_filter_fgf(l, r, lraw, rraw, 8, 1e-4, 4)
    with DispEst(l, r, 64) as de:
        de.setMatchingCost(*BEST)
        de.setSubsampleRate(4)
        de.CostConst_GPU()
        assert de.CostFilter_FGF_GPU() == 0
        assert_same(de.read_cost_volume(0), lf, "FGF s=4 left")
        assert_same(de.read_cost_volume(1), rf, "FGF s=4 right")


@pytest.mark.parametrize("mode", [capi.PSM_CVF_MIXED, capi.PSM_CVF_NAIVE])
def test_with_mixed_and_naive_modes(mode, crops, oracle):
    l, r = crops["Cones"]
    lraw, rraw = CO.cost_volumes(l, r, 24, *BEST)
    with DispEst(l, r, 24) as de:
        de.setMatchingCost(*BEST)
        de.set_option(capi.PSM_OPT_CVF_MODE, mode)
        de.CostConst_GPU()
        de.CostFilter_GPU()
        lf, rf = de.read_cost_volume(0), de.read_cost_volume(1)
    if mode == capi.PSM_CVF_MIXED:
        assert_same(lf, MM.cost_filter_mixed(oracle, l, lraw), "MIXED left vs its CPU model")
        assert_same(rf, MM.cost_filter_mixed(oracle, r, rraw), "MIXED right vs its CPU model")
    else:
        wl, wr = WO.cost_filter(l, r, lraw, rraw)
        assert_same(lf, wl, "NAIVE left")
        assert_same(rf, wr, "NAIVE right")


def test_sharded_keys_match_unsharded(crops):
    torch = pytest.importorskip("torch")
    l, r = crops["Cones"]
    H, W, _ = l.shape
    D = 24
    lraw, rraw = CO.cost_volumes(l, r, D, *BEST)
    lf, rf = WO.cost_filter(l, r, lraw, rraw)
    L = capi.lib()
    keys = torch.empty((2, 2, H * W), dtype=torch.int64, device="cuda")
    shards = [DispEst(l, r, D, d_begin=0, d_count=11), DispEst(l, r, D, d_begin=11, d_count=13)]
    try:
        for rank, de in enumerate(shards):
            de.setMatchingCost(*BEST)
            de.CostConst_GPU(); de.CostFilter_GPU()
            assert_same(de.read_cost_volume(0), lf[de.d_begin:de.d_begin + de.d_count], f"shard {rank} left volume")
            capi.check(L.psm_disp_select_keys(de.handle, keys[0, rank].data_ptr(), keys[1, rank].data_ptr()), de.handle)
            de.sync()
        ld = np.zeros((H, W), np.uint8); rd = np.zeros((H, W), np.uint8)
        de = shards[0]
        capi.check(L.psm_disp_reduce_keys(de.handle, keys[0].data_ptr(), keys[1].data_ptr(), 2,
                                          ld.ctypes.data_as(C.c_void_p), W, rd.ctypes.data_as(C.c_void_p), W), de.handle)
        assert_same(ld, WO.wta(lf), "sharded left map")
        assert_same(rd, WO.wta(rf), "sharded right map")
    finally:
        for de in shards:
            de.close()


def test_switching_settings_between_frames(scenes, oracle_scene_results):
    """defaults, other settings, back to the defaults: today's volumes and maps, and today's launch count every frame."""
    _, _, l, r = scenes["Cones"]
    ref = oracle_scene_results["Cones"]
    with DispEst(l, r, 64) as fresh:
        n0 = fresh.launch_count()
        fresh.CostConst_GPU(); fresh.CostFilter_GPU(); fresh.DispSelect_GPU()
        per_frame = fresh.launch_count() - n0
    with DispEst(l, r, 64) as de:
        for cost in (BEST, (0.9, INF, INF), (0.0, INF, 0.05), (0.9, INF, INF)):
            de.setMatchingCost(*cost)
            n = de.launch_count()
            de.CostConst_GPU()
            raw = de.read_cost_volume(0)
            de.CostFilter_GPU(); de.DispSelect_GPU()
            assert de.launch_count() - n == per_frame, cost
            if cost == (0.9, INF, INF):
                assert_same(raw, ref["lraw"], "back to defaults: left raw volume")
                assert_same(de.lDisMap, ref["ld"], "back to defaults: left map")
                assert_same(de.rDisMap, ref["rd"], "back to defaults: right map")
            else:
                lraw, rraw = CO.cost_volumes(l, r, 64, *cost)
                assert_same(raw, lraw, f"{cost} left raw volume")
                lf, rf = WO.cost_filter(l, r, lraw, rraw)
                assert_same(de.lDisMap, WO.wta(lf), f"{cost} left map")
                assert_same(de.rDisMap, WO.wta(rf), f"{cost} right map")


def test_default_launch_count_unchanged(crops):
    l, r = crops["Teddy"]
    never = run(l, r, 24, None)
    explicit = run(l, r, 24, (0.9, INF, INF))
    other = run(l, r, 24, BEST)
    assert explicit["cvc_launches"] == never["cvc_launches"] == other["cvc_launches"]
    assert_same(explicit["lraw"], never["lraw"], "explicit defaults")
    narrow = np.ascontiguousarray(l[:, :20]), np.ascontiguousarray(r[:, :20])
    assert run(*narrow, 8, None, filt=False)["cvc_launches"] == run(*narrow, 8, BEST, filt=False)["cvc_launches"]


def test_errors_leave_context_unchanged(crops):
    l, r = crops["Teddy"]
    L = capi.lib()
    nan = float("nan")
    with DispEst(l, r, 24) as de:
        assert de.setMatchingCost(*BEST) == 0
        for cost in ((-0.1, INF, INF), (1.01, INF, INF), (nan, INF, INF), (INF, INF, INF), (-INF, INF, INF),
                     (0.5, -1e-6, INF), (0.5, INF, -1.0), (0.5, nan, INF), (0.5, INF, nan), (0.5, -INF, INF)):
            assert L.psm_set_matching_cost(de.handle, *cost) == capi.PSM_EINVAL, cost
            with pytest.raises(capi.PsmError):
                de.setMatchingCost(*cost)
        assert L.psm_set_matching_cost(None, 0.5, 0.1, 0.1) == capi.PSM_EINVAL
        de.CostConst_GPU()
        lraw, rraw = CO.cost_volumes(l, r, 24, *BEST)
        assert_same(de.read_cost_volume(0), lraw, "after rejected calls: the best setting still in force (left)")
        assert_same(de.read_cost_volume(1), rraw, "after rejected calls: right")


def test_cpp_facade_set_matching_cost(tmp_path, scenes, oracle):
    exe = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
    if not os.path.exists(exe):
        pytest.skip("dispest_demo not built")
    _, _, l, r = scenes["Teddy"]
    H, W, _ = l.shape
    l.tofile(tmp_path / "l.f32"); r.tofile(tmp_path / "r.f32")
    out = subprocess.run([exe, str(W), str(H), "64", str(tmp_path / "l.f32"), str(tmp_path / "r.f32"),
                          str(tmp_path / "l.u8"), str(tmp_path / "r.u8"), "8", "0.0001", "0.11", "0.21", "0.008"],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    lraw, rraw = CO.cost_volumes(l, r, 64, *BEST)
    lf, _ = WO.cost_filter(l, r, lraw, rraw)
    ld = np.fromfile(tmp_path / "l.u8", np.uint8).reshape(H, W)
    assert_same(ld, oracle.post_process(l, WO.wta(lf)), "C++ facade lDisMap at the best setting (after PostProcess_GPU)")
