"""GPU: the guided filter at run-time window / epsilon (psm_set_guided_filter), bit-exact against the any-window CPU
restatement tests/window_oracle.py (which reproduces the existing goldens at (8, 1e-4f) and cv2 at the other windows)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from primestereomatch_b200 import DispEst, capi, synth
import window_oracle as WO

pytestmark = pytest.mark.gpu

WINDOWS = [1, 2, 3, 5, 9, 12, 16, 31, 32]
EPSES = [1e-4, 1e-3, 1e-2]


def assert_same(a, b, what):
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {a.size} differ, first at {list(i)}: {a[i]!r} vs {b[i]!r}")


def run(l, r, D, window, eps, raw=None, guide=False, d_begin=0, d_count=None):
    """CostConst (or caller-provided raw volumes) -> CostFilter -> WTA at (window, eps) -> dict of results."""
    out = {}
    with DispEst(l, r, D, d_begin=d_begin, d_count=d_count) as de:
        assert de.setGuidedFilter(window, eps) == 0
        de.CostConst_GPU()
        if raw is not None:
            for v in range(2):
                for d in range(D):
                    de.write_cost_slice(v, d, raw[v][d])
        if guide:
            out["mean"] = np.stack([de.read_guide_plane(0, k) for k in range(3, 6)])
            out["var"] = np.stack([de.read_guide_plane(0, k) for k in range(6, 12)])
        assert de.CostFilter_GPU() == 0
        out["lf"], out["rf"] = de.read_cost_volume(0), de.read_cost_volume(1)
        if d_count is None:
            de.DispSelect_GPU()
            out["ld"], out["rd"] = de.lDisMap.copy(), de.rDisMap.copy()
    return out


def check_against_oracle(l, r, lraw, rraw, window, eps, got, what):
    lf, rf = WO.cost_filter(l, r, lraw, rraw, window, eps)
    if "mean" in got:
        _, mean, var = WO.cvf_preprocess(l, window)
        assert_same(got["mean"], mean, f"{what} mean_I")
        assert_same(got["var"], var, f"{what} var_I")
    assert_same(got["lf"], lf, f"{what} left filtered volume")
    assert_same(got["rf"], rf, f"{what} right filtered volume")
    if "ld" in got:
        assert_same(got["ld"], WO.wta(lf), f"{what} left map")
        assert_same(got["rd"], WO.wta(rf), f"{what} right map")


@pytest.fixture(scope="module")
def crops(scenes, oracle):
    """96 x 160 crops of both scenes, D = 24, raw volumes from the C oracle."""
    out = {}
    for name, (_, _, l, r) in scenes.items():
        lc, rc = np.ascontiguousarray(l[100:196, 150:310]), np.ascontiguousarray(r[100:196, 150:310])
        _, _, lraw, rraw = oracle.cost_const(lc, rc, 24)
        out[name] = (lc, rc, lraw, rraw)
    return out


@pytest.mark.parametrize("eps", EPSES)
@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_window_eps_grid_on_crops(scene, window, eps, crops):
    l, r, lraw, rraw = crops[scene]
    got = run(l, r, 24, window, eps, guide=True)
    check_against_oracle(l, r, lraw, rraw, window, eps, got, f"{scene} crop window {window} eps {eps}")


@pytest.mark.parametrize("window,eps", [(4, 1e-4), (16, 1e-4), (32, 1e-4), (8, 1e-3)])
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_full_scenes(scene, window, eps, scenes, oracle_scene_results):
    _, _, l, r = scenes[scene]
    ref = oracle_scene_results[scene]
    got = run(l, r, 64, window, eps, guide=True)
    check_against_oracle(l, r, ref["lraw"], ref["rraw"], window, eps, got, f"{scene} window {window} eps {eps}")


@pytest.mark.parametrize("W,H,D", [(5, 40, 5), (17, 23, 7), (40, 7, 3), (113, 40, 9), (451, 20, 5), (1, 1, 3), (300, 2, 3)])
@pytest.mark.parametrize("window", [3, 16, 32])
def test_ragged_sizes(W, H, D, window, oracle):
    rng = np.random.default_rng(W * 1000 + H + window)
    l = rng.random((H, W, 3), dtype=np.float32)
    r = np.clip(np.roll(l, -1, axis=1) + rng.normal(0, 0.03, (H, W, 3)), 0, 1).astype(np.float32)
    _, _, lraw, rraw = oracle.cost_const(l, r, D)
    got = run(l, r, D, window, 1e-3, guide=True)
    check_against_oracle(l, r, lraw, rraw, window, 1e-3, got, f"{W}x{H}x{D} window {window}")


@pytest.mark.parametrize("window,eps", [(5, 1e-4), (16, 1e-2), (32, 1e-3)])
def test_read_ab_slice(window, eps, crops):
    l, r, lraw, _ = crops["Teddy"]
    rgb, mean, var = WO.cvf_preprocess(l, window)
    with DispEst(l, r, 24) as de:
        de.setGuidedFilter(window, eps)
        de.CostConst_GPU()
        for d in (1, 13):
            a, b = de.read_ab_slice(0, d)
            _, wa, wb = WO.guided_filter(rgb, mean, var, lraw[d], window, eps, want_ab=True)
            assert_same(a, wa, f"a d={d}")
            assert_same(b, wb, f"b d={d}")


def test_special_values():
    """Negative costs, -0.0 and exact ties, written with psm_write_cost_slice (as test_write_slice_filter_wta_special_values)."""
    rng = np.random.default_rng(11)
    H, W, D = 48, 144, 6
    l = rng.random((H, W, 3), dtype=np.float32)
    vol = rng.normal(0, 1, (D, H, W)).astype(np.float32)
    vol[2, :, :40] = vol[4, :, :40]
    vol[3, 10:20] = -0.0
    for window, eps in ((12, 1e-3), (3, 1e-4)):
        got = run(l, l, D, window, eps, raw=(vol, vol))
        check_against_oracle(l, l, vol, vol, window, eps, got, f"special values window {window}")


def test_sharded_keys_match_unsharded(crops):
    torch = pytest.importorskip("torch")
    l, r, lraw, rraw = crops["Cones"]
    H, W, _ = l.shape
    D, window, eps = 24, 12, 1e-3
    lf, rf = WO.cost_filter(l, r, lraw, rraw, window, eps)
    L = capi.lib()
    keys = torch.empty((2, 2, H * W), dtype=torch.int64, device="cuda")
    shards = [DispEst(l, r, D, d_begin=0, d_count=10), DispEst(l, r, D, d_begin=10, d_count=14)]
    try:
        for rank, de in enumerate(shards):
            de.setGuidedFilter(window, eps)
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


@pytest.mark.parametrize("s", [2, 4, 8])
def test_fgf_window16(s, scenes, oracle_scene_results):
    _, _, l, r = scenes["Teddy"]
    ref = oracle_scene_results["Teddy"]
    lf, rf = WO.cost_filter_fgf(l, r, ref["lraw"], ref["rraw"], 16, 1e-4, s)
    with DispEst(l, r, 64) as de:
        de.setGuidedFilter(16, 1e-4)
        de.setSubsampleRate(s)
        de.CostConst_GPU()
        assert de.CostFilter_FGF_GPU() == 0
        assert_same(de.read_cost_volume(0), lf, f"FGF s={s} left")
        assert_same(de.read_cost_volume(1), rf, f"FGF s={s} right")


def test_fgf_box_limit(crops):
    """window 16 at s = 1 is a 33 x 33 box: more than the FGF kernel's shared memory holds -> PSM_EINVAL, nothing runs."""
    l, r, _, _ = crops["Teddy"]
    L = capi.lib()
    with DispEst(l, r, 24) as de:
        de.CostConst_GPU()
        de.setGuidedFilter(16, 1e-4)
        n = de.launch_count()
        assert L.psm_cost_filter_fgf(de.handle, 1) == capi.PSM_EINVAL
        assert b"shared memory" in L.psm_last_error(de.handle)
        assert de.launch_count() == n
        assert L.psm_cost_filter_fgf(de.handle, 2) == capi.PSM_OK    # 17 x 17 fits


def test_switching_parameters_between_frames(scenes, oracle_scene_results):
    """non-default, then back to the defaults: today's results and today's launch count per frame."""
    _, _, l, r = scenes["Cones"]
    ref = oracle_scene_results["Cones"]
    with DispEst(l, r, 64) as fresh:
        n0 = fresh.launch_count()
        fresh.CostConst_GPU(); fresh.CostFilter_GPU(); fresh.DispSelect_GPU()
        per_frame = fresh.launch_count() - n0
    with DispEst(l, r, 64) as de:
        for window, eps in ((16, 1e-3), (8, 1e-4), (5, 1e-4), (8, 1e-4)):
            de.setGuidedFilter(window, eps)
            n = de.launch_count()
            de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
            if (window, eps) == (8, 1e-4):
                assert de.launch_count() - n == per_frame
                assert_same(de.read_cost_volume(0), ref["lf"], "back to defaults: left volume")
                assert_same(de.lDisMap, ref["ld"], "back to defaults: left map")
                assert_same(de.rDisMap, ref["rd"], "back to defaults: right map")
            else:
                lf, _ = WO.cost_filter(l, r, ref["lraw"], ref["rraw"], window, eps)
                assert_same(de.read_cost_volume(0), lf, f"window {window} left volume")
                assert_same(de.lDisMap, WO.wta(lf), f"window {window} left map")


def test_full_hd_window16_row_band(oracle):
    """1920 x 1080 x 128 at window 16 against the oracle on a row band (top border and interior rows)."""
    W, H, D, window, eps = 1920, 1080, 128, 16, 1e-4
    l8, r8, _ = synth.stereo_pair_u8(W, H, D)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    ds = [0, 1, 37, 127]
    with DispEst(l, r, D) as de:
        de.setGuidedFilter(window, eps)
        de.CostConst_GPU()
        raw = {v: {d: de.read_cost_slice(v, d) for d in ds} for v in (0, 1)}
        de.CostFilter_GPU()
        got = {v: {d: de.read_cost_slice(v, d) for d in ds} for v in (0, 1)}
    for v, img in ((0, l), (1, r)):
        rgb, mean, var = WO.cvf_preprocess(img, window)
        for d in ds:
            q = WO.guided_filter(rgb, mean, var, raw[v][d], window, eps)
            for ys in (slice(0, 40), slice(500, 540), slice(1050, 1080)):
                assert_same(got[v][d][ys], q[ys], f"view {v} d {d} rows {ys}")


def test_errors_leave_context_unchanged(crops):
    l, r, lraw, rraw = crops["Teddy"]
    L = capi.lib()
    with DispEst(l, r, 24) as de:
        assert de.setGuidedFilter(9, 1e-3) == 0
        for window, eps in ((0, 1e-4), (33, 1e-4), (8, 0.0), (8, -1.0), (8, float("nan")), (8, float("inf"))):
            assert L.psm_set_guided_filter(de.handle, window, eps) == capi.PSM_EINVAL, (window, eps)
            with pytest.raises(capi.PsmError):
                de.setGuidedFilter(window, eps)
        de.CostConst_GPU()
        de.CostFilter_GPU()
        lf, _ = WO.cost_filter(l, r, lraw, rraw, 9, 1e-3)
        assert_same(de.read_cost_volume(0), lf, "after rejected calls: (9, 1e-3) still in force")
        for mode in (capi.PSM_CVF_MIXED, capi.PSM_CVF_NAIVE):
            de.set_option(capi.PSM_OPT_CVF_MODE, mode)
            de.CostConst_GPU()
            assert L.psm_cost_filter(de.handle) == capi.PSM_EINVAL
            assert b"PSM_CVF_EXACT" in L.psm_last_error(de.handle)
        de.setGuidedFilter(8, 1e-4)   # back at the defaults every mode runs again
        assert L.psm_cost_filter(de.handle) == capi.PSM_OK


def test_cpp_facade_set_guided_filter(tmp_path, scenes, oracle_scene_results, oracle):
    exe = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
    if not os.path.exists(exe):
        pytest.skip("dispest_demo not built")
    _, _, l, r = scenes["Teddy"]
    ref = oracle_scene_results["Teddy"]
    H, W, _ = l.shape
    l.tofile(tmp_path / "l.f32"); r.tofile(tmp_path / "r.f32")
    out = subprocess.run([exe, str(W), str(H), "64", str(tmp_path / "l.f32"), str(tmp_path / "r.f32"),
                          str(tmp_path / "l.u8"), str(tmp_path / "r.u8"), "12", "0.001"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    lf, _ = WO.cost_filter(l, r, ref["lraw"], ref["rraw"], 12, 1e-3)
    ld = np.fromfile(tmp_path / "l.u8", np.uint8).reshape(H, W)
    assert_same(ld, oracle.post_process(l, WO.wta(lf)), "C++ facade lDisMap at window 12 (after PostProcess_GPU)")
