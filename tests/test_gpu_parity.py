"""GPU parity tests (run on an H100): the CUDA path, called through the C-ABI, against the
CPU oracle on the same inputs.  Bar: bit-exact raw costs, guide planes, a/b, filtered costs and
u8 disparity maps (north_star tolerance is 1e-4 on a/b and +-1 disparity; we hold the stronger
bit-exact bar in the default PSM_CVF_EXACT mode)."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN, read_png
from primestereomatch_b200 import DispEst, capi, synth

pytestmark = pytest.mark.gpu

A_B_TOL = 1e-4  # north_star: "32-bit float within 1e-4 on a/b"


def run_gpu(l, r, D, mode=capi.PSM_CVF_EXACT, variant=0, keep=True, options=()):
    out = {}
    with DispEst(l, r, D, 8, True) as de:
        de.set_option(capi.PSM_OPT_CVF_MODE, mode)
        de.set_option(capi.PSM_OPT_VARIANT, variant)
        for key, value in options:
            de.set_option(key, value)
        assert de.CostConst_GPU() == 0
        if keep:
            out["lraw"], out["rraw"] = de.read_cost_volume(0), de.read_cost_volume(1)
        assert de.CostFilter_GPU() == 0
        if keep:
            out["lf"], out["rf"] = de.read_cost_volume(0), de.read_cost_volume(1)
        assert de.DispSelect_GPU() == 0
        out["ld"], out["rd"] = de.lDisMap.copy(), de.rDisMap.copy()
        out["launches"] = de.launch_count()
    return out


def assert_same(a, b, what):
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        diff = np.abs(a.astype(np.float64) - b.astype(np.float64))
        raise AssertionError(f"{what}: {len(bad)} / {a.size} mismatches, max|d|={np.nanmax(diff):.3e}, "
                             f"first at {bad[0].tolist()}: got {a[tuple(bad[0])]!r} want {b[tuple(bad[0])]!r}")


def test_device_present():
    assert capi.lib().psm_device_count() >= 1


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_ingest_and_guide_planes(scene, scenes, oracle, oracle_scene_results):
    _, _, l, r = scenes[scene]
    rgb, mean, var = oracle.cvf_preprocess(l)
    with DispEst(l, r, 64) as de:
        de.CostConst_GPU()
        for c in range(3):
            assert_same(de.read_guide_plane(0, c), rgb[c], f"split channel {c}")
            assert_same(de.read_guide_plane(0, 3 + c), mean[c], f"mean_I {c}")
        for k in range(6):
            assert_same(de.read_guide_plane(0, 6 + k), var[k], f"var_I {k}")
        assert_same(de.read_guide_plane(0, 12), oracle_scene_results[scene]["lg"], "left x-gradient")
        assert_same(de.read_guide_plane(1, 12), oracle_scene_results[scene]["rg"], "right x-gradient")


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_middlebury_full_path_bit_exact(scene, scenes, oracle_scene_results):
    """BASELINE configs C1/C2: CVC + CVF + WTA vs the CPU path, 450x375, D=64."""
    _, _, l, r = scenes[scene]
    ref = oracle_scene_results[scene]
    g = run_gpu(l, r, 64)
    assert_same(g["lraw"], ref["lraw"], "left raw volume")
    assert_same(g["rraw"], ref["rraw"], "right raw volume")
    assert_same(g["lf"], ref["lf"], "left filtered volume")
    assert_same(g["rf"], ref["rf"], "right filtered volume")
    assert_same(g["ld"], ref["ld"], "lDisMap")
    assert_same(g["rd"], ref["rd"], "rDisMap")
    s = scene.lower()
    assert_same(g["ld"], read_png(os.path.join(GOLDEN, f"{s}_lDis.png")), "lDisMap vs golden PNG")
    assert_same(g["rd"], read_png(os.path.join(GOLDEN, f"{s}_rDis.png")), "rDisMap vs golden PNG")
    assert g["launches"] > 0


def test_uint8_input_mode_bit_exact(scenes, oracle_scene_results):
    """C1 'uint8' reading A (SURVEY 8c): u8 PNG -> x(1/255) on the device -> same fp32 path."""
    l8, r8, _, _ = scenes["Cones"]
    g = run_gpu(l8, r8, 64, keep=False)
    assert_same(g["ld"], oracle_scene_results["Cones"]["ld"], "lDisMap (u8 input)")
    assert_same(g["rd"], oracle_scene_results["Cones"]["rd"], "rDisMap (u8 input)")


@pytest.mark.parametrize("scene", ["Teddy"])
def test_coefficients_a_b(scene, scenes, oracle, oracle_scene_results):
    """a/b within 1e-4 (north_star); in fact bit-exact."""
    _, _, l, r = scenes[scene]
    rgb, mean, var = oracle.cvf_preprocess(l)
    with DispEst(l, r, 64) as de:
        de.CostConst_GPU()
        for d in (1, 20, 63):
            a, b = de.read_ab_slice(0, d)
            _, ra, rb = oracle.guided_filter(rgb, mean, var, oracle_scene_results[scene]["lraw"][d], want_ab=True)
            assert np.max(np.abs(a - ra)) <= A_B_TOL and np.max(np.abs(b - rb)) <= A_B_TOL
            assert_same(a, ra, f"a d={d}")
            assert_same(b, rb, f"b d={d}")


def test_naive_device_kernels_agree(scenes, oracle_scene_results):
    """The unfused direct-sum kernels are an independent device implementation of the same math."""
    _, _, l, r = scenes["Teddy"]
    l, r = l[:120, :200].copy(), r[:120, :200].copy()
    a = run_gpu(l, r, 16, mode=capi.PSM_CVF_NAIVE)
    b = run_gpu(l, r, 16, mode=capi.PSM_CVF_EXACT)
    assert_same(a["lf"], b["lf"], "naive vs streaming, left")
    assert_same(a["rf"], b["rf"], "naive vs streaming, right")


@pytest.mark.parametrize("W,H,D", [(16, 16, 4), (17, 23, 5), (113, 40, 8), (130, 50, 9), (225, 33, 16),
                                   (451, 64, 12), (64, 300, 6), (340, 17, 3), (12, 9, 4), (5, 40, 2)])
def test_ragged_sizes_bit_exact(W, H, D, oracle):
    """Widths that are not multiples of 4 / of the 112-column strip, heights around the segment
    logic, one-strip and many-strip cases, and tiny images (served by the direct-sum kernels)."""
    rng = np.random.default_rng(W * 1000 + H)
    l = rng.random((H, W, 3), dtype=np.float32)
    r = np.roll(l, -3, axis=1) + rng.normal(0, 0.02, (H, W, 3)).astype(np.float32)
    r = np.clip(r, 0, 1).astype(np.float32)
    ref = oracle.pipeline(l, r, D, keep_volumes=True)
    g = run_gpu(l, r, D)
    assert_same(g["lf"], ref["lVol"], f"left filtered {W}x{H}x{D}")
    assert_same(g["rf"], ref["rVol"], f"right filtered {W}x{H}x{D}")
    assert_same(g["ld"], ref["lDis"], "lDisMap")
    assert_same(g["rd"], ref["rDis"], "rDisMap")


def test_exact_zero_costs_and_ties(oracle):
    """A noise-free shifted pair has exact-zero raw costs at the true disparity: zeros must stay
    exact zeros through the fp64 sums, and WTA ties must resolve to the lowest d."""
    l8, r8, dgt = synth.stereo_pair_u8(256, 96, 32, seed=5)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    ref = oracle.pipeline(l, r, 32, keep_volumes=True)
    g = run_gpu(l, r, 32)
    assert_same(g["lf"], ref["lVol"], "left filtered")
    assert_same(g["ld"], ref["lDis"], "lDisMap")
    assert_same(g["rd"], ref["rDis"], "rDisMap")


def test_write_slice_filter_wta_special_values(oracle):
    """Caller-provided raw costs incl. negative values, -0.0 and exact ties go through CVF+WTA
    identically (WTA semantics of DispSel.cpp:93-102)."""
    rng = np.random.default_rng(11)
    H, W, D = 48, 144, 6
    l = rng.random((H, W, 3), dtype=np.float32)
    vol = rng.normal(0, 1, (D, H, W)).astype(np.float32)
    vol[2, :, :40] = vol[4, :, :40]          # exact ties -> lowest d after identical filtering
    vol[3, 10:20] = -0.0
    rgb, mean, var = oracle.cvf_preprocess(l)
    want = np.stack([oracle.guided_filter(rgb, mean, var, vol[d]) for d in range(D)])
    with DispEst(l, l, D) as de:
        de.CostConst_GPU()
        for d in range(D):
            de.write_cost_slice(0, d, vol[d])
            de.write_cost_slice(1, d, vol[d])
        de.CostFilter_GPU()
        got = de.read_cost_volume(0)
        de.DispSelect_GPU()
        assert_same(got, want, "filtered caller-provided volume")
        assert_same(de.lDisMap, oracle.wta(want), "WTA on filtered caller-provided volume")


def test_stage_order_errors():
    l = np.zeros((32, 32, 3), np.float32)
    with DispEst(l, l, 8) as de:
        L = capi.lib()
        assert L.psm_cost_const(de.handle) == capi.PSM_ESTATE      # no images yet
        assert L.psm_cost_filter(de.handle) == capi.PSM_ESTATE     # no raw volume yet
        assert b"before" in L.psm_last_error(de.handle)
        de.CostConst_GPU(); de.CostFilter_GPU()
        assert L.psm_cost_filter(de.handle) == capi.PSM_ESTATE     # already filtered
    with pytest.raises(ValueError):
        DispEst(l, l.astype(np.uint8), 8)                          # DispEst.cpp:26-29 type mismatch
    with DispEst(l, l, 8) as de:
        assert de.setThreads(9) == -1 and de.setThreads(4) == 0    # DispEst.cpp:172-179


def test_full_size_c4_crops_and_properties(oracle):
    """BASELINE config C4 (1920x1080, D=128) at full size: crops at the four image corners, the
    strip / segment seams and the interior are bit-exact against the oracle; WTA map bit-exact
    against the oracle's WTA of the GPU's own filtered volume; two runs are bit-identical."""
    W, H, D = 1920, 1080, 128
    l8, r8, dgt = synth.stereo_pair_u8(W, H, D)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    ds = [0, 1, 37, 127]

    class Box:
        pass

    box = Box()
    with DispEst(l, r, D) as de:
        de.CostConst_GPU()
        box.read_cost_slice_raw = [{d: de.read_cost_slice(v, d) for d in ds} for v in (0, 1)]
        # raw costs: oracle on full rows is cheap for a handful of slices
        lg, rg = oracle.cvc_preprocess(l), oracle.cvc_preprocess(r)
        for d in ds:
            want = np.empty((H, W), np.float32)
            oracle.lib().orc_buildcv_left(l, r, lg, rg, W, H, d, want)
            assert_same(box.read_cost_slice_raw[0][d], want, f"raw left d={d}")
            oracle.lib().orc_buildcv_right(r, l, rg, lg, W, H, d, want)
            assert_same(box.read_cost_slice_raw[1][d], want, f"raw right d={d}")
        de.CostFilter_GPU()
        box.filtered = [{d: de.read_cost_slice(v, d) for d in ds} for v in (0, 1)]
        de.DispSelect_GPU()
        ld1, rd1 = de.lDisMap.copy(), de.rDisMap.copy()
        # crops need a 16-px distance from any cut edge: 8 for the guide means + 8 for the filter
        regions = [(0, 40, 0, 64), (0, 40, W - 64, W), (H - 40, H, 0, 64), (H - 40, H, W - 64, W),
                   (500, 540, 96, 136), (250, 290, 1780, 1830), (520, 560, 900, 960)]
        for (y0, y1, x0, x1) in regions:
            for view in (0, 1):
                Hh, Ww = H, W
                m = 16
                cy0, cy1 = max(0, y0 - m), min(Hh, y1 + m)
                cx0, cx1 = max(0, x0 - m), min(Ww, x1 + m)
                img = (l if view == 0 else r)[cy0:cy1, cx0:cx1].copy()
                rgb, mean, var = oracle.cvf_preprocess(img)
                for d in ds:
                    raw = box.read_cost_slice_raw[view][d][cy0:cy1, cx0:cx1].copy()
                    q = oracle.guided_filter(rgb, mean, var, raw)
                    got = box.filtered[view][d][y0:y1, x0:x1]
                    want = q[y0 - cy0:y1 - cy0, x0 - cx0:x1 - cx0]
                    assert_same(got, want, f"view {view} d={d} crop y{y0}:{y1} x{x0}:{x1}")
        # WTA against the oracle's WTA over the GPU's own filtered volume (row band: D x 64 x W)
        band = slice(512, 576)
        vol = np.stack([de.read_cost_slice(0, d)[band] for d in range(D)])
        assert_same(ld1[band], oracle.wta(vol), "lDisMap band")
        # the interior of the left map mostly recovers the synthetic ground truth
        ok = (ld1[:, D:] == dgt[:, None]).mean()
        assert ok > 0.80, ok
        # determinism
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        assert_same(de.lDisMap, ld1, "second run lDisMap")
        assert_same(de.rDisMap, rd1, "second run rDisMap")


def test_sharded_keys_match_unsharded(scenes, oracle_scene_results):
    """Disparity-sharded path on one GPU: two contexts own d in [0,32) and [32,64); packed
    (cost,d) minima are 'gathered' and reduced; result equals the unsharded maps bit for bit."""
    torch = pytest.importorskip("torch")
    _, _, l, r = scenes["Teddy"]
    H, W, _ = l.shape
    L = capi.lib()
    keys = torch.empty((2, 2, H * W), dtype=torch.int64, device="cuda")  # [view][rank][pix]
    shards = [DispEst(l, r, 64, d_begin=0, d_count=32), DispEst(l, r, 64, d_begin=32, d_count=32)]
    try:
        for rank, de in enumerate(shards):
            de.CostConst_GPU(); de.CostFilter_GPU()
            capi.check(L.psm_disp_select_keys(de.handle, keys[0, rank].data_ptr(), keys[1, rank].data_ptr()), de.handle)
            de.sync()
        ld = np.zeros((H, W), np.uint8); rd = np.zeros((H, W), np.uint8)
        de = shards[0]
        capi.check(L.psm_disp_reduce_keys(de.handle, keys[0].data_ptr(), keys[1].data_ptr(), 2,
                                          ld.ctypes.data_as(C.c_void_p), W, rd.ctypes.data_as(C.c_void_p), W), de.handle)
        assert_same(ld, oracle_scene_results["Teddy"]["ld"], "sharded lDisMap")
        assert_same(rd, oracle_scene_results["Teddy"]["rd"], "sharded rDisMap")
        # an unsharded-only entry point refuses to run on a shard
        assert L.psm_disp_select_device(shards[1].handle) == capi.PSM_ESTATE
    finally:
        for de in shards:
            de.close()


def test_cpp_dispest_facade_demo(tmp_path, scenes, oracle, oracle_scene_results):
    """The C++ DispEst facade (primestereomatch_b200/host), driven like StereoMatch::compute drives the
    reference's DispEst (CostConst_GPU, CostFilter_GPU, DispSelect_GPU, PostProcess_GPU), produces the oracle's
    post-filtered maps on Teddy."""
    import subprocess
    from conftest import ROOT
    exe = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
    if not os.path.exists(exe):
        pytest.skip("dispest_demo not built")
    _, _, l, r = scenes["Teddy"]
    H, W, _ = l.shape
    l.tofile(tmp_path / "l.f32"); r.tofile(tmp_path / "r.f32")
    out = subprocess.run([exe, str(W), str(H), "64", str(tmp_path / "l.f32"), str(tmp_path / "r.f32"),
                          str(tmp_path / "l.u8"), str(tmp_path / "r.u8")], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    ld = np.fromfile(tmp_path / "l.u8", np.uint8).reshape(H, W)
    rd = np.fromfile(tmp_path / "r.u8", np.uint8).reshape(H, W)
    assert_same(ld, oracle.post_process(l, oracle_scene_results["Teddy"]["ld"]), "C++ facade lDisMap (after PostProcess_GPU)")
    assert_same(rd, oracle.post_process(r, oracle_scene_results["Teddy"]["rd"]), "C++ facade rDisMap (after PostProcess_GPU)")


def test_fused_wta_p2p_gather_matches_unsharded(scenes, oracle_scene_results):
    """Fused WTA + exchange: each shard's WTA kernel scatters its packed minima into the exchange block
    of the shard that reduces that pixel chunk; each reducer then writes the winning disparities into
    every shard's result map (here all blocks live on the one GPU; across processes they are NVLink
    peer mappings).  Two frames check that the blocks can be reused."""
    _, _, l, r = scenes["Teddy"]
    H, W, _ = l.shape
    L = capi.lib()
    shards = [DispEst(l, r, 64, d_begin=0, d_count=40), DispEst(l, r, 64, d_begin=40, d_count=24)]
    try:
        bufs = (C.c_void_p * 2)()
        for k, de in enumerate(shards):
            p = C.c_void_p()
            capi.check(L.psm_p2p_create_buffer(de.handle, 2, C.byref(p)), de.handle)
            bufs[k] = p.value
        for k, de in enumerate(shards):
            capi.check(L.psm_p2p_set_peers(de.handle, bufs, 2, k), de.handle)
        for frame in range(2):
            for de in shards:
                de.CostConst_GPU(); de.CostFilter_GPU()
                capi.check(L.psm_disp_select_keys_p2p(de.handle), de.handle)
            for de in shards:
                de.sync()                                   # stands in for the cross-rank barrier
            for de in shards:
                capi.check(L.psm_disp_reduce_p2p(de.handle), de.handle)
            for de in shards:
                de.sync()
            for de in shards:
                ld = np.zeros((H, W), np.uint8); rd = np.zeros((H, W), np.uint8)
                capi.check(L.psm_disp_fetch_p2p(de.handle, ld.ctypes.data_as(C.c_void_p), W,
                                                rd.ctypes.data_as(C.c_void_p), W), de.handle)
                assert_same(ld, oracle_scene_results["Teddy"]["ld"], f"p2p lDisMap frame {frame}")
                assert_same(rd, oracle_scene_results["Teddy"]["rd"], f"p2p rDisMap frame {frame}")
    finally:
        for de in shards:
            de.close()


def test_max_disparity_256(oracle):
    """D = 256 (BASELINE config C5 depth): disparities up to 255 must survive the u8 maps
    (the reference's OpenCL WTA keeps the index in a signed char, dispsel.cl:96; ours is unsigned)."""
    W, H, D = 400, 48, 256
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=9)
    rng = np.random.default_rng(2)
    r8 = np.clip(r8.astype(np.int16) + rng.integers(-3, 4, r8.shape), 0, 255).astype(np.uint8)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    ref = oracle.pipeline(l, r, D, keep_volumes=True)
    g = run_gpu(l, r, D)
    assert_same(g["lf"], ref["lVol"], "left filtered D=256")
    assert_same(g["ld"], ref["lDis"], "lDisMap D=256")
    assert_same(g["rd"], ref["rDis"], "rDisMap D=256")
    assert int(ref["lDis"].max()) > 127  # the test really exercises indices a signed char cannot hold


def test_c5_shape_sharded_eight_ways_on_one_gpu(oracle):
    """BASELINE config C5 structure (D=256 split over 8 ranks, 32 slices each) at a reduced image
    size: eight shard contexts on one GPU, fused WTA+gather buffers, result == unsharded oracle."""
    W, H, D, G = 256, 40, 256, 8
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=21)
    rng = np.random.default_rng(5)
    r8 = np.clip(r8.astype(np.int16) + rng.integers(-3, 4, r8.shape), 0, 255).astype(np.uint8)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    ref = oracle.pipeline(l, r, D)
    L = capi.lib()
    from primestereomatch_b200.sharding import shard_range
    shards = [DispEst(l, r, D, d_begin=shard_range(D, G, k)[0], d_count=shard_range(D, G, k)[1]) for k in range(G)]
    try:
        bufs = (C.c_void_p * G)()
        for k, de in enumerate(shards):
            p = C.c_void_p()
            capi.check(L.psm_p2p_create_buffer(de.handle, G, C.byref(p)), de.handle)
            bufs[k] = p.value
        for k, de in enumerate(shards):
            capi.check(L.psm_p2p_set_peers(de.handle, bufs, G, k), de.handle)
            de.CostConst_GPU(); de.CostFilter_GPU()
            capi.check(L.psm_disp_select_keys_p2p(de.handle), de.handle)
        for de in shards:
            de.sync()
        for de in shards:
            capi.check(L.psm_disp_reduce_p2p(de.handle), de.handle)
        for de in shards:
            de.sync()
        ld = np.zeros((H, W), np.uint8); rd = np.zeros((H, W), np.uint8)
        capi.check(L.psm_disp_fetch_p2p(shards[3].handle, ld.ctypes.data_as(C.c_void_p), W,
                                        rd.ctypes.data_as(C.c_void_p), W), shards[3].handle)
        assert_same(ld, ref["lDis"], "8-way sharded lDisMap")
        assert_same(rd, ref["rDis"], "8-way sharded rDisMap")
    finally:
        for de in shards:
            de.close()


def test_row_steps_like_cv_mat_rois(scenes, oracle_scene_results):
    """cv::Mat inputs/outputs may have row steps larger than the packed width (ROIs, aligned
    allocations): psm_set_images / psm_disp_select honour the byte steps."""
    _, _, l, r = scenes["Teddy"]
    H, W, _ = l.shape
    L = capi.lib()
    lp = np.full((H, W + 37, 3), np.nan, np.float32); lp[:, :W] = l      # padded rows, NaN in the padding
    rp = np.full((H, W + 5, 3), np.nan, np.float32); rp[:, :W] = r
    ld = np.full((H, W + 11), 255, np.uint8); rd = np.full((H, W + 64), 255, np.uint8)
    with DispEst(l, r, 64) as de:
        capi.check(L.psm_set_images(de.handle, lp.ctypes.data_as(C.c_void_p), lp.strides[0],
                                    rp.ctypes.data_as(C.c_void_p), rp.strides[0]), de.handle)
        capi.check(L.psm_cost_const(de.handle), de.handle)
        capi.check(L.psm_cost_filter(de.handle), de.handle)
        capi.check(L.psm_disp_select(de.handle, ld.ctypes.data_as(C.c_void_p), ld.strides[0],
                                     rd.ctypes.data_as(C.c_void_p), rd.strides[0]), de.handle)
        # a step smaller than one packed row is rejected
        assert L.psm_set_images(de.handle, lp.ctypes.data_as(C.c_void_p), W * 12 - 4,
                                rp.ctypes.data_as(C.c_void_p), rp.strides[0]) == capi.PSM_EINVAL
    assert_same(ld[:, :W], oracle_scene_results["Teddy"]["ld"], "lDisMap with row steps")
    assert_same(rd[:, :W], oracle_scene_results["Teddy"]["rd"], "rDisMap with row steps")
    assert np.all(ld[:, W:] == 255) and np.all(rd[:, W:] == 255)  # padding untouched


@pytest.mark.parametrize("lo,hi", [(-12, 3), (-40, 10)])
def test_wide_dynamic_range_costs_stay_bit_exact(lo, hi, oracle):
    """fp64 running sums are exact only while a window spans < 2^23 in magnitude; beyond that both
    OpenCV's order and ours round in fp64 (differently).  The final rounding to float hides those
    2^-53 effects except with probability ~2^-28 per mean, so even costs spanning e^50 must come out
    bit-identical here."""
    rng = np.random.default_rng(5)
    H, W, D = 96, 256, 4
    l = rng.random((H, W, 3), dtype=np.float32)
    rgb, mean, var = oracle.cvf_preprocess(l)
    vol = (np.abs(rng.standard_normal((D, H, W))) * np.exp(rng.uniform(lo, hi, (D, H, W)))).astype(np.float32)
    want = np.stack([oracle.guided_filter(rgb, mean, var, vol[d]) for d in range(D)])
    with DispEst(l, l, D) as de:
        de.CostConst_GPU()
        for d in range(D):
            de.write_cost_slice(0, d, vol[d]); de.write_cost_slice(1, d, vol[d])
        de.CostFilter_GPU()
        assert_same(de.read_cost_volume(0), want, f"filtered volume, cost range e^{lo}..e^{hi}")
