"""GPU tests of the CVF kernel's modes and paths (all through the C-ABI):
  * PSM_CVF_EXACT in its builds (integer widening / F2F conversions, prefetch and staging options; variant 0 is
    shipped, variant 1 is the round-1 kernel) -- all bit-exact;
  * inputs outside the integer-widening domain (negative / -0 costs, negative guide values) -- bit-exact through
    the per-row slow path and the guide flag;
  * PSM_CVF_MIXED -- bit-exact against its CPU model (tests/mixed_model.py), within tolerance of the exact path;
  * BASELINE config C3 (1280x720x64) at full size against the oracle."""
import numpy as np
import pytest

import mixed_model as MM
from primestereomatch_b200 import DispEst, capi, synth
from test_gpu_parity import assert_same, run_gpu

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("variant", [0, 1, 2, 3, 6, 9, 11, 12])
def test_exact_variants_bit_exact(variant, scenes, oracle_scene_results):
    _, _, l, r = scenes["Teddy"]
    ref = oracle_scene_results["Teddy"]
    g = run_gpu(l, r, 64, variant=variant)
    assert_same(g["lf"], ref["lf"], f"left filtered, variant {variant}")
    assert_same(g["rf"], ref["rf"], f"right filtered, variant {variant}")
    assert_same(g["ld"], ref["ld"], "lDisMap")
    assert_same(g["rd"], ref["rd"], "rDisMap")


@pytest.mark.parametrize("variant", [0, 9, 11])
def test_costs_outside_the_integer_domain(variant, oracle):
    """Negative and -0 costs in a few rows (the rest of the volume is ordinary): the affected warps leave
    the integer-widening loop for the F2F loop mid-segment; everything stays bit-exact."""
    rng = np.random.default_rng(17)
    H, W, D = 300, 260, 5
    l = rng.random((H, W, 3), dtype=np.float32)
    vol = np.abs(rng.normal(0, 1, (D, H, W))).astype(np.float32)
    vol[1, 140:143, 30:60] *= -1.0        # negative costs in the steady part of a segment
    vol[2, 5, :] = -0.0                   # -0 in the warm-up rows
    vol[3, 290:, 200:] *= -1.0            # negative costs at the bottom
    vol[4, :, :] = 0.0                    # exact zeros everywhere stay on the fast path
    rgb, mean, var = oracle.cvf_preprocess(l)
    want = np.stack([oracle.guided_filter(rgb, mean, var, vol[d]) for d in range(D)])
    with DispEst(l, l, D) as de:
        de.set_option(capi.PSM_OPT_VARIANT, variant)
        de.CostConst_GPU()
        for d in range(D):
            de.write_cost_slice(0, d, vol[d]); de.write_cost_slice(1, d, vol[d])
        de.CostFilter_GPU()
        assert_same(de.read_cost_volume(0), want, "filtered volume with negative / -0 costs")
        assert_same(de.read_cost_volume(1), want, "right view")


def test_guide_outside_the_integer_domain(oracle):
    """Images are in [0,1] by contract; a negative channel value raises the guide flag and the whole
    launch of that view converts with F2F -- still the oracle's result."""
    rng = np.random.default_rng(23)
    H, W, D = 64, 150, 6
    l = rng.random((H, W, 3), dtype=np.float32)
    r = np.roll(l, -2, axis=1).copy()
    l[10, 20, 1] = -0.25
    ref = oracle.pipeline(l, r, D, keep_volumes=True)
    g = run_gpu(l, r, D)
    assert_same(g["lf"], ref["lVol"], "left filtered (negative guide value)")
    assert_same(g["rf"], ref["rVol"], "right filtered")
    assert_same(g["ld"], ref["lDis"], "lDisMap")


# CVC builds (option 106): 0 = shipped (interior fast path for the warps that are matched inside the image at every owned
# disparity + scalar window loads elsewhere), 2 = no fast path (the round-1 loop), 1 / 3 = fast path + one 128-bit window load
# per plane per four disparities for the other warps when the shard starts at a multiple of 4.  Raw volumes equal the oracle's
# for aligned / unaligned shards, depths that are not multiples of 4, widths that are not multiples of 4 (partial warps), wide
# rows where most warps take the fast path, and disparities beyond the image width (no warp does).
@pytest.mark.parametrize("cvc_variant", [0, 1, 2, 3])
@pytest.mark.parametrize("W,H,D,d_begin,d_count", [(450, 37, 64, 0, 64), (451, 20, 21, 0, 21), (130, 24, 40, 8, 13),
                                                   (130, 24, 40, 7, 9), (37, 16, 48, 0, 48), (1280, 9, 64, 32, 32),
                                                   (253, 12, 256, 128, 128), (66, 10, 7, 4, 3)])
def test_cvc_builds_raw_volumes(W, H, D, d_begin, d_count, cvc_variant, oracle):
    rng = np.random.default_rng(W + 31 * D)
    l = rng.random((H, W, 3), dtype=np.float32)
    r = np.clip(np.roll(l, -5, axis=1) + rng.normal(0, 0.05, (H, W, 3)), 0, 1).astype(np.float32)
    _, _, lraw, rraw = oracle.cost_const(l, r, D)
    with DispEst(l, r, D, d_begin=d_begin, d_count=d_count) as de:
        de.set_option(106, cvc_variant)
        assert de.CostConst_GPU() == 0
        assert_same(de.read_cost_volume(0), lraw[d_begin:d_begin + d_count], f"left raw volume, CVC build {cvc_variant}")
        assert_same(de.read_cost_volume(1), rraw[d_begin:d_begin + d_count], f"right raw volume, CVC build {cvc_variant}")


@pytest.mark.parametrize("chunk", [5, 8, 16, 100])
def test_cvc_slice_chunks(chunk, oracle):
    """Option 108: slices per CTA of the CVC kernel (the grid then walks the volume chunk by chunk); incl. a ragged last chunk."""
    rng = np.random.default_rng(chunk)
    W, H, D = 300, 21, 37
    l = rng.random((H, W, 3), dtype=np.float32)
    r = np.clip(np.roll(l, -4, axis=1) + rng.normal(0, 0.05, (H, W, 3)), 0, 1).astype(np.float32)
    _, _, lraw, rraw = oracle.cost_const(l, r, D)
    for d_begin, d_count in ((0, D), (8, 20)):
        with DispEst(l, r, D, d_begin=d_begin, d_count=d_count) as de:
            de.set_option(108, chunk)
            assert de.CostConst_GPU() == 0
            assert_same(de.read_cost_volume(0), lraw[d_begin:d_begin + d_count], f"left raw volume, chunk {chunk}")
            assert_same(de.read_cost_volume(1), rraw[d_begin:d_begin + d_count], f"right raw volume, chunk {chunk}")


# Packed remainder strips (psm_cvf_stream.cuh): the W % 112 rightmost columns are filtered 4 slices per warp (remainder
# <= 16 columns: 113, 128, 227, 240), 2 slices per warp (<= 48 columns: 129, 160, 260) or by a whole warp per slice
# (161, 300: the round-1 decomposition, also what option 105 = 1 forces).  D = 5, 9, 13 leave slice groups of the last
# packed warp without a slice.  Exact: equal to the oracle; mixed: equal to the CPU model of the mode.
@pytest.mark.parametrize("no_pack", [0, 1])
@pytest.mark.parametrize("W,H,D", [(113, 30, 5), (128, 26, 9), (129, 40, 4), (160, 33, 13), (161, 24, 5), (227, 31, 6),
                                   (240, 300, 3), (260, 50, 7), (300, 20, 2)])
def test_packed_remainder_strips(W, H, D, no_pack, oracle):
    rng = np.random.default_rng(W * 7 + H)
    l = rng.random((H, W, 3), dtype=np.float32)
    r = np.clip(np.roll(l, -2, axis=1) + rng.normal(0, 0.03, (H, W, 3)), 0, 1).astype(np.float32)
    ref = oracle.pipeline(l, r, D, keep_volumes=True)
    g = run_gpu(l, r, D, options=[(105, no_pack)])
    assert_same(g["lf"], ref["lVol"], f"left filtered volume, no_pack={no_pack}")
    assert_same(g["rf"], ref["rVol"], f"right filtered volume, no_pack={no_pack}")
    assert_same(g["ld"], ref["lDis"], "lDisMap")
    assert_same(g["rd"], ref["rDis"], "rDisMap")
    m = run_gpu(l, r, D, mode=capi.PSM_CVF_MIXED, options=[(105, no_pack)])
    for img, raw, key in ((l, g["lraw"], "lf"), (r, g["rraw"], "rf")):
        assert_same(m[key], MM.cost_filter_mixed(oracle, img, raw), f"MIXED {key} vs CPU model, no_pack={no_pack}")


@pytest.mark.parametrize("rows", [8, 12, 16, 24, 100])
def test_guide_precompute_segment_rows(rows, scenes, oracle):
    """Option 107: rows per warp of the guide precompute (each segment restarts its fp64 column sums)."""
    _, _, l, r = scenes["Teddy"]
    _, mean, var = oracle.cvf_preprocess(l)
    with DispEst(l, r, 8) as de:
        de.set_option(107, rows)
        de.CostConst_GPU()
        for c in range(3):
            assert_same(de.read_guide_plane(0, 3 + c), mean[c], f"mean_I {c}, {rows} rows per warp")
        for k in range(6):
            assert_same(de.read_guide_plane(0, 6 + k), var[k], f"var_I {k}, {rows} rows per warp")


@pytest.mark.parametrize("log2_scale", [0, 40, 70])
def test_guide_planes_with_large_values(log2_scale, oracle):
    """The guide precompute widens I and I*I with the integer trick only while every product is finite: images below 2^63
    stay on that path (scale 1 and 2^40), larger ones (scale 2^70: squares overflow to inf) raise the
    guide flag and convert with F2F.  The image is k/256 * scale, so every fp64 window sum is exact and the comparison does
    not depend on the summation order; means and variances equal the CPU result (NaN == NaN where the CPU has NaN)."""
    rng = np.random.default_rng(5)
    H, W = 40, 150
    l = (rng.integers(0, 256, (H, W, 3)).astype(np.float32) / 256.0) * np.float32(2.0 ** log2_scale)
    with np.errstate(all="ignore"):
        _, mean, var = oracle.cvf_preprocess(l)
        with DispEst(l, l, 4) as de:
            de.CostConst_GPU()
            for c in range(3):
                assert np.array_equal(de.read_guide_plane(0, 3 + c), mean[c], equal_nan=True), f"mean_I {c}"
            for k in range(6):
                assert np.array_equal(de.read_guide_plane(0, 6 + k), var[k], equal_nan=True), f"var_I {k}"
    if log2_scale == 70:
        assert not np.isfinite(var).all()      # the case really left the finite domain


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_mixed_mode_matches_its_model_and_tolerance(scene, scenes, oracle, oracle_scene_results):
    _, _, l, r = scenes[scene]
    ref = oracle_scene_results[scene]
    g = run_gpu(l, r, 64, mode=capi.PSM_CVF_MIXED)
    assert_same(g["lraw"], ref["lraw"], "raw volume is mode-independent")
    for view, img, raw, key in ((0, l, ref["lraw"], "lf"), (1, r, ref["rraw"], "rf")):
        want = MM.cost_filter_mixed(oracle, img, raw)
        assert_same(g[key], want, f"MIXED filtered volume vs CPU model, view {view}")
        assert np.max(np.abs(g[key] - ref[key])) <= 1e-5
    for got, exact in ((g["ld"], ref["ld"]), (g["rd"], ref["rd"])):
        diff = np.abs(got.astype(np.int16) - exact.astype(np.int16))
        assert int((diff > 1).sum()) == 0          # north-star: +-1 disparity level
        assert int((diff > 0).sum()) == 0          # in fact identical maps on both scenes


@pytest.mark.parametrize("variant", [0, 9, 10, 12, 13, 14, 15])
@pytest.mark.parametrize("W,H,D", [(16, 16, 4), (17, 23, 5), (113, 40, 8), (130, 50, 9), (225, 33, 16),
                                   (451, 64, 12), (64, 300, 6), (340, 17, 3)])
def test_mixed_mode_ragged_sizes(W, H, D, variant, oracle):
    """variant 9 = guide rows staged in shared memory by bulk async copies (TMA); same results."""
    rng = np.random.default_rng(W * 1000 + H)
    l = rng.random((H, W, 3), dtype=np.float32)
    r = np.clip(np.roll(l, -3, axis=1) + rng.normal(0, 0.02, (H, W, 3)), 0, 1).astype(np.float32)
    _, _, lraw, rraw = oracle.cost_const(l, r, D)
    g = run_gpu(l, r, D, mode=capi.PSM_CVF_MIXED, variant=variant)
    assert_same(g["lf"], MM.cost_filter_mixed(oracle, l, lraw), f"MIXED left {W}x{H}x{D}")
    assert_same(g["rf"], MM.cost_filter_mixed(oracle, r, rraw), f"MIXED right {W}x{H}x{D}")


def test_mixed_mode_full_size_c4_against_exact():
    """C4: MIXED vs EXACT on the same device volumes: |dq| and the disparity maps."""
    W, H, D = 1920, 1080, 128
    l8, r8, _ = synth.stereo_pair_u8(W, H, D)
    rng = np.random.default_rng(4)
    r8 = np.clip(r8.astype(np.int16) + rng.integers(-5, 6, r8.shape), 0, 255).astype(np.uint8)
    maps, slices = {}, {}
    for mode in (capi.PSM_CVF_EXACT, capi.PSM_CVF_MIXED):
        with DispEst(l8, r8, D) as de:
            de.set_option(capi.PSM_OPT_CVF_MODE, mode)
            de.CostConst_GPU(); de.CostFilter_GPU()
            slices[mode] = [de.read_cost_slice(0, d) for d in (1, 40, 127)]
            de.DispSelect_GPU()
            maps[mode] = (de.lDisMap.copy(), de.rDisMap.copy())
    for a, b in zip(slices[capi.PSM_CVF_EXACT], slices[capi.PSM_CVF_MIXED]):
        assert np.max(np.abs(a - b)) <= 1e-5
    for a, b in zip(maps[capi.PSM_CVF_EXACT], maps[capi.PSM_CVF_MIXED]):
        diff = np.abs(a.astype(np.int16) - b.astype(np.int16))
        assert int((diff > 1).sum()) == 0, (int((diff > 1).sum()), np.argwhere(diff > 1)[:5].tolist())
        print("C4 mixed vs exact: +-1 flips", int((diff == 1).sum()), "of", diff.size)


def test_full_size_c3_bit_exact(oracle):
    """BASELINE config C3 (synthetic 1280x720, D=64) at FULL size: both filtered volumes and both maps
    against the oracle (noise added so that costs are not trivially zero)."""
    W, H, D = 1280, 720, 64
    l8, r8, _ = synth.stereo_pair_u8(W, H, D)
    rng = np.random.default_rng(33)
    r8 = np.clip(r8.astype(np.int16) + rng.integers(-4, 5, r8.shape), 0, 255).astype(np.uint8)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    ref = oracle.pipeline(l, r, D, threads=64, keep_volumes=True)
    g = run_gpu(l, r, D)
    assert_same(g["lf"], ref["lVol"], "C3 left filtered volume")
    assert_same(g["rf"], ref["rVol"], "C3 right filtered volume")
    assert_same(g["ld"], ref["lDis"], "C3 lDisMap")
    assert_same(g["rd"], ref["rDis"], "C3 rDisMap")


def test_async_upload_pipeline_matches_synchronous_calls(scenes, oracle_scene_results):
    """psm_set_images_async / _commit + psm_disp_select_async (two-deep pipeline: frame k+1 uploads while frame k
    computes) give the same maps as the synchronous reference-style calls, for alternating frames and for u8 frames."""
    import ctypes as C
    torch = pytest.importorskip("torch")
    l8, r8, l, r = scenes["Teddy"]
    H, W, _ = l.shape
    L = capi.lib()
    frames = [(torch.from_numpy(l).pin_memory(), torch.from_numpy(r).pin_memory()),
              (torch.from_numpy(r).pin_memory(), torch.from_numpy(l).pin_memory())]   # second frame: views swapped
    want = []
    with DispEst(l, r, 64) as de:
        for fl, fr in frames:
            de.setInputImages(fl.numpy(), fr.numpy())
            de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
            want.append((de.lDisMap.copy(), de.rDisMap.copy()))
        assert np.array_equal(want[0][0], oracle_scene_results["Teddy"]["ld"])
        maps = [(torch.empty((H, W), dtype=torch.uint8).pin_memory(), torch.empty((H, W), dtype=torch.uint8).pin_memory()) for _ in range(4)]
        order = [0, 1, 1, 0]
        step = W * 3 * 4
        assert L.psm_set_images_commit(de.handle) == capi.PSM_ESTATE            # nothing pending
        capi.check(L.psm_set_images_async(de.handle, frames[order[0]][0].data_ptr(), step, frames[order[0]][1].data_ptr(), step), de.handle)
        assert L.psm_set_images_async(de.handle, frames[0][0].data_ptr(), step, frames[0][1].data_ptr(), step) == capi.PSM_ESTATE   # one in flight
        for k in range(4):
            capi.check(L.psm_set_images_commit(de.handle), de.handle)
            if k + 1 < 4:
                nxt = frames[order[k + 1]]
                capi.check(L.psm_set_images_async(de.handle, nxt[0].data_ptr(), step, nxt[1].data_ptr(), step), de.handle)
            capi.check(L.psm_cost_const(de.handle), de.handle)
            capi.check(L.psm_cost_filter(de.handle), de.handle)
            capi.check(L.psm_disp_select_async(de.handle, maps[k][0].data_ptr(), W, maps[k][1].data_ptr(), W), de.handle)
        de.sync()
        for k in range(4):
            assert_same(maps[k][0].numpy(), want[order[k]][0], f"pipelined frame {k} lDisMap")
            assert_same(maps[k][1].numpy(), want[order[k]][1], f"pipelined frame {k} rDisMap")
        # 8-bit frames through the same pipeline
        l8p, r8p = torch.from_numpy(l8).pin_memory(), torch.from_numpy(r8).pin_memory()
        capi.check(L.psm_set_images_u8_async(de.handle, l8p.data_ptr(), W * 3, r8p.data_ptr(), W * 3), de.handle)
        capi.check(L.psm_set_images_commit(de.handle), de.handle)
        capi.check(L.psm_cost_const(de.handle), de.handle)
        capi.check(L.psm_cost_filter(de.handle), de.handle)
        capi.check(L.psm_disp_select_async(de.handle, maps[0][0].data_ptr(), W, maps[0][1].data_ptr(), W), de.handle)
        de.sync()
        assert_same(maps[0][0].numpy(), want[0][0], "u8 pipelined lDisMap")


def test_selection_requires_a_filtered_volume():
    """ADVICE round 1: the select entry points used to run on zero / raw volumes when called out of order."""
    l = np.random.default_rng(0).random((32, 48, 3), dtype=np.float32)
    with DispEst(l, l, 8) as de:
        L = capi.lib()
        assert L.psm_disp_select_device(de.handle) == capi.PSM_ESTATE          # nothing computed yet
        de.CostConst_GPU()
        assert L.psm_disp_select_device(de.handle) == capi.PSM_ESTATE          # raw costs only
        de.CostFilter_GPU()
        assert L.psm_disp_select_device(de.handle) == capi.PSM_OK
        de.CostConst_GPU()
        assert L.psm_disp_select_device(de.handle) == capi.PSM_ESTATE          # a new CVC invalidates the filtered volume
