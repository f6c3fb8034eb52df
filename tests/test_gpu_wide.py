"""GPU: 16-bit disparity maps (psm_create_u16, max_disp up to 4096), bit for bit through the C-ABI against the CPU
oracle (oracle/ for the volumes, tests/wide_oracle.c for the arg-min and the post-filter), the stored reference
results of golden_wide.json and the u8 contexts at D <= 256."""
import ctypes as C
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle import oracle as O
from primestereomatch_b200 import DispEst, capi, synth
from primestereomatch_b200.sharding import shard_range
import wide_oracle as WO

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN, "golden_wide.json")) as f:
    GOLD = json.load(f)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def assert_same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, f"{what}: shape {a.shape} vs {b.shape}"
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {a.size} differ, first at {list(i)}: {a[i]!r} vs {b[i]!r}")


def posterise(img8, masks=(0xE0, 0xE0, 0xC0)):
    return (img8 & np.array(masks, np.uint8)).astype(np.uint8)


def inject_maps(de, ld, rd):
    """Make the context's maps exactly ld / rd (values in 1 .. maxDis - 1) with one-hot cost slices."""
    assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
    for d in range(de.maxDis):
        de.write_cost_slice(0, d, (ld != d).astype(np.float32))
        de.write_cost_slice(1, d, (rd != d).astype(np.float32))
    assert de.DispSelect_GPU() == 0
    assert_same(de.lDisMap, ld, "injected left"); assert_same(de.rDisMap, rd, "injected right")


def oracle_maps(l, r, D):
    _, _, lraw, rraw = O.cost_const(l, r, D)
    lf, rf = O.cost_filter(l, r, lraw, rraw)
    return lf, rf, WO.wta16(lf), WO.wta16(rf)


# ---- 1. same maps as a u8 context at D <= 256 -------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
@pytest.mark.parametrize("u8", [False, True])
def test_same_maps_at_d64(scene, u8, scenes, oracle_scene_results):
    l8, r8, l, r = scenes[scene]
    li, ri = (l8, r8) if u8 else (l, r)
    ref = oracle_scene_results[scene]
    with DispEst(li, ri, 64) as a, DispEst(li, ri, 64, map_bits=16) as b:
        assert a.map_bits == 8 and a.lDisMap.dtype == np.uint8
        assert b.map_bits == 16 and b.lDisMap.dtype == np.uint16
        for de in (a, b):
            de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        assert_same(b.lDisMap, a.lDisMap.astype(np.uint16), "u16 vs u8 left")
        assert_same(b.rDisMap, a.rDisMap.astype(np.uint16), "u16 vs u8 right")
        assert_same(b.lDisMap, ref["ld"].astype(np.uint16), "u16 vs oracle left")
        for de in (a, b):
            de.PostProcess_GPU()
        assert_same(b.lDisMap, a.lDisMap.astype(np.uint16), "post-filtered u16 vs u8 left")
        assert_same(b.rDisMap, a.rDisMap.astype(np.uint16), "post-filtered u16 vs u8 right")
        assert_same(b.lDisMap, O.post_process(l, ref["ld"]).astype(np.uint16), "post-filtered u16 vs orc_wmf")
        for setting in ((16, 25.5, 1, "exp"), (5, 10.0, 2, "iv2")):
            for de in (a, b):
                de.setPostFilter(*setting); de.DispSelect_GPU(); de.PostProcess_GPU()
            assert_same(b.lDisMap, a.lDisMap.astype(np.uint16), f"u16 vs u8 left at {setting}")
        for de in (a, b):   # FGF branch
            de.CostConst_GPU(); de.CostFilter_FGF_GPU(); de.DispSelect_GPU()
        assert_same(b.lDisMap, a.lDisMap.astype(np.uint16), "FGF u16 vs u8 left")
        assert_same(b.rDisMap, a.rDisMap.astype(np.uint16), "FGF u16 vs u8 right")


def test_default_map_bits_follow_maxdis():
    l, r, _ = synth.stereo_pair_f32(40, 8, 300)
    for D, bits in ((2, 8), (256, 8), (257, 16), (4096, 16)):
        with DispEst(l, r, D) as de:
            assert de.map_bits == bits and de.lDisMap.dtype == (np.uint16 if bits == 16 else np.uint8)
    with pytest.raises(capi.PsmError):
        DispEst(l, r, 300, map_bits=8)
    with pytest.raises(ValueError):
        DispEst(l, r, 64, map_bits=12)


# ---- 2. wide synthetic pairs ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", GOLD["wta"], ids=lambda c: f"D{c['D']}")
def test_selection_low_byte_is_the_stored_reference(case):
    D, W, H = case["D"], case["W"], case["H"]
    vol, _ = WO.argmin_volume(W, H, D, case["seed"])
    l, r, _ = synth.stereo_pair_f32(W, H, 8)
    with DispEst(l, r, D) as de:
        de.CostConst_GPU(); de.CostFilter_GPU()
        for d in range(D):
            de.write_cost_slice(0, d, vol[d]); de.write_cost_slice(1, d, vol[D - d] if d else vol[0])
        de.DispSelect_GPU()
        assert sha((de.lDisMap & 0xFF).astype(np.uint8)) == case["ref_sha"]
        assert sha(de.lDisMap) == case["sha16"] and int(de.lDisMap.max()) > 255
        rv = np.concatenate([vol[:1], vol[:0:-1]])
        assert_same(de.rDisMap, WO.wta16(rv), "right view")


def band_crop(W, D):
    """rows of the synthetic pair around the first 40-row band whose d_gt exceeds 255 (the largest d_gt of the first
    200 bands where none does: D = 257 gives at most 239)"""
    dg = [1 + (k * 17) % (D - 2) for k in range(1, 200)]
    k = 1 + next((i for i, g in enumerate(dg) if g > 255), int(np.argmax(dg)))
    return k, 40 * k - 8, 40 * k + 48


@pytest.mark.parametrize("D", [257, 300, 511, 600, 1024])
def test_wide_pairs_against_the_oracle(D):
    W = D + 96
    k, y0, y1 = band_crop(W, D)
    l8, r8, dgt = synth.stereo_pair_u8(W, y1, D)
    l, r = synth.to_f32(l8[y0:y1]), synth.to_f32(r8[y0:y1])
    dgt = dgt[y0:y1]
    lf, rf, ld, rd = oracle_maps(l, r, D)
    with DispEst(l, r, D) as de:
        de.CostConst_GPU(); de.CostFilter_GPU()
        for d in sorted({1, 17, 255, 256, D // 2, D - 1, int(dgt[20])}):
            assert_same(de.read_cost_slice(0, d), lf[d], f"D={D} left slice {d}")
            assert_same(de.read_cost_slice(1, d), rf[d], f"D={D} right slice {d}")
        de.DispSelect_GPU()
        assert_same(de.lDisMap, ld, f"D={D} left map"); assert_same(de.rDisMap, rd, f"D={D} right map")
        g = int(dgt[20])
        if D >= 300:
            assert g > 255 and int(de.lDisMap.max()) > 255
        # functional check: the band's interior recovers d_gt.  The cost there is exactly 0 at d_gt, but the guided
        # filter's output at another disparity can dip just below 0 (q = a.I + b is not monotone), so a few pixels may
        # select that one instead; the maps themselves are pinned bit for bit above.
        inner = de.lDisMap[16:40, g + 8:W - 8]
        assert np.mean(inner == g) >= 0.99, (g, np.unique(inner, return_counts=True))


# ---- 3. ragged sizes, D > W -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,H,D", [(1, 1, 300), (5, 40, 257), (70, 3, 600), (37, 21, 1024), (300, 9, 400), (17, 17, 4096)])
def test_ragged_sizes(W, H, D):
    rng = np.random.default_rng(W * 7 + H)
    l = synth.to_f32(rng.integers(0, 256, (H, W, 3)).astype(np.uint8))
    r = synth.to_f32(np.roll(rng.integers(0, 256, (H, W, 3)).astype(np.uint8), 0))
    lf, rf, ld, rd = oracle_maps(l, r, D)
    with DispEst(l, r, D) as de:
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        assert_same(de.lDisMap, ld, f"{W}x{H}x{D} left"); assert_same(de.rDisMap, rd, f"{W}x{H}x{D} right")
        de.PostProcess_GPU()
        assert_same(de.lDisMap, WO.post_process16(l, ld), f"{W}x{H}x{D} post-filtered left")


# ---- 4. with the other per-context settings ---------------------------------------------------------------------------
@pytest.mark.parametrize("stage", ["window", "cost", "fgf"])
def test_settings_and_fgf(stage):
    W, H, D = 400, 48, 300
    l, r, _ = synth.stereo_pair_f32(W, H, 64, seed=9)
    with DispEst(l, r, D) as a, DispEst(l, r, 256) as b:
        for de in (a, b):
            if stage == "window":
                de.setGuidedFilter(13, 1e-3)
            if stage == "cost":
                de.setMatchingCost(0.11, 0.21, 0.008)
            de.CostConst_GPU()
            de.CostFilter_FGF_GPU() if stage == "fgf" else de.CostFilter_GPU()
        la, ra = a.read_cost_volume(0), a.read_cost_volume(1)
        for d in (0, 1, 100, 255):   # a slice does not depend on D: the u8 context's slices, pinned by the existing tests
            assert_same(la[d], b.read_cost_slice(0, d), f"{stage} left slice {d}")
            assert_same(ra[d], b.read_cost_slice(1, d), f"{stage} right slice {d}")
        a.DispSelect_GPU()
        assert_same(a.lDisMap, WO.wta16(la), f"{stage} left"); assert_same(a.rDisMap, WO.wta16(ra), f"{stage} right")
        if stage == "fgf":
            _, _, lraw, rraw = O.cost_const(l, r, D)
            lf, _ = O.cost_filter_fgf(l, r, lraw, rraw, s=4)
            assert_same(la, lf, "FGF volume")


# ---- 5. post-filter on wide maps --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def wide_scenes(scenes, oracle_scene_results):
    out = {}
    for name, (l8, r8, _, _) in scenes.items():
        res = oracle_scene_results[name]
        out[name] = (O.u8_to_f32(posterise(l8)), O.u8_to_f32(posterise(r8)), WO.widen(res["ld"], 7), WO.widen(res["rd"], 8))
    return out


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_post_filter_at_every_golden_wide_setting(scene, wide_scenes):
    l, r, ld, rd = wide_scenes[scene]
    with DispEst(l, r, GOLD["wmf"]["max_disp"]) as de:
        inject_maps(de, ld, rd)
        for ent in GOLD["wmf"]["settings"]:
            de.setPostFilter(ent["radius"], float.fromhex(ent["sigma"]), ent["iterations"], ent["weight"])
            de.DispSelect_GPU(); de.PostProcess_GPU()
            assert sha(de.lDisMap) == ent["scenes"][scene]["l"]["sha"], f"{ent['key']} {scene} left"
            assert sha(de.rDisMap) == ent["scenes"][scene]["r"]["sha"], f"{ent['key']} {scene} right"


def test_post_filter_every_radius_iterations_and_switching(wide_scenes):
    l, r, ld, rd = (np.ascontiguousarray(a[100:164, 150:246]) for a in wide_scenes["Cones"])
    D = 1024
    ld, rd = (ld * 2 + 1).astype(np.uint16), (rd * 2 + 1).astype(np.uint16)   # values up to 1023
    with DispEst(l, r, D) as de:
        inject_maps(de, ld, rd)
        for setting in [(radius, 25.5, 1, "exp") for radius in range(1, 33)] + \
                       [(9, 25.5, 16, "exp"), (6, 7.0, 16, "iv2"), (9, 25.5, 1, "off"), (12, 60.0, 2, "iv1"), (9, 25.5, 1, "exp")]:
            de.setPostFilter(*setting)
            de.DispSelect_GPU(); de.PostProcess_GPU()
            assert_same(de.lDisMap, WO.post_process16(l, ld, *setting), f"left at {setting}")
            assert_same(de.rDisMap, WO.post_process16(r, rd, *setting), f"right at {setting}")


# ---- 6. sharded -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("G", [2, 8])
def test_sharded_on_one_gpu(G):
    W, H, D = 700, 40, 600
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=21)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    L = capi.lib()
    with DispEst(l, r, D) as full:
        full.CostConst_GPU(); full.CostFilter_GPU(); full.DispSelect_GPU()
        want_l, want_r = full.lDisMap.copy(), full.rDisMap.copy()
        full.PostProcess_GPU()
        want_pl, want_pr = full.lDisMap.copy(), full.rDisMap.copy()
    assert int(want_l.max()) > 255
    shards = [DispEst(l, r, D, d_begin=shard_range(D, G, k)[0], d_count=shard_range(D, G, k)[1], map_bits=16) for k in range(G)]
    try:
        import torch
        keys = [torch.empty((2, W * H), dtype=torch.int64, device="cuda") for _ in range(G)]
        for k, de in enumerate(shards):
            de.CostConst_GPU(); de.CostFilter_GPU()
            capi.check(L.psm_disp_select_keys(de.handle, keys[k][0].data_ptr(), keys[k][1].data_ptr()), de.handle)
            de.sync()
        gathered = torch.stack(keys, 1).contiguous()   # [2, G, H*W]
        ld = np.zeros((H, W), np.uint16); rd = np.zeros((H, W), np.uint16)
        u8 = np.zeros((H, W), np.uint8)
        de = shards[G - 1]
        assert L.psm_disp_reduce_keys(de.handle, gathered[0].data_ptr(), gathered[1].data_ptr(), G, ptr(u8), W, ptr(u8), W) \
            == capi.PSM_EINVAL
        assert b"psm_disp_reduce_keys_u16" in L.psm_last_error(de.handle)
        capi.check(L.psm_disp_reduce_keys_u16(de.handle, gathered[0].data_ptr(), gathered[1].data_ptr(), G,
                                              ptr(ld), 2 * W, ptr(rd), 2 * W), de.handle)
        assert_same(ld, want_l, f"{G}-way keys left"); assert_same(rd, want_r, f"{G}-way keys right")
        # fused P2P path
        bufs = (C.c_void_p * G)()
        for k, de in enumerate(shards):
            p = C.c_void_p()
            capi.check(L.psm_p2p_create_buffer(de.handle, G, C.byref(p)), de.handle)
            bufs[k] = p.value
        for k, de in enumerate(shards):
            capi.check(L.psm_p2p_set_peers(de.handle, bufs, G, k), de.handle)
            capi.check(L.psm_disp_select_keys_p2p(de.handle), de.handle)
        for de in shards:
            de.sync()
        for de in shards:
            capi.check(L.psm_disp_reduce_p2p(de.handle), de.handle)
        for de in shards:
            de.sync()
        for k in (0, G - 1):
            ld[:] = 0; rd[:] = 0
            capi.check(L.psm_disp_fetch_p2p_u16(shards[k].handle, ptr(ld), 2 * W, ptr(rd), 2 * W), shards[k].handle)
            assert_same(ld, want_l, f"{G}-way p2p left, rank {k}"); assert_same(rd, want_r, f"{G}-way p2p right, rank {k}")
        assert L.psm_disp_fetch_p2p(shards[0].handle, ptr(u8), W, ptr(u8), W) == capi.PSM_EINVAL
        # post-filter of the exchanged maps
        de = shards[1]
        de.PostProcess_GPU()
        assert_same(de.lDisMap, want_pl, f"{G}-way post-filtered left"); assert_same(de.rDisMap, want_pr, f"{G}-way post-filtered right")
    finally:
        for de in shards:
            de.close()


# ---- 7. past 32-bit offsets -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,band", [(600, "top"), (1040, "bottom")])
def test_full_width_frame_past_32_bit_offsets(D, band):
    import torch
    W, H, B, CROP = 1920, 1080, 16, 32
    need = 4 * (W + 64) * H * D * 4
    free, _ = torch.cuda.mem_get_info()
    if need * 1.1 > free:
        pytest.skip(f"needs about {need / 2**30:.0f} GiB of device memory, {free / 2**30:.0f} GiB free")
    l8, r8, _ = synth.stereo_pair_u8(W, H, 256, seed=D)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    with DispEst(l, r, D) as de:
        assert 4 * de.d_count * H * W > 2 ** 32
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        rows = slice(0, CROP) if band == "top" else slice(H - CROP, H)
        lf, rf, ld, rd = oracle_maps(np.ascontiguousarray(l[rows]), np.ascontiguousarray(r[rows]), D)
        sel = slice(0, B) if band == "top" else slice(CROP - B, CROP)
        got_l, got_r = de.lDisMap[rows][sel], de.rDisMap[rows][sel]
        assert_same(got_l, ld[sel], f"D={D} {band} band left"); assert_same(got_r, rd[sel], f"D={D} {band} band right")
        sl = de.read_cost_slice(0, D - 1)[rows][sel]
        assert_same(sl, lf[D - 1][sel], f"D={D} last slice, {band} band")


# ---- 8. errors --------------------------------------------------------------------------------------------------------
def test_error_cases():
    L = capi.lib()
    ctx = C.c_void_p()
    for args in ((64, 64, 1, 0, 1), (64, 64, 4097, 0, 4097), (0, 8, 300, 0, 300), (8, 0, 300, 0, 300),
                 (64, 64, 600, 590, 20), (64, 64, 600, -1, 10), (64, 64, 600, 0, 0)):
        assert L.psm_create_u16(C.byref(ctx), *args, 0) == capi.PSM_EINVAL, args
        assert not ctx and L.psm_last_error(None)
    assert L.psm_create_u16(None, 64, 64, 300, 0, 300, 0) == capi.PSM_EINVAL
    W, H = 24, 16
    l, r, _ = synth.stereo_pair_f32(W, H, 8)
    u8 = np.zeros((H, W), np.uint8); u16 = np.zeros((H, W), np.uint16)
    with DispEst(l, r, 300) as w, DispEst(l, r, 64) as n:
        # out-of-order stages
        assert L.psm_disp_select_u16(w.handle, ptr(u16), 2 * W, ptr(u16), 2 * W) == capi.PSM_ESTATE
        assert L.psm_post_process_u16(w.handle, ptr(u16), 2 * W, ptr(u16), 2 * W) == capi.PSM_ESTATE
        for de in (w, n):
            de.CostConst_GPU(); de.CostFilter_GPU()
        # a map call of the other format
        for fn, h, buf, step, right in ((L.psm_disp_select, w, u8, W, b"psm_disp_select_u16"),
                                        (L.psm_disp_select_async, w, u8, W, b"psm_disp_select_u16_async"),
                                        (L.psm_post_process, w, u8, W, b"psm_post_process_u16"),
                                        (L.psm_disp_fetch_p2p, w, u8, W, b"psm_disp_fetch_p2p_u16"),
                                        (L.psm_disp_select_u16, n, u16, 2 * W, b"use psm_disp_select"),
                                        (L.psm_disp_select_u16_async, n, u16, 2 * W, b"use psm_disp_select_async"),
                                        (L.psm_post_process_u16, n, u16, 2 * W, b"use psm_post_process"),
                                        (L.psm_disp_fetch_p2p_u16, n, u16, 2 * W, b"use psm_disp_fetch_p2p")):
            assert fn(h.handle, ptr(buf), step, ptr(buf), step) == capi.PSM_EINVAL
            assert right in L.psm_last_error(h.handle), L.psm_last_error(h.handle)
        assert L.psm_disp_reduce_keys_u16(n.handle, None, None, 1, ptr(u16), 2 * W, ptr(u16), 2 * W) == capi.PSM_EINVAL
        # null or short steps
        assert L.psm_disp_select_u16(w.handle, None, 2 * W, ptr(u16), 2 * W) == capi.PSM_EINVAL
        assert L.psm_disp_select_u16(w.handle, ptr(u16), 2 * W - 1, ptr(u16), 2 * W) == capi.PSM_EINVAL
        assert L.psm_disp_select_u16(w.handle, ptr(u16), 2 * W, ptr(u16), W) == capi.PSM_EINVAL
        assert L.psm_disp_select_u16(w.handle, ptr(u16), 2 * W, ptr(u16), 2 * W) == capi.PSM_OK
        assert L.psm_post_process_u16(w.handle, ptr(u16), W, ptr(u16), 2 * W) == capi.PSM_EINVAL
        assert L.psm_disp_fetch_p2p_u16(w.handle, ptr(u16), 2 * W, ptr(u16), 2 * W) == capi.PSM_ESTATE
        for fn in (L.psm_disp_select_u16, L.psm_post_process_u16, L.psm_disp_fetch_p2p_u16):
            assert fn(None, ptr(u16), 2 * W, ptr(u16), 2 * W) == capi.PSM_EINVAL
        # device pointers: the 16-bit maps, pitch W
        p, pitch = C.c_void_p(), C.c_size_t()
        for what in (2, 3):
            capi.check(L.psm_device_ptr(w.handle, what, C.byref(p), C.byref(pitch)), w.handle)
            assert p.value and pitch.value == W
        # a sharded u16 context cannot select unsharded
    with DispEst(l, r, 600, d_begin=300, d_count=300) as s:
        s.CostConst_GPU(); s.CostFilter_GPU()
        assert L.psm_disp_select_u16(s.handle, ptr(u16), 2 * W, ptr(u16), 2 * W) == capi.PSM_ESTATE


# ---- 9. launch counts -------------------------------------------------------------------------------------------------
def test_launch_counts_match_the_u8_context():
    l, r, _ = synth.stereo_pair_f32(200, 40, 32, seed=3)
    counts = {}
    for bits in (8, 16):
        with DispEst(l, r, 200, map_bits=bits) as de:
            c = []
            for stage in (de.CostConst_GPU, de.CostFilter_GPU, de.DispSelect_GPU, de.PostProcess_GPU, de.CostFilter_FGF_GPU):
                if stage == de.CostFilter_FGF_GPU:
                    de.CostConst_GPU()
                n = de.launch_count(); stage(); c.append(de.launch_count() - n)
            for setting in ((16, 25.5, 1, "exp"), (9, 25.5, 3, "exp"), (5, 2.0, 2, "iv2")):
                de.setPostFilter(*setting)
                n = de.launch_count(); de.PostProcess_GPU(); c.append(de.launch_count() - n)
            counts[bits] = c
    assert counts[8] == counts[16], counts


# ---- 10. the C++ demo -------------------------------------------------------------------------------------------------
def test_cpp_demo_at_d300(tmp_path):
    exe = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
    if not os.path.exists(exe):
        pytest.skip("dispest_demo not built")
    W, H, D = 400, 48, 300
    k, y0, y1 = band_crop(W, D)
    l8, r8, _ = synth.stereo_pair_u8(W, y1, D)
    l, r = synth.to_f32(l8[y0:y1]), synth.to_f32(r8[y0:y1])
    H = l.shape[0]
    l.tofile(tmp_path / "l.f32"); r.tofile(tmp_path / "r.f32")
    out = subprocess.run([exe, str(W), str(H), str(D), str(tmp_path / "l.f32"), str(tmp_path / "r.f32"),
                          str(tmp_path / "l.u16"), str(tmp_path / "r.u16")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    _, _, ld, rd = oracle_maps(l, r, D)
    got_l = np.fromfile(tmp_path / "l.u16", np.uint16).reshape(H, W)
    got_r = np.fromfile(tmp_path / "r.u16", np.uint16).reshape(H, W)
    assert int(ld.max()) > 255
    assert_same(got_l, WO.post_process16(l, ld), "C++ demo left"); assert_same(got_r, WO.post_process16(r, rd), "C++ demo right")
