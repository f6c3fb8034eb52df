"""GPU: the filtered costs beside each winner (PSM_OPT_COSTS, psm_copy_costs_device, psm_read_costs).  Every context kind
(unblocked, blocked at B = 1, 2, 3, a ragged B and B = D, multi-device with 2, 3 and 8 co-located shards, unblocked and
blocked) returns, as uint32 bit patterns, the oracle's filtered volume gathered at the oracle's own map (cost_triple_cases
.gather): the scenes, the flagged kinds under the exact filter and the FGF, MIXED against its CPU model, 16-bit maps at
D = 300, left-only frames, the seam-tie frames, ragged and tiny sizes, and a 1920 x 1080 x 2560 band at B = 128.  Then the
option's launches and state rules, and TorchStereo with a held-back stream."""
import ctypes as C
import os

import numpy as np
import pytest

import cost_triple_cases as CT
import image_cases as IC
import mixed_model as MM
import test_gpu_selection_seams as SEAMS
from gif_cases import assert_same
from oracle import oracle as O
from output_checks import assert_bits, expect, frame_counts, ptr
from primestereomatch_b200 import DispEst, capi, synth

pytestmark = pytest.mark.gpu

U8, U16, U32 = np.uint8, np.uint16, np.uint32


def run(l, r, D, dtype=U8, *, setup=None, fgf=None, left_only=False, volumes=False, **kw):
    """one frame with setCostOutput(True) -> (lmap, rmap, lcosts, rcosts), and with volumes the filtered volumes the
    context selected from (an unblocked single-device context)"""
    with DispEst(l, r, D, map_bits=8 * np.dtype(dtype).itemsize, **kw) as de:
        if setup:
            setup(de)
        if left_only:
            de.setViews("left")
        de.setCostOutput(True)
        assert de.CostConst_GPU() == 0
        if fgf:
            de.setSubsampleRate(fgf)
            assert de.CostFilter_FGF_GPU() == 0
        else:
            assert de.CostFilter_GPU() == 0
        assert de.DispSelect_GPU() == 0
        rm = None if de.rDisMap is None else de.rDisMap.copy()
        out = (de.lDisMap.copy(), rm, de.lCosts, de.rCosts)
        if volumes:
            out += tuple(de.read_cost_volume(v) for v in range(1 if left_only else 2))
        return out


def check(l, r, D, vols, what, dtype=U8, cases=None, left_only=False, **kw):
    """every context's maps equal O.wta of vols and its costs equal the gather of vols at those maps (NaN payloads
    aside).  The first case is the unblocked context: its costs equal the gather of its own filtered volumes bit for
    bit, payloads included, and every other context's costs equal its costs bit for bit."""
    maps = [O.wta(v, dtype) for v in vols]
    want = [CT.gather(v, m) for v, m in zip(vols, maps)]
    cases = SEAMS.contexts(D) if cases is None else cases
    assert cases[0][1] == {}
    ref = None
    for name, ctx, _ in cases:
        got = run(l, r, D, dtype, left_only=left_only, volumes=ref is None, **ctx, **kw)
        views = ((0, "left"),) if left_only else ((0, "left"), (1, "right"))
        if left_only:
            assert got[1] is None and got[3] is None
        for v, side in views:
            assert_same(got[v], maps[v], f"{what}, {name}: {side} map")
            assert_bits(got[2 + v], want[v], f"{what}, {name}: {side} costs vs the oracle", nan_any=True)
            if ref is None:
                assert_bits(got[2 + v], CT.gather(got[4 + v], got[v].astype(np.int64)), f"{what}: {side} costs vs the "
                            "device's own volume")
            else:
                assert_bits(got[2 + v], ref[2 + v].view(U32), f"{what}, {name}: {side} costs vs the unblocked context's")
        ref = ref or got
    return maps


SCENE_CASES = [("unblocked", {}, None), ("B=7", dict(block_slices=7), None), ("B=64", dict(block_slices=64), None),
               ("2 shards", dict(devices=[0, 0]), None), ("3 shards B=5", dict(devices=[0, 0, 0], block_slices=5), None)]


# ---- the scenes, exact filter, u8 and float frames ----------------------------------------------------------------------
@pytest.mark.parametrize("u8", [True, False])
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_scenes(scene, u8, scenes, oracle_scene_results):
    l8, r8, l, r = scenes[scene]
    res = oracle_scene_results[scene]
    frame = (l8, r8) if u8 else (l, r)
    check(*frame, 64, (res["lf"], res["rf"]), f"{scene} u8={u8}", cases=SCENE_CASES)


# ---- flagged kinds: costs +-inf, NaN, FLT_MAX, exact filter and FGF -----------------------------------------------------
@pytest.mark.parametrize("kind", IC.FLAGGED)
def test_flagged_exact(kind):
    W, H, D = IC.MAIN
    l, r = IC.frame(kind, W, H, D)
    check(l, r, D, SEAMS.filtered(l, r, D), f"{kind} exact")


@pytest.mark.parametrize("s", [2, 4])
@pytest.mark.parametrize("kind", ["nan", "posinf", "fltmax"])
def test_flagged_fgf(kind, s):
    W, H, D = IC.MAIN
    l, r = IC.frame(kind, W, H, D)
    check(l, r, D, SEAMS.filtered(l, r, D, fgf=s), f"{kind} FGF s={s}", fgf=s)


def test_mixed():
    W, H, D = 227, 61, 40
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=5)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    _, _, lraw, rraw = O.cost_const(l, r, D)
    vols = (MM.cost_filter_mixed(O, l, lraw), MM.cost_filter_mixed(O, r, rraw))
    check(l, r, D, vols, "MIXED", setup=lambda de: de.set_option(capi.PSM_OPT_CVF_MODE, capi.PSM_CVF_MIXED))


@pytest.mark.parametrize("kind", ["nan", "fltmax"])
def test_wide_u16(kind):
    l, r = IC.wide_frame(kind)
    W, H, D = IC.WIDE
    maps = check(l, r, D, SEAMS.filtered(l, r, D), f"{kind} D=300", U16,
                 cases=SEAMS.contexts(D, blocks=(7, 128, 200, D), shard_block=7))
    assert int(maps[0].max()) > 255


# ---- left-only frames ----------------------------------------------------------------------------------------------------
def test_left_only():
    W, H, D = IC.MAIN
    l, r = IC.frame("nan", W, H, D)
    check(l, r, D, SEAMS.filtered(l, r, D), "left-only nan", left_only=True)


# ---- exact ties across the seams, ragged and tiny sizes -----------------------------------------------------------------
@pytest.mark.parametrize("name", list(SEAMS.TIES))
def test_ties_across_seams(name):
    make, D, dtype = SEAMS.TIES[name]
    l8, r8 = make()
    check(l8, r8, D, SEAMS.filtered(O.u8_to_f32(l8), O.u8_to_f32(r8), D), name, dtype)


@pytest.mark.parametrize("W,H,D", SEAMS.GEOMETRIES)
def test_geometry_edges(W, H, D):
    rng = np.random.default_rng([W, H, D])
    base = rng.integers(0, 256, (H, W + 2, 3), dtype=U8)
    l8, r8 = np.ascontiguousarray(base[:, 2:]), np.ascontiguousarray(base[:, :W])
    vols = SEAMS.filtered(O.u8_to_f32(l8), O.u8_to_f32(r8), D)
    check(l8, r8, D, vols, f"{W}x{H} D={D}", cases=SEAMS.contexts(D, shard_block=1 if D == 2 else 3))


# ---- full HD at D = 2560, B = 128: winners in late blocks -----------------------------------------------------------------
def test_full_hd_late_blocks():
    import torch
    W, H, D, B, CROP = 1920, 1080, 2560, 128, 32
    free, _ = torch.cuda.mem_get_info()
    if free < 12 * 2 ** 30:
        pytest.skip(f"needs about 10 GiB of device memory, {free / 2**30:.1f} GiB free")
    l8, _, _ = synth.stereo_pair_u8(W, H, 256, seed=D)
    dgt = np.array([300, 700, 1100, 1500])[(np.arange(H) // 40) % 4]
    r8 = np.take_along_axis(l8, ((np.arange(W)[None, :] + dgt[:, None]) % W)[:, :, None].repeat(3, 2), 1)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    lm, rm, lc, rc = run(l, r, D, U16, block_slices=B)
    y0 = 13 * 40   # an interior band of disparity 700, 16 rows with an 8-row margin in its crop
    c0 = y0 - 8
    with np.errstate(all="ignore"):
        _, _, lraw, rraw = O.cost_const(l[c0:c0 + CROP], r[c0:c0 + CROP], D, threads=os.cpu_count())
        lf, rf = O.cost_filter(l[c0:c0 + CROP], r[c0:c0 + CROP], lraw, rraw, threads=os.cpu_count())
    del lraw, rraw
    rows, ys = slice(8, 24), slice(y0, y0 + 16)
    for what, vol, m, costs in (("left", lf, lm, lc), ("right", rf, rm, rc)):
        want_m = O.wta(vol, U16)[rows]
        assert_same(m[ys], want_m, f"rows {ys} {what} map")
        assert_bits(costs[:, ys], CT.gather(vol[:, rows], want_m.astype(np.int64)), f"rows {ys} {what} costs", nan_any=True)
    assert (lm[ys] > 255).mean() > 0.5
    del lf, rf
    multi = run(l, r, D, U16, devices=[0, 0], block_slices=B)
    for got, want, what in zip(multi, (lm, rm, lc, rc), ("left map", "right map", "left costs", "right costs")):
        assert_bits(got, np.ascontiguousarray(want).view(U32) if want.dtype == np.float32 else want, f"[0, 0] blocked {what}")


# ---- launches and state rules ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw,extra", [({}, 2), (dict(block_slices=7), 2), (dict(devices=[0, 0]), 4),
                                      (dict(devices=[0, 0, 0], block_slices=4), 6)])
def test_launches_and_maps(kw, extra):
    """off: a context that had the option on and off again launches and selects as one that never had it; on: the same
    maps, one more launch per view and shard in stage 3 (a blocked context's folds track the costs in the launches they
    make anyway)"""
    W, H, D = 200, 40, 50
    l, r, _ = synth.stereo_pair_u8(W, H, D, seed=4)
    with DispEst(l, r, D, **kw) as plain, DispEst(l, r, D, **kw) as toggled:
        toggled.setCostOutput(True)
        toggled.setCostOutput(False)
        base = frame_counts(plain)
        off = frame_counts(toggled)
        assert off[0] == base[0]
        assert_same(off[1], base[1], "off: left"); assert_same(off[2], base[2], "off: right")
        toggled.setCostOutput(True)
        on = frame_counts(toggled)
        assert on[0] == [base[0][0], base[0][1], base[0][2] + extra], (on[0], base[0])
        assert_same(on[1], base[1], "on: left"); assert_same(on[2], base[2], "on: right")


@pytest.mark.parametrize("kw", [{}, dict(block_slices=4), dict(devices=[0, 0])])
def test_state_rules(kw):
    import torch
    W, H, D = 64, 24, 12
    l, r, _ = synth.stereo_pair_u8(W, H, D, seed=2)
    L = capi.lib()
    plane = np.full((3, H, W), 7.0, np.float32)
    dev = torch.full((2, 3, H, W), 7.0, device="cuda:0")
    with DispEst(l, r, D, **kw) as de:
        h = de.handle
        # nothing written before a selection with the option on
        expect(L.psm_read_costs(h, 0, ptr(plane), W * 4), capi.PSM_ESTATE, de, "no costs")
        for bad in (2, -1):
            expect(L.psm_set_option(h, capi.PSM_OPT_COSTS, bad), capi.PSM_EINVAL, de, "PSM_OPT_COSTS")
        de.setCostOutput(True)
        de.CostConst_GPU(); de.CostFilter_GPU()
        n1 = de.launch_count()
        # rejected calls: nothing enqueued or written
        expect(L.psm_copy_costs_device(h, None, dev[1].data_ptr(), W * 4), capi.PSM_EINVAL, de, "pointer")
        expect(L.psm_copy_costs_device(h, dev[0].data_ptr(), None, W * 4), capi.PSM_EINVAL, de, "pointer")
        expect(L.psm_copy_costs_device(h, dev[0].data_ptr(), dev[1].data_ptr(), W * 4 - 4), capi.PSM_EINVAL, de, "step")
        expect(L.psm_read_costs(h, 2, ptr(plane), W * 4), capi.PSM_EINVAL, de, "view")
        expect(L.psm_read_costs(h, 0, None, W * 4), capi.PSM_EINVAL, de, "pointer")
        expect(L.psm_read_costs(h, 0, ptr(plane), W * 4 - 1), capi.PSM_EINVAL, de, "step")
        expect(L.psm_read_costs(h, 0, ptr(plane), W * 4), capi.PSM_ESTATE, de, "no costs")
        assert de.launch_count() == n1 and (plane == 7.0).all() and bool((dev == 7.0).all())
        de.DispSelect_GPU()
        lc, rc = de.lCosts.copy(), de.rCosts.copy()
        capi.check(L.psm_copy_costs_device(h, dev[0].data_ptr(), dev[1].data_ptr(), W * 4), h)
        de.sync()
        assert_bits(dev[0].cpu().numpy(), lc.view(U32), "device copy left")
        assert_bits(dev[1].cpu().numpy(), rc.view(U32), "device copy right")
        # a bad value changes nothing
        expect(L.psm_set_option(h, capi.PSM_OPT_COSTS, 3), capi.PSM_EINVAL, de, "PSM_OPT_COSTS")
        capi.check(L.psm_read_costs(h, 1, ptr(plane), W * 4), h)
        assert_bits(plane, rc.view(U32), "after a rejected value")
        # the post-filter and the left-right check do not change them
        de.setLRCheck(capi.PSM_LR_FILL_WMF)
        de.PostProcess_GPU()
        capi.check(L.psm_read_costs(h, 0, ptr(plane), W * 4), h)
        assert_bits(plane, lc.view(U32), "after the post-process")
        # the same value again keeps the stages; a change resets them
        capi.check(L.psm_set_option(h, capi.PSM_OPT_COSTS, 1), h)
        capi.check(L.psm_read_costs(h, 0, ptr(plane), W * 4), h)
        de.setCostOutput(False)
        expect(L.psm_read_costs(h, 0, ptr(plane), W * 4), capi.PSM_ESTATE, de, "PSM_OPT_COSTS")
        expect(L.psm_cost_filter(h), capi.PSM_ESTATE, de, "psm_cost_const")
        # a selection with the option off writes no costs
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        expect(L.psm_read_costs(h, 0, ptr(plane), W * 4), capi.PSM_ESTATE, de, "no costs")
    if "devices" not in kw:   # psm_disp_select_keys is rejected on multi-device contexts
        with DispEst(l, r, D, **kw) as de:
            h = de.handle
            de.setCostOutput(True)
            de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
            keys = torch.empty((2, H * W), dtype=torch.int64, device="cuda:0")
            capi.check(L.psm_disp_select_keys(h, keys[0].data_ptr(), keys[1].data_ptr()), h)
            expect(L.psm_read_costs(h, 0, ptr(plane), W * 4), capi.PSM_ESTATE, de, "no costs")


@pytest.mark.parametrize("kw", [{}, dict(block_slices=3), dict(devices=[0, 0]), dict(devices=[0, 0, 0], block_slices=2)])
def test_costs_outlive_the_next_filter(kw):
    """select frame f, then psm_cost_const and psm_cost_filter of frame f + 1: the costs and the selection maps are still
    frame f's on every context kind (a blocked walk tracks in planes of its own); the next select gives frame f + 1's"""
    import torch
    W, H, D = 96, 32, 12
    frames = [synth.stereo_pair_u8(W, H, D, seed=s)[:2] for s in (21, 22)]
    want = [run(l, r, D, **kw) for l, r in frames]
    assert not np.array_equal(want[0][2], want[1][2])
    L = capi.lib()
    dev = torch.full((2, 3, H, W), 7.0, device="cuda:0")
    maps = torch.zeros((2, H, W), dtype=torch.uint8, device="cuda:0")
    with DispEst(*frames[0], D, **kw) as de:
        h = de.handle
        de.setCostOutput(True)
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        de.setInputImages(*frames[1])
        de.CostConst_GPU(); de.CostFilter_GPU()
        capi.check(L.psm_copy_costs_device(h, dev[0].data_ptr(), dev[1].data_ptr(), W * 4), h)
        capi.check(L.psm_copy_maps_device(h, 0, maps[0].data_ptr(), W, maps[1].data_ptr(), W), h)
        de.sync()
        for v, side in ((0, "left"), (1, "right")):
            assert_same(maps[v].cpu().numpy(), want[0][v], f"{side} map after the next filter")
            assert_bits(dev[v].cpu().numpy(), want[0][2 + v].view(U32), f"{side} costs after the next filter")
            plane = np.empty((3, H, W), np.float32)
            capi.check(L.psm_read_costs(h, v, plane.ctypes.data_as(C.c_void_p), W * 4), h)
            assert_bits(plane, want[0][2 + v].view(U32), f"{side} costs read after the next filter")
        de.DispSelect_GPU()
        assert_bits(de.lCosts, want[1][2].view(U32), "left costs of frame f + 1")
        assert_bits(de.rCosts, want[1][3].view(U32), "right costs of frame f + 1")


def test_left_only_calls():
    import torch
    W, H, D = 64, 24, 12
    l, r, _ = synth.stereo_pair_u8(W, H, D, seed=2)
    L = capi.lib()
    plane = np.zeros((3, H, W), np.float32)
    dev = torch.zeros((2, 3, H, W), device="cuda:0")
    with DispEst(l, r, D) as de:
        h = de.handle
        de.setViews("left")
        de.setCostOutput(True)
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        assert de.rCosts is None
        expect(L.psm_copy_costs_device(h, dev[0].data_ptr(), dev[1].data_ptr(), W * 4), capi.PSM_EINVAL, de, "NULL")
        expect(L.psm_read_costs(h, 1, ptr(plane), W * 4), capi.PSM_ESTATE, de, "left-only")
        capi.check(L.psm_copy_costs_device(h, dev[0].data_ptr(), None, W * 4), h)
        de.sync()
        assert_bits(dev[0].cpu().numpy(), de.lCosts.view(U32), "left-only device copy")


@pytest.mark.parametrize("how", ["sharded", "u16 part", "blocked part"])
def test_partial_range_rejected(how):
    W, H, D = 32, 8, 12
    L = capi.lib()
    h = C.c_void_p()
    if how == "sharded":
        capi.check(L.psm_create_sharded(C.byref(h), W, H, D, 4, 8, 0))
    elif how == "u16 part":
        capi.check(L.psm_create_u16(C.byref(h), W, H, D, 0, 8, 0))
    else:
        capi.check(L.psm_create_blocked(C.byref(h), W, H, D, 0, 8, 2, 8, 0))
    try:
        assert L.psm_set_option(h, capi.PSM_OPT_COSTS, 1) == capi.PSM_EINVAL
        assert b"owns slices" in L.psm_last_error(h)
        assert L.psm_set_option(h, capi.PSM_OPT_COSTS, 0) == capi.PSM_OK   # the default stays settable
        assert L.psm_set_option(h, capi.PSM_OPT_COSTS, 1) == capi.PSM_EINVAL
    finally:
        L.psm_destroy(h)


def test_dispest_rejects_partial_range():
    l, r, _ = synth.stereo_pair_u8(32, 8, 12, seed=1)
    with DispEst(l, r, 12, d_begin=4, d_count=8) as de:
        with pytest.raises(capi.PsmError):
            de.setCostOutput(True)


# ---- TorchStereo ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [{}, dict(block_slices=5), dict(devices=[0, 0])])
def test_torch_held_back_stream(kw):
    import torch
    from primestereomatch_b200.torch_stereo import TorchStereo
    W, H, D = 160, 48, 24
    frames = [synth.stereo_pair_u8(W, H, D, seed=s)[:2] for s in (11, 12)]
    want = []
    for l, r in frames:
        lm, rm, lc, rc = run(l, r, D, **kw)
        want.append((lm, rm, lc.view(U32), rc.view(U32)))
    lsrc = torch.from_numpy(np.stack([f[0] for f in frames])).to("cuda:0")
    rsrc = torch.from_numpy(np.stack([f[1] for f in frames])).to("cuda:0")
    torch.cuda.synchronize()
    with TorchStereo(W, H, D, **kw) as ts:
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            lt, rt = torch.zeros_like(lsrc), torch.zeros_like(rsrc)
            torch.cuda._sleep(200_000_000)   # the frames are written only after the held-back work, on the same stream
            lt.copy_(lsrc)
            rt.copy_(rsrc)
            out = ts.match(lt, rt, costs=True)
            single = ts.match(lt[1], rt[1], costs=True)
            plain = ts.match(lt[0], rt[0])
        s.synchronize()
    assert len(out) == 4 and out[2].shape == (2, 3, H, W) and single[2].shape == (3, H, W) and len(plain) == 2
    for b in range(2):
        for k, what in enumerate(("left map", "right map", "left costs", "right costs")):
            got = out[k][b].cpu().numpy()
            assert_bits(got.view(U32) if k >= 2 else got, want[b][k], f"batch frame {b} {what}")
    for k in range(4):
        got = single[k].cpu().numpy()
        assert_bits(got.view(U32) if k >= 2 else got, want[1][k], f"single frame {k}")
    assert_same(plain[0].cpu().numpy(), want[0][0], "costs off again: left map")
