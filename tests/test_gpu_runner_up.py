"""GPU: the runner-up away from the winner (PSM_OPT_RUNNER_UP, psm_copy_runner_up_device, psm_read_runner_up).  Every
context kind (unblocked with 8- and 16-bit maps, blocked at B = 1, a B that does not divide D and B = D, multi-device
with co-located shards, unblocked and blocked, shards on two devices where they exist, left-only frames) returns, as
uint32 bit patterns, the definition (runner_up_cases.definition) applied to the oracle's filtered volume and map: the
scenes, the flagged kinds under the exact filter and the FGF, MIXED against its CPU model, the seam-tie frames.  The
unblocked context also equals the definition on its own volume bit for bit, and every other kind equals it.  Then the
maps and launches, both options together, the state rules, persistence through the next frame's stages, TorchStereo
with a held-back stream, and the intended use: OpenCV's uniqueness test from the planes against a brute force over the
oracle's volume."""
import ctypes as C

import numpy as np
import pytest

import cost_triple_cases as CT
import image_cases as IC
import mixed_model as MM
import runner_up_cases as RU
import test_gpu_selection_seams as SEAMS
from gif_cases import assert_same
from oracle import oracle as O
from output_checks import assert_bits, expect, frame_counts, ptr
from primestereomatch_b200 import DispEst, capi, synth

pytestmark = pytest.mark.gpu

U8, U16 = np.uint8, np.uint16


def run(l, r, D, dtype=U8, *, setup=None, fgf=None, left_only=False, volumes=False, costs=False, runner_up=True, **kw):
    """one frame -> dict: maps, runner (lRunnerUp, rRunnerUp), costs (lCosts, rCosts), and with volumes the filtered
    volumes the context selected from (an unblocked single-device context)"""
    with DispEst(l, r, D, map_bits=8 * np.dtype(dtype).itemsize, **kw) as de:
        if setup:
            setup(de)
        if left_only:
            de.setViews("left")
        if runner_up:
            de.setRunnerUpOutput(True)
        if costs:
            de.setCostOutput(True)
        assert de.CostConst_GPU() == 0
        if fgf:
            de.setSubsampleRate(fgf)
            assert de.CostFilter_FGF_GPU() == 0
        else:
            assert de.CostFilter_GPU() == 0
        assert de.DispSelect_GPU() == 0
        out = dict(maps=(de.lDisMap.copy(), None if de.rDisMap is None else de.rDisMap.copy()),
                   runner=(de.lRunnerUp, de.rRunnerUp), costs=(de.lCosts, de.rCosts))
        if volumes:
            out["vols"] = tuple(de.read_cost_volume(v) for v in range(1 if left_only else 2))
        return out


def contexts(D, shard_block=3):
    ragged = next((b for b in (7, 5, 3, 2) if b < D and D % b), None)
    blocks = tuple(b for b in (1, ragged, D) if b)
    return SEAMS.contexts(D, blocks=blocks, shards=(2, 3), shard_block=shard_block)


def check(l, r, D, vols, what, dtype=U8, cases=None, left_only=False, **kw):
    """every context's maps equal O.wta of vols and its runner-up equals the definition on vols (NaN payloads aside).
    The first case is the unblocked context: it equals the definition on its own volumes bit for bit, payloads
    included, and every other context equals it bit for bit."""
    maps = [O.wta(v, dtype) for v in vols]
    want = [RU.definition(v, m) for v, m in zip(vols, maps)]
    cases = contexts(D) if cases is None else cases
    assert cases[0][1] == {}
    ref = None
    for name, ctx, _ in cases:
        got = run(l, r, D, dtype, left_only=left_only, volumes=ref is None, **ctx, **kw)
        views = ((0, "left"),) if left_only else ((0, "left"), (1, "right"))
        if left_only:
            assert got["maps"][1] is None and got["runner"][1] is None
        for v, side in views:
            assert_same(got["maps"][v], maps[v], f"{what}, {name}: {side} map")
            assert_bits(got["runner"][v], want[v], f"{what}, {name}: {side} runner-up vs the oracle", nan_any=True)
            if ref is None:
                assert_bits(got["runner"][v], RU.definition(got["vols"][v], got["maps"][v]),
                            f"{what}: {side} runner-up vs the device's own volume")
            else:
                assert_bits(got["runner"][v], ref["runner"][v], f"{what}, {name}: {side} runner-up vs the unblocked context's")
        ref = ref or got
    return maps, want


SCENE_CASES = [("unblocked", {}, None), ("B=1", dict(block_slices=1), None), ("B=7", dict(block_slices=7), None),
               ("B=64", dict(block_slices=64), None), ("2 shards", dict(devices=[0, 0]), None),
               ("3 shards B=5", dict(devices=[0, 0, 0], block_slices=5), None)]


# ---- the scenes, u8 and float frames --------------------------------------------------------------------------------------
@pytest.mark.parametrize("u8", [True, False])
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_scenes(scene, u8, scenes, oracle_scene_results):
    l8, r8, l, r = scenes[scene]
    res = oracle_scene_results[scene]
    frame = (l8, r8) if u8 else (l, r)
    _, want = check(*frame, 64, (res["lf"], res["rf"]), f"{scene} u8={u8}", cases=SCENE_CASES)
    assert (want[0][0].view(np.float32) > 0).mean() > 0.9


# ---- flagged kinds: +-inf, NaN, FLT_MAX; exact filter, FGF and MIXED -------------------------------------------------------
@pytest.mark.parametrize("kind", IC.FLAGGED)
def test_flagged_exact(kind):
    W, H, D = IC.MAIN
    l, r = IC.frame(kind, W, H, D)
    check(l, r, D, SEAMS.filtered(l, r, D), f"{kind} exact")


@pytest.mark.parametrize("kind", ["nan", "posinf", "fltmax"])
def test_flagged_fgf(kind):
    W, H, D = IC.MAIN
    l, r = IC.frame(kind, W, H, D)
    check(l, r, D, SEAMS.filtered(l, r, D, fgf=4), f"{kind} FGF", fgf=4)


def test_mixed():
    W, H, D = 227, 61, 40
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=5)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    _, _, lraw, rraw = O.cost_const(l, r, D)
    vols = (MM.cost_filter_mixed(O, l, lraw), MM.cost_filter_mixed(O, r, rraw))
    check(l, r, D, vols, "MIXED", setup=lambda de: de.set_option(capi.PSM_OPT_CVF_MODE, capi.PSM_CVF_MIXED))


def test_wide_u16():
    l, r = IC.wide_frame("nan")
    W, H, D = IC.WIDE
    maps, _ = check(l, r, D, SEAMS.filtered(l, r, D), "nan D=300", U16,
                    cases=SEAMS.contexts(D, blocks=(7, 128, D), shards=(2,), shard_block=7))
    assert int(maps[0].max()) > 255


def test_left_only():
    W, H, D = IC.MAIN
    l, r = IC.frame("nan", W, H, D)
    check(l, r, D, SEAMS.filtered(l, r, D), "left-only nan", left_only=True)


# ---- exact ties across the seams, tiny ranges ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SEAMS.TIES))
def test_ties_across_seams(name):
    make, D, dtype = SEAMS.TIES[name]
    l8, r8 = make()
    check(l8, r8, D, SEAMS.filtered(O.u8_to_f32(l8), O.u8_to_f32(r8), D), name, dtype)


@pytest.mark.parametrize("D", [2, 3, 4])
def test_tiny_ranges(D):
    """D <= 3 has no runner-up anywhere; D = 4 only where m = 1 and r = 3 or m = 3 and r = 1"""
    W, H = 43, 13
    rng = np.random.default_rng([W, H, D])
    base = rng.integers(0, 256, (H, W + 2, 3), dtype=U8)
    l8, r8 = np.ascontiguousarray(base[:, 2:]), np.ascontiguousarray(base[:, :W])
    _, want = check(l8, r8, D, SEAMS.filtered(O.u8_to_f32(l8), O.u8_to_f32(r8), D), f"D={D}",
                    cases=contexts(D, shard_block=1))
    if D <= 3:
        assert (want[0][0] == 0).all() and (want[0][1] == 0x7FC00000).all()


def test_distinct_devices():
    if capi.lib().psm_device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    W, H, D = IC.MAIN
    l, r = IC.frame("nan", W, H, D)
    cases = [("unblocked", {}, None), ("[0, 1]", dict(devices=[0, 1]), None),
             ("[0, 1] B=2", dict(devices=[0, 1], block_slices=2), None)]
    check(l, r, D, SEAMS.filtered(l, r, D), "nan on [0, 1]", cases=cases)


# ---- maps, launches, both options ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw,extra", [({}, 0), (dict(block_slices=7), 2), (dict(devices=[0, 0]), 6),
                                      (dict(devices=[0, 0, 0], block_slices=4), 8)])
def test_launches_and_maps(kw, extra):
    """off: a context that had the option on and off again launches and selects as one that never had it.  On: the same
    maps; an unblocked context selects in the kernel it launches anyway, a blocked one adds one pick per view, a
    multi-device one a pick per view and shard and one slot reduce per view"""
    W, H, D = 200, 40, 50
    l, r, _ = synth.stereo_pair_u8(W, H, D, seed=4)
    with DispEst(l, r, D, **kw) as plain, DispEst(l, r, D, **kw) as toggled:
        toggled.setRunnerUpOutput(True)
        toggled.setRunnerUpOutput(False)
        base = frame_counts(plain)
        off = frame_counts(toggled)
        assert off[0] == base[0]
        assert_same(off[1], base[1], "off: left"); assert_same(off[2], base[2], "off: right")
        toggled.setRunnerUpOutput(True)
        on = frame_counts(toggled)
        assert on[0] == [base[0][0], base[0][1], base[0][2] + extra], (on[0], base[0])
        assert_same(on[1], base[1], "on: left"); assert_same(on[2], base[2], "on: right")


@pytest.mark.parametrize("kw", [{}, dict(block_slices=5), dict(devices=[0, 0]), dict(devices=[0, 0, 0], block_slices=2)])
def test_both_options(kw):
    W, H, D = 120, 32, 24
    l, r = IC.frame("nan", W, H, D)
    both = run(l, r, D, costs=True, **kw)
    alone = run(l, r, D, **kw)
    costs = run(l, r, D, costs=True, runner_up=False, **kw)
    for v in range(2):
        assert_same(both["maps"][v], alone["maps"][v], f"view {v} maps")
        assert_bits(both["runner"][v], alone["runner"][v], f"view {v} runner-up with the costs on")
        assert_bits(both["costs"][v], costs["costs"][v], f"view {v} costs with the runner-up on")
    # stage 3 adds both options' launches: the costs one write per view and shard, the runner-up one pick per view on a
    # blocked context, and a pick per view and shard plus one slot reduce per view on a multi-device one (the extras
    # test_launches_and_maps pins here and in test_gpu_costs)
    shards = len(kw.get("devices", [0]))
    costs_extra = 2 * shards
    runner_up_extra = 2 * shards + 2 if "devices" in kw else 2 if kw.get("block_slices") else 0
    with DispEst(l, r, D, **kw) as plain, DispEst(l, r, D, **kw) as de:
        de.setCostOutput(True)
        de.setRunnerUpOutput(True)
        base, on = frame_counts(plain)[0], frame_counts(de)[0]
    assert on == [base[0], base[1], base[2] + costs_extra + runner_up_extra], (on, base)


# ---- state rules ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [{}, dict(block_slices=4), dict(devices=[0, 0])])
def test_state_rules(kw):
    import torch
    W, H, D = 64, 24, 12
    l, r, _ = synth.stereo_pair_u8(W, H, D, seed=2)
    L = capi.lib()
    plane = np.full((2, H, W), 7.0, np.float32)
    dev = torch.full((2, 2, H, W), 7.0, device="cuda:0")
    with DispEst(l, r, D, **kw) as de:
        h = de.handle
        expect(L.psm_read_runner_up(h, 0, ptr(plane), W * 4), capi.PSM_ESTATE, de, "no runner-up")
        for bad in (2, -1):
            expect(L.psm_set_option(h, capi.PSM_OPT_RUNNER_UP, bad), capi.PSM_EINVAL, de, "PSM_OPT_RUNNER_UP")
        de.setRunnerUpOutput(True)
        de.CostConst_GPU(); de.CostFilter_GPU()
        n1 = de.launch_count()
        expect(L.psm_copy_runner_up_device(h, None, dev[1].data_ptr(), W * 4), capi.PSM_EINVAL, de, "pointer")
        expect(L.psm_copy_runner_up_device(h, dev[0].data_ptr(), None, W * 4), capi.PSM_EINVAL, de, "pointer")
        expect(L.psm_copy_runner_up_device(h, dev[0].data_ptr(), dev[1].data_ptr(), W * 4 - 4), capi.PSM_EINVAL, de, "step")
        expect(L.psm_read_runner_up(h, 2, ptr(plane), W * 4), capi.PSM_EINVAL, de, "view")
        expect(L.psm_read_runner_up(h, 0, None, W * 4), capi.PSM_EINVAL, de, "pointer")
        expect(L.psm_read_runner_up(h, 0, ptr(plane), W * 4 - 1), capi.PSM_EINVAL, de, "step")
        expect(L.psm_read_runner_up(h, 0, ptr(plane), W * 4), capi.PSM_ESTATE, de, "no runner-up")
        assert de.launch_count() == n1 and (plane == 7.0).all() and bool((dev == 7.0).all())
        de.DispSelect_GPU()
        lu, ru = de.lRunnerUp.copy(), de.rRunnerUp.copy()
        capi.check(L.psm_copy_runner_up_device(h, dev[0].data_ptr(), dev[1].data_ptr(), W * 4), h)
        de.sync()
        assert_bits(dev[0].cpu().numpy(), lu, "device copy left")
        assert_bits(dev[1].cpu().numpy(), ru, "device copy right")
        expect(L.psm_set_option(h, capi.PSM_OPT_RUNNER_UP, 3), capi.PSM_EINVAL, de, "PSM_OPT_RUNNER_UP")
        capi.check(L.psm_read_runner_up(h, 1, ptr(plane), W * 4), h)
        assert_bits(plane, ru, "after a rejected value")
        de.setLRCheck(capi.PSM_LR_FILL_WMF)
        de.PostProcess_GPU()
        capi.check(L.psm_read_runner_up(h, 0, ptr(plane), W * 4), h)
        assert_bits(plane, lu, "after the post-process")
        capi.check(L.psm_set_option(h, capi.PSM_OPT_RUNNER_UP, 1), h)   # the same value keeps the stages
        capi.check(L.psm_read_runner_up(h, 0, ptr(plane), W * 4), h)
        de.setCostOutput(True)   # another option's change resets them too
        expect(L.psm_read_runner_up(h, 0, ptr(plane), W * 4), capi.PSM_ESTATE, de, "psm_cost_const")
        de.setCostOutput(False)
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        capi.check(L.psm_read_runner_up(h, 0, ptr(plane), W * 4), h)
        assert_bits(plane, lu, "selected again")
        de.setRunnerUpOutput(False)
        expect(L.psm_read_runner_up(h, 0, ptr(plane), W * 4), capi.PSM_ESTATE, de, "PSM_OPT_RUNNER_UP")
        expect(L.psm_cost_filter(h), capi.PSM_ESTATE, de, "psm_cost_const")
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        expect(L.psm_read_runner_up(h, 0, ptr(plane), W * 4), capi.PSM_ESTATE, de, "no runner-up")
    if "devices" not in kw:   # psm_disp_select_keys is rejected on multi-device contexts
        with DispEst(l, r, D, **kw) as de:
            h = de.handle
            de.setRunnerUpOutput(True)
            de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
            keys = torch.empty((2, H * W), dtype=torch.int64, device="cuda:0")
            capi.check(L.psm_disp_select_keys(h, keys[0].data_ptr(), keys[1].data_ptr()), h)
            expect(L.psm_read_runner_up(h, 0, ptr(plane), W * 4), capi.PSM_ESTATE, de, "no runner-up")


@pytest.mark.parametrize("kw", [{}, dict(block_slices=3), dict(devices=[0, 0]), dict(devices=[0, 0, 0], block_slices=2)])
def test_runner_up_outlives_the_next_filter(kw):
    """select frame f, then psm_cost_const and psm_cost_filter of frame f + 1: the runner-up is still frame f's on every
    context kind; the next select gives frame f + 1's"""
    import torch
    W, H, D = 96, 32, 12
    frames = [synth.stereo_pair_u8(W, H, D, seed=s)[:2] for s in (21, 22)]
    want = [run(l, r, D, **kw)["runner"] for l, r in frames]
    assert not np.array_equal(want[0][0], want[1][0])
    L = capi.lib()
    dev = torch.full((2, 2, H, W), 7.0, device="cuda:0")
    with DispEst(*frames[0], D, **kw) as de:
        h = de.handle
        de.setRunnerUpOutput(True)
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        de.setInputImages(*frames[1])
        de.CostConst_GPU(); de.CostFilter_GPU()
        capi.check(L.psm_copy_runner_up_device(h, dev[0].data_ptr(), dev[1].data_ptr(), W * 4), h)
        de.sync()
        for v in range(2):
            assert_bits(dev[v].cpu().numpy(), want[0][v], f"view {v} runner-up after the next filter")
            plane = np.empty((2, H, W), np.float32)
            capi.check(L.psm_read_runner_up(h, v, ptr(plane), W * 4), h)
            assert_bits(plane, want[0][v], f"view {v} runner-up read after the next filter")
        de.DispSelect_GPU()
        assert_bits(de.lRunnerUp, want[1][0], "left runner-up of frame f + 1")
        assert_bits(de.rRunnerUp, want[1][1], "right runner-up of frame f + 1")


def test_left_only_calls():
    import torch
    W, H, D = 64, 24, 12
    l, r, _ = synth.stereo_pair_u8(W, H, D, seed=2)
    L = capi.lib()
    plane = np.zeros((2, H, W), np.float32)
    dev = torch.zeros((2, 2, H, W), device="cuda:0")
    with DispEst(l, r, D) as de:
        h = de.handle
        de.setViews("left")
        de.setRunnerUpOutput(True)
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        assert de.rRunnerUp is None
        expect(L.psm_copy_runner_up_device(h, dev[0].data_ptr(), dev[1].data_ptr(), W * 4), capi.PSM_EINVAL, de, "NULL")
        expect(L.psm_read_runner_up(h, 1, ptr(plane), W * 4), capi.PSM_ESTATE, de, "left-only")
        capi.check(L.psm_copy_runner_up_device(h, dev[0].data_ptr(), None, W * 4), h)
        de.sync()
        assert_bits(dev[0].cpu().numpy(), de.lRunnerUp, "left-only device copy")


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
        assert L.psm_set_option(h, capi.PSM_OPT_RUNNER_UP, 1) == capi.PSM_EINVAL
        assert b"owns slices" in L.psm_last_error(h)
        assert L.psm_set_option(h, capi.PSM_OPT_RUNNER_UP, 0) == capi.PSM_OK
        assert L.psm_set_option(h, capi.PSM_OPT_RUNNER_UP, 1) == capi.PSM_EINVAL
    finally:
        L.psm_destroy(h)


# ---- TorchStereo -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [{}, dict(block_slices=5), dict(devices=[0, 0])])
def test_torch_held_back_stream(kw):
    import torch
    from primestereomatch_b200.torch_stereo import TorchStereo
    W, H, D = 160, 48, 24
    frames = [synth.stereo_pair_u8(W, H, D, seed=s)[:2] for s in (11, 12)]
    want = []
    for l, r in frames:
        o = run(l, r, D, costs=True, **kw)
        want.append(o["maps"] + o["costs"] + o["runner"])
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
            out = ts.match(lt, rt, costs=True, runner_up=True)
            single = ts.match(lt[1], rt[1], runner_up=True)
            plain = ts.match(lt[0], rt[0])
        s.synchronize()
    assert len(out) == 6 and out[4].shape == (2, 2, H, W) and len(single) == 4 and single[2].shape == (2, H, W)
    assert len(plain) == 2
    for b in range(2):
        for k in range(6):
            assert_bits(out[k][b].cpu().numpy(), want[b][k], f"batch frame {b} output {k}")
    for k, w in ((0, 0), (1, 1), (2, 4), (3, 5)):
        assert_bits(single[k].cpu().numpy(), want[1][w], f"single frame output {k}")
    assert_same(plain[0].cpu().numpy(), want[0][0], "runner-up off again: left map")


# ---- the intended use, outside the library -----------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [{}, dict(block_slices=16), dict(devices=[0, 0])])
def test_uniqueness_mask(kw, scenes, oracle_scene_results):
    """OpenCV's uniqueness test at ratios 5, 10 and 15 from the runner-up planes, the map and q(m) (PSM_OPT_COSTS' middle
    plane) equals a brute force over every d with |d - m| > 1 on the oracle's volume"""
    l8, r8, _, _ = scenes["Cones"]
    res = oracle_scene_results["Cones"]
    got = run(l8, r8, 64, costs=True, **kw)
    for v, vol in enumerate((res["lf"], res["rf"])):
        m = got["maps"][v]
        for u in (5, 10, 15):
            mask = RU.uniqueness_from_planes(got["runner"][v], got["costs"][v][1], u)
            brute = RU.uniqueness_brute(vol, m, u)
            assert np.array_equal(mask, brute), (v, u, int((mask != brute).sum()))
            assert 0.05 < mask.mean() < 1.0
