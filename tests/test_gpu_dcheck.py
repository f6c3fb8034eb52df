"""GPU: the one-view disparity check (psm_set_disparity_check) bit for bit through the C-ABI against the CPU
restatement tests/dcheck_oracle.py (pinned to cv2.validateDisparity by golden_dcheck.json), applied to each context's
own selection maps and psm_read_costs plane 1: every mode with every speckle mode, left-right check mode and
post-filter setting, every kind of context against the unblocked one, the left-only fill, rows wider than shared
memory, the selection's outputs left untouched, launch counts, argument and state checks, TorchStereo and the C++
demo."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from primestereomatch_b200 import DispEst, capi, synth
import dcheck_oracle as DC
import lr_oracle as LR
import pp_chain as PP
import speckle_oracle as SP

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN, "golden_dcheck.json")) as f:
    GOLD = json.load(f)
OFF, FIRST, ONLY = capi.PSM_DCHECK_OFF, capi.PSM_DCHECK_FIRST, capi.PSM_DCHECK_ONLY
GENERIC = (3, 25.5, 2, "iv1")
DEFAULT = (9, 25.5, 1, "exp")


def assert_same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, f"{what}: shape {a.shape} vs {b.shape}"
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {a.size} differ, first at {list(i)}: {a[i]!r} vs {b[i]!r}")


def noisy_pair(W, H, D, seed):
    """a synthetic pair with noise on the right view, so the maps hold mismatches for the check to find"""
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=seed)
    rng = np.random.default_rng(seed)
    r8 = np.clip(r8.astype(np.int16) + rng.integers(-40, 41, r8.shape), 0, 255).astype(np.uint8)
    return synth.to_f32(l8), synth.to_f32(r8)


def select(de):
    """one frame with the costs on -> (ld, rd or None, lc, rc or None): the selection maps and plane 1 of the costs"""
    de.setCostOutput(True)
    assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0 and de.DispSelect_GPU() == 0
    rd = None if de.rDisMap is None else de.rDisMap.copy()
    return de.lDisMap.copy(), rd, de.lCosts[1].copy(), None if rd is None else de.rCosts[1].copy()


def post(de, dcheck, speckle=(0, 0, 0), lr=0, setting=DEFAULT):
    de.setDisparityCheck(*dcheck); de.setSpeckleFilter(*speckle); de.setLRCheck(lr); de.setPostFilter(*setting)
    assert de.PostProcess_GPU() == 0
    return de.lDisMap.copy(), None if de.rDisMap is None else de.rDisMap.copy()


def want(l, r, sel, D, dcheck, speckle=(0, 0, 0), lr=0, setting=DEFAULT):
    ld, rd, lc, rc = sel
    return PP.chain(l, r, ld, rd, dcheck=dcheck, costs=(lc, rc), D=D, speckle=speckle, lr=lr, setting=setting)


def check_against(de, l, r, sel, D, what, **kw):
    got = post(de, **kw)
    ref = want(l, r, sel, D, **kw)
    assert_same(got[0], ref[0], what + " left")
    if sel[1] is not None:
        assert_same(got[1], ref[1], what + " right")
    return got, ref


# ---- cv2's own results ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_full_scenes_against_the_golden(scene, scenes, oracle_scene_results):
    _, _, l, r = scenes[scene]
    ref = oracle_scene_results[scene]
    g = GOLD["scenes"][scene]
    with DispEst(l, r, 64) as de:
        sel = select(de)
        assert_same(sel[0], ref["ld"], "WTA left"); assert_same(sel[1], ref["rd"], "WTA right")
        # the device's costs are the oracle's filtered volume at each winner
        assert sel[2].tobytes() == DC.winner_costs(ref["lf"], ref["ld"]).tobytes()
        for sl, sr in zip(g["l"], g["r"]):
            gl, gr = post(de, (ONLY, sl["max_diff"]))
            assert [SP.sha(gl), SP.sha(gr)] == [sl["sha"], sr["sha"]], (scene, sl["max_diff"])
        oracle_sel = (ref["ld"], ref["rd"], DC.winner_costs(ref["lf"], ref["ld"]), DC.winner_costs(ref["rf"], ref["rd"]))
        for lr in (2, 1):
            got = post(de, (FIRST, 1), (1, 100, 32), lr)
            exp = want(l, r, oracle_sel, 64, (FIRST, 1), (1, 100, 32), lr)
            assert_same(got[0], exp[0], f"{scene} first + speckle + lr {lr} left")
            assert_same(got[1], exp[1], f"{scene} first + speckle + lr {lr} right")


# ---- the chain: every mode with every speckle mode, check mode and post-filter setting ------------------------------------
@pytest.mark.parametrize("bits", [8, 16])
def test_every_mode_with_every_speckle_and_check_mode(bits):
    W, H, D = (140, 48, 48) if bits == 8 else (400, 32, 300)
    l, r = noisy_pair(W, H, 48, seed=3)
    with DispEst(l, r, D, map_bits=bits) as de:
        sel = select(de)
        assert (DC.check(sel[0], sel[2], D, 0) != sel[0]).any(), "the maps have nothing for the check to remove"
        for setting in (DEFAULT, GENERIC):
            for dc in ((FIRST, 1), (ONLY, 0), (FIRST, 0)):
                for sp in ((0, 0, 0), (1, 6, 1), (2, 6, 1)):
                    for lr in (0, 1, 2):
                        what = f"u{bits} dcheck {dc} speckle {sp} lr {lr} {setting}"
                        _, ref = check_against(de, l, r, sel, D, what, dcheck=dc, speckle=sp, lr=lr, setting=setting)
                        ran = lr and dc[0] != ONLY and sp[0] != 2
                        if ran:
                            lv, rv = ref[2]
                            assert_same(de.lValid, lv, what + " left mask"); assert_same(de.rValid, rv, what + " right mask")


def test_rows_wider_than_shared_memory():
    """W > 6144: the claims live in global scratch"""
    W, H, D = 7000, 12, 40
    l, r = noisy_pair(W, H, D, seed=21)
    with DispEst(l, r, D) as de:
        sel = select(de)
        for diff in (0, 1, 3):
            got, ref = check_against(de, l, r, sel, D, f"wide rows max_diff {diff}", dcheck=(ONLY, diff))
            assert (got[0] != sel[0]).any()
        check_against(de, l, r, sel, D, "wide rows first + fill", dcheck=(FIRST, 1), lr=2)


# ---- every kind of context against the unblocked one; the selection's outputs stay as they were ------------------------
KINDS = [("unblocked", {}), ("blocked B=1", {"block_slices": 1}), ("blocked B=7", {"block_slices": 7}),
         ("blocked B=D", {"block_slices": 64}), ("range", {"min_disp": 9}), ("left-only", {}),
         ("multi-2", {"devices": [0, 0]}), ("multi-3-blocked", {"devices": [0, 0, 0], "block_slices": 8}),
         ("multi-3", {"devices": [0, 0, 0]}), ("multi-2-blocked", {"devices": [0, 0], "block_slices": 5})]


@pytest.fixture(scope="module")
def unblocked_results():
    """the unblocked context's selection and check results on the kinds' frame"""
    W, H, D = 200, 64, 64
    l, r = noisy_pair(W, H, D, seed=8)
    with DispEst(l, r, D) as de:
        sel = select(de)
        return l, r, sel, post(de, (ONLY, 1)), post(de, (FIRST, 1), (1, 20, 1), 1)


@pytest.mark.parametrize("kind,kw", KINDS, ids=[k for k, _ in KINDS])
def test_context_kinds(kind, kw, unblocked_results):
    l, r, sel0, only0, first0 = unblocked_results
    D = 64
    L = capi.lib()
    left_only = kind == "left-only"
    with DispEst(l, r, D, **kw) as de:
        if left_only:
            de.setViews("left")
        de.setRunnerUpOutput(True)
        sel = select(de)
        costs, runner = (de.lCosts, de.rCosts), (de.lRunnerUp, de.rRunnerUp)
        got_only = check_against(de, l, r, sel, D, f"{kind} only", dcheck=(ONLY, 1))[0]
        got_first = check_against(de, l, r, sel, D, f"{kind} first", dcheck=(FIRST, 1), speckle=(1, 20, 1),
                                  lr=1)[0]
        if kind != "range":                       # the same maps as the unblocked context's
            assert_same(sel[0], sel0[0], f"{kind} selection"); assert_same(got_only[0], only0[0], f"{kind} only left")
            if not left_only:
                assert_same(got_only[1], only0[1], f"{kind} only right")
                assert_same(got_first[0], first0[0], f"{kind} first left")
        # the selection's maps, costs and runner-up are the selection's
        for got, was in ((de._read_output(L.psm_read_costs, 3), costs), (de._read_output(L.psm_read_runner_up, 2), runner)):
            for v in (0,) if left_only else (0, 1):
                assert got[v].tobytes() == was[v].tobytes(), f"{kind} costs / runner-up of view {v} changed"
        assert de.stage_ms(5) > 0


@pytest.mark.parametrize("bits,D", [(16, 300), (8, 64)])
def test_u16_and_blocked_against_unblocked(bits, D):
    W, H = 420, 40
    l, r = noisy_pair(W, H, 64, seed=30)
    results = []
    for kw in ({}, {"block_slices": 7}, {"devices": [0, 0]}):
        with DispEst(l, r, D, map_bits=bits, **kw) as de:
            sel = select(de)
            got = check_against(de, l, r, sel, D, f"u{bits} D={D} {kw}", dcheck=(FIRST, 2), lr=2)[0]
            results.append((sel[0], got[0], got[1]))
    for k in (1, 2):
        for a, b in zip(results[0], results[k]):
            assert_same(b, a, f"u{bits} kind {k} against unblocked")


# ---- the left-only fill -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [8, 16])
def test_left_only_fill(bits):
    W, H, D = 180, 50, 40
    l, r = noisy_pair(W, H, D, seed=17)
    L = capi.lib()
    mask = np.zeros((H, W), np.uint8)
    with DispEst(l, r, D, map_bits=bits) as de:
        de.setViews("left")
        sel = select(de)
        for lr in (1, 2):
            for setting in (DEFAULT, GENERIC):
                for sp in ((0, 0, 0), (1, 10, 1)):
                    got, ref = check_against(de, l, r, sel, D, f"left-only lr {lr} {sp} {setting}", dcheck=(FIRST, 1),
                                             speckle=sp, lr=lr, setting=setting)
                    assert_same(de.lValid, ref[2][0], f"left-only mask lr {lr} {sp}")
        assert L.psm_read_valid_mask(de.handle, capi.PSM_RIGHT, mask.ctypes.data, W) == capi.PSM_ESTATE
        # ONLY runs no fill: no mask; without the check the two-view check's PSM_ESTATE stays
        de.setDisparityCheck(ONLY, 1)
        assert de.PostProcess_GPU() == 0
        assert L.psm_read_valid_mask(de.handle, capi.PSM_LEFT, mask.ctypes.data, W) == capi.PSM_ESTATE
        de.setDisparityCheck(OFF, 1)
        with pytest.raises(capi.PsmError) as e:
            de.PostProcess_GPU()
        assert e.value.code == capi.PSM_ESTATE


class DeviceArray:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 3}


def device_bytes(torch, de, what, n):
    p, pitch = C.c_void_p(), C.c_size_t()
    capi.check(capi.lib().psm_device_ptr(de.handle, what, C.byref(p), C.byref(pitch)), de.handle)
    return p.value, torch.as_tensor(DeviceArray(p.value, n), device="cuda")


@pytest.mark.parametrize("bits", [8, 16])
def test_left_only_fill_leaves_the_right_view_untouched(bits):
    """the right selection map, post-processed map and mask (selectors 3, 5, 7) keep a pattern through left-only
    frames that check and fill, in both fill modes"""
    torch = pytest.importorskip("torch")
    W, H, D = 150, 40, 32
    l, r = noisy_pair(W, H, D, seed=19)
    nbytes = H * W * (2 if bits == 16 else 1)
    with DispEst(l, r, D, map_bits=bits) as de:
        select(de)
        post(de, (OFF, 1), lr=1)                                           # allocates the right buffers
        de.sync()
        bufs = {w: device_bytes(torch, de, w, n) for w, n in ((3, nbytes), (5, nbytes), (7, H * W))}
        de.setViews("left")
        pattern = torch.arange(nbytes, device="cuda", dtype=torch.int64).remainder(251).to(torch.uint8)
        for _, t in bufs.values():
            t.copy_(pattern[:t.numel()])
        torch.cuda.synchronize()
        for lr in (2, 1):
            sel = select(de)
            check_against(de, l, r, sel, D, f"left-only lr {lr}", dcheck=(FIRST, 1), lr=lr)
        de.sync()
        for w, (addr, t) in bufs.items():
            assert device_bytes(torch, de, w, 1)[0] == addr, f"psm_device_ptr {w} moved"
            assert torch.equal(t, pattern[:t.numel()]), f"psm_device_ptr {w}: a left-only fill wrote the right view"


# ---- launches, arguments and state --------------------------------------------------------------------------------------
def test_launch_counts_and_stage_time():
    l, r = noisy_pair(64, 48, 16, seed=11)
    with DispEst(l, r, 16) as de:
        select(de)
        for dc in (OFF, FIRST, ONLY):
            for sp in (0, 1, 2):
                for lr in (0, 1, 2):
                    for it in (1, 3):
                        de.setDisparityCheck(dc, 1); de.setSpeckleFilter(sp, 5, 1); de.setLRCheck(lr)
                        de.setPostFilter(9, 25.5, it, "exp")
                        n = de.launch_count()
                        assert de.PostProcess_GPU() == 0
                        base = {0: 4 * it, 1: 1 + 4 * it, 2: 1}[lr]
                        base = {0: base, 1: 4 + base, 2: 4}[sp]
                        assert de.launch_count() - n == {OFF: base, FIRST: 1 + base, ONLY: 1}[dc], (dc, sp, lr, it)
                        assert de.stage_ms(5) > 0


def test_invalid_arguments_and_states():
    W, H, D = 90, 40, 16
    l, r = noisy_pair(W, H, D, seed=2)
    L = capi.lib()
    with DispEst(l, r, D) as de:
        h = de.handle
        sel = select(de)
        de.setLRCheck(2)
        good = post(de, (FIRST, 1), lr=2)
        for mode, diff in ((-1, 1), (3, 1), (FIRST, -1), (ONLY, 4096), (OFF, -1), (OFF, 4096)):
            assert L.psm_set_disparity_check(h, mode, diff) == capi.PSM_EINVAL and L.psm_last_error(h), (mode, diff)
            assert de.PostProcess_GPU() == 0
            assert_same(de.lDisMap, good[0], f"left after rejected ({mode}, {diff})")
        assert L.psm_set_disparity_check(None, FIRST, 1) == capi.PSM_EINVAL
        with pytest.raises(capi.PsmError):
            de.setDisparityCheck(FIRST, 5000)
        assert L.psm_set_disparity_check(h, ONLY, 4095) == 0
        assert_same(post(de, (ONLY, 4095), lr=2)[0], sel[0], "max_diff 4095 removes nothing")
        # costs are required: a selection without them refuses the stage and names the option
        de.setCostOutput(False)
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        with pytest.raises(capi.PsmError) as e:
            post(de, (FIRST, 1), lr=2)
        assert e.value.code == capi.PSM_ESTATE and b"PSM_OPT_COSTS" in L.psm_last_error(h)
        assert_same(post(de, (OFF, 1), lr=2)[0], LR.lr_check_fill(sel[0], sel[1])[2], "off after the refusal")
    # a context owning part of the range takes OFF alone; a multi-device context forwards to every shard
    with DispEst(l, r, D, d_begin=0, d_count=8) as de:
        assert L.psm_set_disparity_check(de.handle, FIRST, 1) == capi.PSM_EINVAL
        assert L.psm_set_disparity_check(de.handle, OFF, 1) == 0
    with DispEst(l, r, D, devices=[0, 0]) as de:
        assert L.psm_set_disparity_check(de.handle, 5, 1) == capi.PSM_EINVAL
        sel = select(de)
        check_against(de, l, r, sel, D, "multi after a rejected mode", dcheck=(ONLY, 2))


# ---- TorchStereo and the demo ------------------------------------------------------------------------------------------------
def test_torch_stereo_and_held_back_stream():
    import torch
    from primestereomatch_b200.torch_stereo import TorchStereo
    W, H, D = 160, 96, 48
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=13)
    rng = np.random.default_rng(13)
    r8 = np.clip(r8.astype(np.int16) + rng.integers(-40, 41, r8.shape), 0, 255).astype(np.uint8)
    lt, rt = torch.from_numpy(l8).cuda(), torch.from_numpy(r8).cuda()
    with TorchStereo(W, H, D) as ts:
        lm, rm, lc, rc = ts.match(lt, rt, costs=True)
        ld, rd, lq, rq = lm.cpu().numpy(), rm.cpu().numpy(), lc[1].cpu().numpy(), rc[1].cpu().numpy()
        ts.match(lt, rt)                                                    # costs off again
        assert ts.costs is False
        ts.setDisparityCheck(ONLY, 1)
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)                                   # the frames' stream is held back
            out = ts.match(lt, rt, post_process=True)
        torch.cuda.synchronize()
        assert len(out) == 2 and ts.costs is True                            # costs set for the check, not returned
        assert_same(out[0].cpu().numpy(), DC.check(ld, lq, D, 1), "TorchStereo only left")
        assert_same(out[1].cpu().numpy(), DC.check(rd, rq, D, 1, view=1), "TorchStereo only right")
        ts.setDisparityCheck(FIRST, 0); ts.setLRCheck(2)
        lm, rm, lc2, _ = ts.match(lt, rt, post_process=True, costs=True)
        exp = LR.lr_check_fill(DC.check(ld, lq, D, 0), DC.check(rd, rq, D, 0, view=1))
        assert_same(lm.cpu().numpy(), exp[2], "TorchStereo first + fill left")
        assert lc2[1].cpu().numpy().tobytes() == lq.tobytes()
        with pytest.raises(capi.PsmError):
            ts.setDisparityCheck(7, 1)


def test_cpp_demo_disp_check_flag(tmp_path, scenes, oracle_scene_results):
    exe = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
    if not os.path.exists(exe):
        pytest.skip("dispest_demo not built")
    _, _, l, r = scenes["Cones"]
    H, W, _ = l.shape
    l.tofile(tmp_path / "l.f32"); r.tofile(tmp_path / "r.f32")
    ref = oracle_scene_results["Cones"]
    tail = [str(W), str(H), "64", str(tmp_path / "l.f32"), str(tmp_path / "r.f32"), str(tmp_path / "l.u8"),
            str(tmp_path / "r.u8"), "8", "0.0001", "0.9", "inf", "inf", "9", "25.5", "1", "exp"]
    g = {e["max_diff"]: e["sha"] for e in GOLD["scenes"]["Cones"]["l"]}

    def got():
        return [np.fromfile(tmp_path / f, np.uint8).reshape(H, W) for f in ("l.u8", "r.u8")]
    out = subprocess.run([exe, "--disp-check", "2", "2"] + tail + ["1"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert SP.sha(got()[0]) == g[2]
    out = subprocess.run([exe, "--disp-check", "1", "1", "--speckle", "1", "100", "1"] + tail + ["2"],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    sel = (ref["ld"], ref["rd"], DC.winner_costs(ref["lf"], ref["ld"]), DC.winner_costs(ref["rf"], ref["rd"]))
    exp = want(l, r, sel, 64, (FIRST, 1), (1, 100, 1), 2)
    assert_same(got()[0], exp[0], "demo first + speckle + fill left"); assert_same(got()[1], exp[1], "demo right")
    bad = subprocess.run([exe, "--disp-check", "1", "-3"] + tail, capture_output=True, text=True, timeout=300)
    assert bad.returncode == 1 and "disparity check" in bad.stderr
