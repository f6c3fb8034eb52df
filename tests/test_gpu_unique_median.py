"""GPU: the uniqueness test (psm_set_uniqueness_check) and the median (psm_set_median_blur) bit for bit through the C-ABI
against sgbm_chain.chain, whose steps are the CPU restatements tests/unique_oracle.py and tests/median_oracle.py (pinned
by golden_median.json), applied to each context's own selection maps, psm_read_costs plane 1 and psm_read_runner_up
plane 1: every mode of both steps alone and with every existing step, every kind of context, the left-only fill and
its mask, the selection's outputs left untouched, launch counts, argument and state checks, reprojection of the new
maps, TorchStereo on a held-back stream, the C++ demo, and a small pairwise sweep over config_sweep's kinds, formats
and post-process levels."""
import itertools
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from primestereomatch_b200 import DispEst, capi, synth
import config_sweep as CS
import median_oracle as MD
import sgbm_chain as SC
import reproject_oracle as RP
import unique_oracle as UN

pytestmark = pytest.mark.gpu

U_OFF, U_FIRST, U_ONLY = capi.PSM_UNIQUE_OFF, capi.PSM_UNIQUE_FIRST, capi.PSM_UNIQUE_ONLY
M_OFF, M_FIRST, M_ONLY = capi.PSM_MEDIAN_OFF, capi.PSM_MEDIAN_FIRST, capi.PSM_MEDIAN_ONLY
DEFAULT = (9, 25.5, 1, "exp")
GENERIC = (3, 25.5, 2, "iv1")
UNIQUES = ((U_OFF, 10), (U_FIRST, 10), (U_ONLY, 15), (U_FIRST, 0), (U_FIRST, 100))
MEDIANS = ((M_OFF, 3), (M_FIRST, 3), (M_ONLY, 5), (M_FIRST, 5))
# the reference's StereoSGBM post-processing: uniquenessRatio 10, disp12MaxDiff 1, medianBlur 3, speckle (100, 32)
SGBM = dict(uniqueness=(U_FIRST, 10), dcheck=(1, 1), median=(M_FIRST, 3), speckle=(1, 100, 32))


def assert_same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, f"{what}: shape {a.shape} vs {b.shape}"
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {a.size} differ, first at {list(i)}: {a[i]!r} vs {b[i]!r}")


def noisy_pair(W, H, D, seed):
    """a synthetic pair with noise on the right view, so the maps hold ambiguous pixels for the test to find"""
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=seed)
    rng = np.random.default_rng(seed)
    r8 = np.clip(r8.astype(np.int16) + rng.integers(-40, 41, r8.shape), 0, 255).astype(np.uint8)
    return synth.to_f32(l8), synth.to_f32(r8)


def select(de):
    """one frame with the costs and the runner-up on -> dict of the selection maps, q(m) and q(r) per view"""
    de.setCostOutput(True); de.setRunnerUpOutput(True)
    assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0 and de.DispSelect_GPU() == 0
    two = de.rDisMap is not None
    return {"maps": (de.lDisMap.copy(), de.rDisMap.copy() if two else None),
            "qm": (de.lCosts[1].copy(), de.rCosts[1].copy() if two else None),
            "qr": (de.lRunnerUp[1].copy(), de.rRunnerUp[1].copy() if two else None),
            "costs": (de.lCosts.copy(), de.rCosts.copy() if two else None),
            "runner": (de.lRunnerUp.copy(), de.rRunnerUp.copy() if two else None)}


def configure(de, uniqueness=(U_OFF, 10), dcheck=(0, 1), median=(M_OFF, 3), speckle=(0, 0, 0), lr=0, setting=DEFAULT):
    de.setUniquenessCheck(*uniqueness); de.setDisparityCheck(*dcheck); de.setMedianBlur(*median)
    de.setSpeckleFilter(*speckle); de.setLRCheck(lr); de.setPostFilter(*setting)


def post(de, **kw):
    configure(de, **kw)
    assert de.PostProcess_GPU() == 0
    return de.lDisMap.copy(), None if de.rDisMap is None else de.rDisMap.copy()


def want(l, r, sel, D, **kw):
    ld, rd = sel["maps"]
    return SC.chain(l, r, ld, rd, costs=sel["qm"], runner=sel["qr"], D=D, **kw)


def check_against(de, l, r, sel, D, what, **kw):
    got = post(de, **kw)
    ref = want(l, r, sel, D, **kw)
    assert_same(got[0], ref[0], what + " left")
    if sel["maps"][1] is not None:
        assert_same(got[1], ref[1], what + " right")
    return got, ref


def ended(kw):
    return any(kw.get(k, (0,))[0] == 2 for k in ("uniqueness", "dcheck", "median", "speckle"))


# ---- every mode alone and with every existing step ----------------------------------------------------------------------
@pytest.mark.parametrize("bits", [8, 16])
def test_every_mode_with_every_existing_step(bits):
    W, H, D = (140, 48, 48) if bits == 8 else (400, 32, 300)
    l, r = noisy_pair(W, H, 48, seed=3)
    with DispEst(l, r, D, map_bits=bits) as de:
        sel = select(de)
        ld = sel["maps"][0]
        assert (UN.check(ld, sel["qm"][0], sel["qr"][0], 10) != ld).any(), "nothing for the uniqueness test to reject"
        assert (MD.median(ld, 3) != ld).any(), "nothing for the median to change"
        for un, md in itertools.product(UNIQUES, MEDIANS):
            for dc, sp, lr, setting in ((((0, 1), (0, 0, 0), 0, DEFAULT)), ((1, 1), (0, 0, 0), 0, DEFAULT),
                                        ((2, 1), (0, 0, 0), 0, DEFAULT), ((0, 1), (1, 6, 1), 0, DEFAULT),
                                        ((0, 1), (2, 6, 1), 0, DEFAULT), ((0, 1), (0, 0, 0), 1, DEFAULT),
                                        ((1, 1), (1, 6, 1), 2, DEFAULT), ((0, 1), (0, 0, 0), 1, GENERIC)):
                kw = dict(uniqueness=un, median=md, dcheck=dc, speckle=sp, lr=lr, setting=setting)
                what = f"u{bits} {kw}"
                _, ref = check_against(de, l, r, sel, D, what, **kw)
                if lr and not ended(kw):
                    assert_same(de.lValid, ref[2][0], what + " left mask")
                    assert_same(de.rValid, ref[2][1], what + " right mask")


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_scenes_with_the_reference_sgbm_setting(scene, scenes):
    _, _, l, r = scenes[scene]
    with DispEst(l, r, 64) as de:
        sel = select(de)
        for lr in (0, 2, 1):
            for sp_only in (False, True):
                kw = dict(SGBM, lr=lr)
                if sp_only:
                    kw["speckle"] = (2, 100, 32)
                check_against(de, l, r, sel, 64, f"{scene} SGBM lr {lr} speckle only {sp_only}", **kw)
        for k in MD.KSIZES:
            check_against(de, l, r, sel, 64, f"{scene} median only {k}", median=(M_ONLY, k))


# ---- every kind of context; the selection's outputs stay as they were ------------------------------------------------------
KINDS = [("unblocked", {}, 8, 64), ("blocked B=7", {"block_slices": 7}, 8, 64), ("blocked B=1", {"block_slices": 1}, 8, 64),
         ("multi-2", {"devices": [0, 0]}, 8, 64), ("range", {"min_disp": 9}, 8, 64), ("left-only", {}, 8, 64),
         ("u16 D=300", {}, 16, 300), ("u16 range multi-2", {"min_disp": 9, "devices": [0, 0]}, 16, 300)]


@pytest.mark.parametrize("kind,kw,bits,D", KINDS, ids=[k[0] for k in KINDS])
def test_context_kinds(kind, kw, bits, D):
    W, H = 380, 40
    l, r = noisy_pair(W, H, 64, seed=8)
    L = capi.lib()
    left_only = kind == "left-only"
    with DispEst(l, r, D, map_bits=bits, **kw) as de:
        if left_only:
            de.setViews("left")
        sel = select(de)
        for un, md in itertools.product(UNIQUES[1:3], MEDIANS[1:3]):
            for extra in ({}, {"dcheck": (1, 1), "speckle": (1, 20, 1), "lr": 1}, {"lr": 2}, {**SGBM, "lr": 2}):
                args = {"uniqueness": un, "median": md, **extra}
                got, ref = check_against(de, l, r, sel, D, f"{kind} {args}", **args)
                if args.get("lr") and not ended(args):
                    assert_same(de.lValid, ref[2][0], f"{kind} {args} left mask")
        # the selection's maps, costs and runner-up are the selection's
        views = (0,) if left_only else (0, 1)
        for got, was in ((de._read_output(L.psm_read_costs, 3), sel["costs"]),
                         (de._read_output(L.psm_read_runner_up, 2), sel["runner"])):
            for v in views:
                assert got[v].tobytes() == was[v].tobytes(), f"{kind} costs / runner-up of view {v} changed"
        # the selection maps too: their points are those of the maps the selection returned
        for v in views:
            RP.assert_points_equal(de.reproject(CS.Q, ("left", "right")[v], "selection"), RP.reproject(sel["maps"][v], CS.Q),
                                   f"{kind} selection map {v}")
        assert de.stage_ms(5) > 0


# ---- the left-only fill -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [8, 16])
def test_left_only_fill_and_mask(bits):
    W, H, D = 180, 50, 40
    l, r = noisy_pair(W, H, D, seed=17)
    L = capi.lib()
    mask = np.zeros((H, W), np.uint8)
    with DispEst(l, r, D, map_bits=bits) as de:
        de.setViews("left")
        sel = select(de)
        for lr in (1, 2):
            for md in ((M_OFF, 3), (M_FIRST, 3), (M_FIRST, 5)):
                for sp in ((0, 0, 0), (1, 10, 1)):
                    kw = dict(uniqueness=(U_FIRST, 10), median=md, speckle=sp, lr=lr)
                    _, ref = check_against(de, l, r, sel, D, f"left-only {kw}", **kw)
                    assert_same(de.lValid, ref[2][0], f"left-only mask {kw}")
        assert L.psm_read_valid_mask(de.handle, capi.PSM_RIGHT, mask.ctypes.data, W) == capi.PSM_ESTATE
        # ONLY runs no fill: no mask; the median alone does not make a left-only context fill
        post(de, uniqueness=(U_ONLY, 10), lr=1)
        assert L.psm_read_valid_mask(de.handle, capi.PSM_LEFT, mask.ctypes.data, W) == capi.PSM_ESTATE
        configure(de, median=(M_FIRST, 3), lr=1)
        with pytest.raises(capi.PsmError) as e:
            de.PostProcess_GPU()
        assert e.value.code == capi.PSM_ESTATE


# ---- launches, arguments and state -------------------------------------------------------------------------------------------
def test_launch_counts():
    l, r = noisy_pair(64, 48, 16, seed=11)
    with DispEst(l, r, 16) as de:
        select(de)
        for un, md, dc, sp, lr in itertools.product((0, 1, 2), (0, 1, 2), (0, 1, 2), (0, 1, 2), (0, 1, 2)):
            configure(de, uniqueness=(un, 10), median=(md, 3), dcheck=(dc, 1), speckle=(sp, 5, 1), lr=lr)
            n = de.launch_count()
            assert de.PostProcess_GPU() == 0
            steps = [(un, 1), (dc, 1), (md, 1), (sp, 4)]
            count = 0
            for mode, k in steps:
                if mode:
                    count += k
                if mode == 2:
                    break
            else:
                count += {0: 4, 1: 1 + 4, 2: 1}[lr]
            assert de.launch_count() - n == count, (un, md, dc, sp, lr)


def test_invalid_arguments_and_states():
    W, H, D = 90, 40, 16
    l, r = noisy_pair(W, H, D, seed=2)
    L = capi.lib()
    with DispEst(l, r, D) as de:
        h = de.handle
        sel = select(de)
        good = post(de, uniqueness=(U_FIRST, 10), median=(M_FIRST, 5), lr=2)
        for mode, ratio in ((-1, 10), (3, 10), (U_FIRST, -1), (U_ONLY, 101), (U_OFF, -1), (U_OFF, 101)):
            assert L.psm_set_uniqueness_check(h, mode, ratio) == capi.PSM_EINVAL and L.psm_last_error(h), (mode, ratio)
            assert de.PostProcess_GPU() == 0
            assert_same(de.lDisMap, good[0], f"left after rejected uniqueness ({mode}, {ratio})")
        for mode, k in ((-1, 3), (3, 3), (M_FIRST, 4), (M_ONLY, 7), (M_OFF, 1), (M_FIRST, 0)):
            assert L.psm_set_median_blur(h, mode, k) == capi.PSM_EINVAL and L.psm_last_error(h), (mode, k)
            assert de.PostProcess_GPU() == 0
            assert_same(de.lDisMap, good[0], f"left after rejected median ({mode}, {k})")
        assert L.psm_set_uniqueness_check(None, U_FIRST, 10) == capi.PSM_EINVAL
        assert L.psm_set_median_blur(None, M_FIRST, 3) == capi.PSM_EINVAL
        # ratio 0 rejects nothing
        assert_same(post(de, uniqueness=(U_ONLY, 0))[0], sel["maps"][0], "ratio 0")
        # both planes are required: a selection without either refuses the stage and names the options
        for costs, runner in ((False, True), (True, False), (False, False)):
            de.setCostOutput(costs); de.setRunnerUpOutput(runner)
            de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
            configure(de, uniqueness=(U_FIRST, 10), lr=2)
            with pytest.raises(capi.PsmError) as e:
                de.PostProcess_GPU()
            assert e.value.code == capi.PSM_ESTATE and b"PSM_OPT_RUNNER_UP" in L.psm_last_error(h)
            # the median needs neither
            got = post(de, median=(M_ONLY, 3))
            assert_same(got[0], MD.median(sel["maps"][0], 3), "median without costs")
    # a context owning part of the range takes the uniqueness test OFF alone, the median at any mode
    with DispEst(l, r, D, d_begin=0, d_count=8) as de:
        assert L.psm_set_uniqueness_check(de.handle, U_FIRST, 10) == capi.PSM_EINVAL
        assert L.psm_set_uniqueness_check(de.handle, U_OFF, 10) == 0
        assert L.psm_set_median_blur(de.handle, M_FIRST, 3) == 0
    with DispEst(l, r, D, devices=[0, 0]) as de:
        assert L.psm_set_uniqueness_check(de.handle, 5, 1) == capi.PSM_EINVAL
        assert L.psm_set_median_blur(de.handle, M_FIRST, 9) == capi.PSM_EINVAL
        sel = select(de)
        check_against(de, l, r, sel, D, "multi after rejected settings", uniqueness=(U_ONLY, 12))


def test_reproject_the_new_maps():
    W, H, D = 160, 48, 32
    l, r = noisy_pair(W, H, D, seed=5)
    with DispEst(l, r, D) as de:
        sel = select(de)
        for kw in ({"uniqueness": (U_ONLY, 10)}, {"median": (M_ONLY, 5)}, {**SGBM, "lr": 2}):
            got = post(de, **kw)
            for v, view in enumerate(("left", "right")):
                RP.assert_points_equal(de.reproject(CS.Q, view, "post", True), RP.reproject(got[v], CS.Q, True),
                                       f"{kw} {view}")


# ---- TorchStereo and the demo --------------------------------------------------------------------------------------------------
def test_torch_stereo_on_a_held_back_stream():
    import torch
    from primestereomatch_b200.torch_stereo import TorchStereo
    W, H, D = 160, 96, 48
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=13)
    rng = np.random.default_rng(13)
    r8 = np.clip(r8.astype(np.int16) + rng.integers(-40, 41, r8.shape), 0, 255).astype(np.uint8)
    lt, rt = torch.from_numpy(l8).cuda(), torch.from_numpy(r8).cuda()
    with TorchStereo(W, H, D) as ts:
        lm, rm, lc, rc, lr_, rr = ts.match(lt, rt, costs=True, runner_up=True)
        sel = [x.cpu().numpy() for x in (lm, rm, lc[1], rc[1], lr_[1], rr[1])]
        ts.match(lt, rt)                                                    # both off again
        assert ts.costs is False and ts.runner_up is False
        ts.setUniquenessCheck(U_ONLY, 10)
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)                                   # the frames' stream is held back
            out = ts.match(lt, rt, post_process=True)
        torch.cuda.synchronize()
        assert len(out) == 2 and ts.costs is True and ts.runner_up is True  # set for the test, not returned
        assert_same(out[0].cpu().numpy(), UN.check(sel[0], sel[2], sel[4], 10), "TorchStereo only left")
        assert_same(out[1].cpu().numpy(), UN.check(sel[1], sel[3], sel[5], 10), "TorchStereo only right")
        ts.setUniquenessCheck(U_FIRST, 15); ts.setMedianBlur(M_FIRST, 3); ts.setLRCheck(2)
        lm, rm, lru, _ = ts.match(lt, rt, post_process=True, runner_up=True)
        exp = SC.chain(None, None, sel[0], sel[1], uniqueness=(U_FIRST, 15), costs=(sel[2], sel[3]),
                       runner=(sel[4], sel[5]), median=(M_FIRST, 3), lr=2)
        assert_same(lm.cpu().numpy(), exp[0], "TorchStereo first + median + fill left")
        assert lru[1].cpu().numpy().tobytes() == sel[4].tobytes()
        with pytest.raises(capi.PsmError):
            ts.setUniquenessCheck(7, 10)
        with pytest.raises(capi.PsmError):
            ts.setMedianBlur(M_FIRST, 4)


def test_cpp_demo_flags(tmp_path, scenes):
    exe = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
    if not os.path.exists(exe):
        pytest.skip("dispest_demo not built")
    _, _, l, r = scenes["Cones"]
    H, W, _ = l.shape
    l.tofile(tmp_path / "l.f32"); r.tofile(tmp_path / "r.f32")
    with DispEst(l, r, 64) as de:
        sel = select(de)
    tail = [str(W), str(H), "64", str(tmp_path / "l.f32"), str(tmp_path / "r.f32"), str(tmp_path / "l.u8"),
            str(tmp_path / "r.u8"), "8", "0.0001", "0.9", "inf", "inf", "9", "25.5", "1", "exp"]

    def got():
        return [np.fromfile(tmp_path / f, np.uint8).reshape(H, W) for f in ("l.u8", "r.u8")]
    out = subprocess.run([exe, "--uniqueness", "2", "10"] + tail + ["1"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert_same(got()[0], want(l, r, sel, 64, uniqueness=(U_ONLY, 10))[0], "demo uniqueness only")
    out = subprocess.run([exe, "--uniqueness", "1", "10", "--disp-check", "1", "1", "--median", "1", "3", "--speckle",
                          "1", "100", "32"] + tail + ["2"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    exp = want(l, r, sel, 64, **SGBM, lr=2)
    assert_same(got()[0], exp[0], "demo SGBM set left"); assert_same(got()[1], exp[1], "demo SGBM set right")
    out = subprocess.run([exe, "--median", "2", "5"] + tail, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert_same(got()[0], MD.median(sel["maps"][0], 5), "demo median only")
    bad = subprocess.run([exe, "--median", "1", "4"] + tail, capture_output=True, text=True, timeout=300)
    assert bad.returncode == 1 and "median" in bad.stderr
    bad = subprocess.run([exe, "--uniqueness", "1", "101"] + tail, capture_output=True, text=True, timeout=300)
    assert bad.returncode == 1 and "uniqueness" in bad.stderr


# ---- a small pairwise sweep over config_sweep's kinds, formats and post-process levels ---------------------------------------
def sweep_cases():
    """every (kind, format) pair of config_sweep once, each running every POSTS level with the new levels rotated so that
    every pair of (uniqueness level, median level) and every pair of (new level, POSTS level) occurs"""
    news = list(itertools.product(UNIQUES, MEDIANS))
    posts = [p for p in CS.POSTS if CS.POSTS[p] is not None]
    cases = []
    for k, (kind, fmt) in enumerate(itertools.product(CS.KINDS, CS.FORMATS)):
        cases.append((kind, fmt, [(posts[(k + i) % len(posts)], news[(k * 7 + i) % len(news)]) for i in range(len(news))]))
    return cases


@pytest.mark.parametrize("kind,fmt,steps", sweep_cases(), ids=[f"{k}-{f}" for k, f, _ in sweep_cases()])
def test_pairwise_sweep(kind, fmt, steps):
    config = dict(CS.DEFAULT, kind=kind, format=fmt)
    W, H, D, bits = CS.geometry(config)
    l8, r8 = CS.frames(config, CS.SEED)["src"]
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    with DispEst(l, r, D, map_bits=bits, **CS.KINDS[kind]) as de:
        sel = select(de)
        for post_name, (un, md) in steps:
            dcheck, speckle, lr, setting = CS.POSTS[post_name]
            kw = dict(uniqueness=un, median=md, dcheck=dcheck, speckle=speckle, lr=lr, setting=setting)
            check_against(de, l, r, sel, D, f"{kind} {fmt} {post_name} {un} {md}", **kw)
