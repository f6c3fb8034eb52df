"""GPU: speckle removal (psm_set_speckle_filter) bit for bit through the C-ABI against the CPU restatement
tests/speckle_oracle.py (pinned to cv2.filterSpeckles by golden_speckle.json): blobs at and across tile seams, long
union chains, adversarial maps, both map formats, every mode with every left-right check mode and post-filter
setting, every kind of context, the selection's outputs left untouched, launch counts, argument checks, TorchStereo and
the C++ demo.

Maps are injected as tests/test_gpu_lr.py does: after CostConst / CostFilter, one-hot cost slices (0 at the wanted
disparity, 1 elsewhere; +inf everywhere for a wanted 0) are written with psm_write_cost_slice."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from primestereomatch_b200 import DispEst, capi, synth
import lr_oracle as LR
import pp_chain as PP
import speckle_oracle as SP

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN, "golden_speckle.json")) as f:
    GOLD = json.load(f)
CASES = np.load(os.path.join(GOLDEN, "speckle_cases.npz"))
DEFAULT = (9, 25.5, 1, "exp")
OFF, FIRST, ONLY = capi.PSM_SPECKLE_OFF, capi.PSM_SPECKLE_FIRST, capi.PSM_SPECKLE_ONLY


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def assert_same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, f"{what}: shape {a.shape} vs {b.shape}"
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {a.size} differ, first at {list(i)}: {a[i]!r} vs {b[i]!r}")


def images(W, H, seed):
    rng = np.random.default_rng(seed)
    l8 = (rng.integers(0, 4, (H, W, 3)) * 85).astype(np.uint8)
    return synth.to_f32(l8), synth.to_f32(np.roll(l8, -1, axis=1).copy())


def inject_maps(de, ld, rd=None):
    assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
    for d in range(de.maxDis):
        de.write_cost_slice(0, d, np.where(ld == 0, np.inf, ld != d).astype(np.float32))
        if rd is not None:
            de.write_cost_slice(1, d, np.where(rd == 0, np.inf, rd != d).astype(np.float32))
    assert de.DispSelect_GPU() == 0
    assert_same(de.lDisMap, ld, "injected left")
    if rd is not None:
        assert_same(de.rDisMap, rd, "injected right")


def context_for(ld, D=None):
    H, W = ld.shape
    D = D or int(ld.max()) + 1
    bits = 16 if ld.dtype == np.uint16 else 8
    return DispEst(*images(W, H, seed=W + H), max(D, 2), map_bits=bits)


def speckle(de, mode, size, diff):
    """post-process with speckle mode `mode` -> (left, right) copies"""
    assert de.setSpeckleFilter(mode, size, diff) == 0
    assert de.PostProcess_GPU() == 0
    return de.lDisMap.copy(), None if de.rDisMap is None else de.rDisMap.copy()


def check_only(de, ld, rd, size, diff, what):
    gl, gr = speckle(de, ONLY, size, diff)
    assert_same(gl, SP.filter_speckles(ld, size, diff), f"{what} left ({size}, {diff})")
    if rd is not None:
        assert_same(gr, SP.filter_speckles(rd, size, diff), f"{what} right ({size}, {diff})")
    return gl, gr


def blobby(H, W, D, seed, dtype=np.uint8):
    """piecewise-constant regions with +-1 noise, islands and zeros: blobs of every size"""
    rng = np.random.default_rng(seed)
    cell = 5
    coarse = rng.integers(1, D, ((H + cell - 1) // cell, (W + cell - 1) // cell))
    m = np.kron(coarse, np.ones((cell, cell), np.int64))[:H, :W]
    m = m + rng.integers(-1, 2, (H, W)) * (rng.random((H, W)) < 0.2)
    m = np.where(rng.random((H, W)) < 0.05, rng.integers(1, D, (H, W)), m)
    m = np.where(rng.random((H, W)) < 0.05, 0, m)
    return np.clip(m, 0, D - 1).astype(dtype)


def device_maps(de, which):
    """psm_copy_maps_device(which) into CUDA tensors -> host (left, right or None)"""
    import torch
    dt = torch.uint16 if de.map_bits == 16 else torch.uint8
    both = de.rDisMap is not None
    lt = torch.empty((de.hei, de.wid), dtype=dt, device="cuda")
    rt = torch.empty_like(lt) if both else None
    row = de.wid * lt.element_size()
    capi.check(capi.lib().psm_copy_maps_device(de.handle, which, lt.data_ptr(), row,
                                               rt.data_ptr() if both else None, row), de.handle)
    de.sync()
    return lt.cpu().numpy(), (rt.cpu().numpy() if both else None)


# ---- cv2's own results --------------------------------------------------------------------------------------------------
def test_synthetic_golden_cases():
    """u8 and u16 (differences above 255) maps, W or H = 1, max_diff 0 to 100000: sha256 of cv2.filterSpeckles"""
    for ent in GOLD["synthetic"]:
        m = CASES[ent["key"]]
        D = 4096 if m.dtype == np.uint16 else 256
        with context_for(m, D) as de:
            inject_maps(de, m, m[::-1].copy())
            for s in ent["settings"]:
                gl, gr = speckle(de, ONLY, s["max_size"], s["max_diff"])
                assert SP.sha(gl) == s["sha"], (ent["key"], s)
                assert_same(gr, SP.filter_speckles(m[::-1], s["max_size"], s["max_diff"]), f"{ent['key']} right {s}")


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_full_scenes_against_the_golden(scene, scenes, oracle_scene_results):
    _, _, l, r = scenes[scene]
    ref = oracle_scene_results[scene]
    g = GOLD["scenes"][scene]
    with DispEst(l, r, 64) as de:
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        assert_same(de.lDisMap, ref["ld"], "WTA left")
        for sl, sr in zip(g["l"], g["r"]):
            gl, gr = speckle(de, ONLY, sl["max_size"], sl["max_diff"])
            assert [SP.sha(gl), SP.sha(gr)] == [sl["sha"], sr["sha"]], (scene, sl["max_size"], sl["max_diff"])
        for lr in (1, 2, 0):
            de.setLRCheck(lr)
            gl, gr = speckle(de, FIRST, 400, 2)
            want = PP.chain(l, r, ref["ld"], ref["rd"], speckle=(FIRST, 400, 2), lr=lr)
            assert_same(gl, want[0], f"{scene} first + lr {lr} left"); assert_same(gr, want[1], f"{scene} first + lr {lr} right")


# ---- blob sizes at tile seams, long chains, adversarial maps ----------------------------------------------------------
@pytest.mark.parametrize("size", [1, 5, 40])
def test_blob_of_max_size_and_one_more_across_seams(size):
    """blobs of exactly `size` and `size + 1` pixels on one tile, across the vertical seam at x = 32 (both ways), the
    horizontal seam at y = 32 (both ways) and the corner at (32, 32), in a 100 x 90 map (not a multiple of the tile)"""
    H, W = 90, 100
    spots = [(5, 5, "h"), (40, 24, "h"), (60, 50, "h-"), (3, 31, "v"), (30, 60, "v"), (70, 80, "v-"), (31, 31, "c")]
    with DispEst(*images(W, H, seed=size), 64) as de:
        for y0, x0, how in spots:
            for n in (size, size + 1):
                m = np.full((H, W), 50, np.uint8)
                if how == "c":   # a staircase through the corner
                    pix = [(y0 + i // 2, x0 + (i + 1) // 2) for i in range(n)]
                else:
                    step = (0, 1) if how[0] == "h" else (1, 0)
                    sign = -1 if how.endswith("-") else 1
                    pix = [(y0 + sign * i * step[0], x0 + sign * i * step[1]) for i in range(n)]
                for y, x in pix:
                    m[y, x] = 7
                assert np.count_nonzero(m == 7) == n
                rd = m[::-1].copy()
                inject_maps(de, m, rd)
                gl, gr = check_only(de, m, rd, size, 1, f"blob of {n} ({how} at {y0}, {x0})")
                assert np.count_nonzero(gl == 0) == (n if n <= size else 0), (n, size, how)
                assert np.count_nonzero(gr == 0) == np.count_nonzero(gl == 0)


def test_squares_across_tile_corners():
    """k x k squares centred on tile corners: each corner pixel is reached across both seams at once"""
    H, W = 130, 100
    with DispEst(*images(W, H, seed=6), 16) as de:
        for k in (2, 3, 4):
            m = np.full((H, W), 9, np.uint8)
            for cy in (32, 64, 96):
                for cx in (32, 64, 96):
                    m[cy - k // 2:cy - k // 2 + k, cx - k // 2:cx - k // 2 + k] = 3
            inject_maps(de, m, m[:, ::-1].copy())
            for size in (k * k - 1, k * k):
                gl, gr = check_only(de, m, m[:, ::-1].copy(), size, 1, f"{k} x {k} squares")
                assert np.count_nonzero(gl == 0) == (9 * k * k if size == k * k else 0), (k, size)


def test_serpentine_blob_across_1080p():
    """one blob winding across every row of a 1920 x 1080 map: unions chain through every tile"""
    H, W = 1080, 1920
    m = np.full((H, W), 3, np.uint8)
    m[0::2, :] = 1
    m[1::4, -1] = 1
    m[3::4, 0] = 1
    snake = int(np.count_nonzero(m == 1))
    stripe = W - 1                                                      # each odd row: one blob of value 3
    with DispEst(*images(W, H, seed=1), 4) as de:
        inject_maps(de, m, m[:, ::-1].copy())
        for size in (stripe - 1, snake - 1, snake):
            gl, gr = check_only(de, m, m[:, ::-1].copy(), size, 1, f"serpentine max_size {size}")
            assert np.count_nonzero(gl == 0) == (snake if size >= snake else 0) + \
                (stripe * (H // 2) if size >= stripe else 0), size
            assert de.stage_ms(5) > 0


@pytest.mark.parametrize("H,W", [(1080, 1920), (97, 61), (1, 300), (300, 1), (1, 1)])
def test_constant_checkerboard_and_zero_maps(H, W):
    const = np.full((H, W), 2, np.uint8)
    chk = (1 + (np.indices((H, W)).sum(0) % 2)).astype(np.uint8)
    zero = np.zeros((H, W), np.uint8)
    with DispEst(*images(W, H, seed=2), 3) as de:
        inject_maps(de, const, chk)
        for size in sorted({1, max(1, H * W - 1), H * W}):
            gl, gr = check_only(de, const, chk, size, 0, f"constant / checkerboard {H}x{W}")
            assert (gl == 0).all() == (size >= H * W)
            assert (gr == 0).all()                                      # every checkerboard pixel is its own blob
        gl, gr = check_only(de, const, chk, 1, 1, "checkerboard joined at max_diff 1")
        assert (gr == 0).all() == (H * W == 1)
        inject_maps(de, zero, zero)
        gl, gr = check_only(de, zero, zero, 10, 3, "all-zero")
        assert not gl.any() and not gr.any()


def test_u16_differences_above_255():
    H, W, D = 24, 40, 1400
    m = np.full((H, W), 1000, np.uint16)
    m[5:8, 5:9] = 1300                                                  # 12 pixels, 300 away
    m[15:17, 20:30] = 1299                                              # 20 pixels, 299 away
    m[20, 35] = 1                                                       # a single pixel, 999 away
    with context_for(m, D) as de:
        inject_maps(de, m, m[::-1].copy())
        for diff in (0, 1, 298, 299, 300, 998, 999, 255, 4096):
            for size in (1, 12, 20, 900):
                check_only(de, m, m[::-1].copy(), size, diff, f"u16 diff {diff}")


# ---- the chain: every mode with every check mode and post-filter setting ------------------------------------------------
@pytest.mark.parametrize("bits", [8, 16])
def test_every_mode_with_every_check_mode(bits):
    H, W, D = 61, 83, 32 if bits == 8 else 300
    dt = np.uint16 if bits == 16 else np.uint8
    ld, rd = blobby(H, W, D, seed=3, dtype=dt), blobby(H, W, D, seed=4, dtype=dt)
    l, r = images(W, H, seed=5)
    with DispEst(l, r, D, map_bits=bits) as de:
        inject_maps(de, ld, rd)
        for setting in (DEFAULT, (3, 25.5, 2, "iv1")):
            de.setPostFilter(*setting)
            for sp in ((OFF, 0, 0), (FIRST, 6, 1), (ONLY, 6, 1), (FIRST, 30, 0)):
                for lr in (0, 1, 2):
                    de.setLRCheck(lr)
                    gl, gr = speckle(de, *sp)
                    want = PP.chain(l, r, ld, rd, speckle=sp, lr=lr, setting=setting)
                    what = f"u{bits} speckle {sp} lr {lr} {setting}"
                    assert_same(gl, want[0], what + " left"); assert_same(gr, want[1], what + " right")
                    if lr and sp[0] != ONLY:
                        src = (SP.filter_speckles(ld, *sp[1:]), SP.filter_speckles(rd, *sp[1:])) if sp[0] else (ld, rd)
                        lv, rv = LR.lr_check(*src)
                        assert_same(de.lValid, lv, what + " left mask"); assert_same(de.rValid, rv, what + " right mask")
                        if sp[0]:
                            assert not lv[(src[0] == 0) & (ld != 0)].any(), "a removed pixel passed the check"


# ---- every kind of context; the selection's outputs stay as they were --------------------------------------------------
KINDS = [("unblocked", {}), ("blocked", {"block_slices": 16}), ("multi", {"devices": [0, 0]}),
         ("multi-blocked", {"devices": [0, 0, 0], "block_slices": 8}), ("range", {"min_disp": 17}),
         ("left-only", {}), ("u16", {"map_bits": 16}), ("u16 range multi", {"map_bits": 16, "min_disp": 5, "devices": [0, 0]})]


@pytest.mark.parametrize("kind,kw", KINDS, ids=[k for k, _ in KINDS])
def test_context_kinds(kind, kw):
    W, H, D = 200, 120, 64
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=8)
    rng = np.random.default_rng(8)
    r8 = np.clip(r8.astype(np.int16) + rng.integers(-40, 41, r8.shape), 0, 255).astype(np.uint8)   # speckled maps
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    L = capi.lib()
    with DispEst(l, r, D, **kw) as de:
        left_only = kind == "left-only"
        if left_only:
            de.setViews("left")
        de.setCostOutput(True); de.setRunnerUpOutput(True)
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        ld, rd = de.lDisMap.copy(), None if left_only else de.rDisMap.copy()
        costs, runner = (de.lCosts, de.rCosts), (de.lRunnerUp, de.rRunnerUp)
        assert (SP.filter_speckles(ld, 20, 1) != ld).any(), "the maps have no speckles to remove"
        for size, diff in ((20, 1), (200, 0)):
            check_only(de, ld, rd, size, diff, kind)
        de.setLRCheck(0 if left_only else 1)
        gl, gr = speckle(de, FIRST, 20, 1)
        want = PP.chain(l, r, ld, rd, speckle=(FIRST, 20, 1), lr=0 if left_only else 1)
        assert_same(gl, want[0], f"{kind} first left")
        if not left_only:
            assert_same(gr, want[1], f"{kind} first right")
        assert_same(device_maps(de, 1)[0], gl, f"{kind} post-processed maps on the device")
        # the selection's maps, costs and runner-up are the selection's
        sl, sr = device_maps(de, 0)
        assert_same(sl, ld, f"{kind} selection map left after the stage")
        if not left_only:
            assert_same(sr, rd, f"{kind} selection map right after the stage")
        for got, was in ((de._read_output(L.psm_read_costs, 3), costs), (de._read_output(L.psm_read_runner_up, 2), runner)):
            for v in (0,) if left_only else (0, 1):
                assert got[v].tobytes() == was[v].tobytes(), f"{kind} costs / runner-up of view {v} changed"
        if left_only:
            de.setLRCheck(1)
            with pytest.raises(capi.PsmError) as e:
                speckle(de, FIRST, 20, 1)
            assert e.value.code == capi.PSM_ESTATE
            check_only(de, ld, None, 20, 1, "left-only, only, with a check mode set")


# ---- launches, masks and arguments --------------------------------------------------------------------------------------
def test_launch_counts_and_stage_time():
    ld, rd = blobby(48, 64, 16, seed=11), blobby(48, 64, 16, seed=12)
    with DispEst(*images(64, 48, seed=11), 16) as de:
        inject_maps(de, ld, rd)
        for sp in (OFF, FIRST, ONLY):
            for lr in (0, 1, 2):
                for it in (1, 3):
                    de.setLRCheck(lr); de.setPostFilter(9, 25.5, it, "exp"); de.setSpeckleFilter(sp, 5, 1)
                    n = de.launch_count()
                    assert de.PostProcess_GPU() == 0
                    base = {0: 4 * it, 1: 1 + 4 * it, 2: 1}[lr]
                    want = {OFF: base, FIRST: 4 + base, ONLY: 4}[sp]
                    assert de.launch_count() - n == want, (sp, lr, it)
                    assert de.stage_ms(5) > 0


def test_masks_and_invalid_arguments():
    ld, rd = blobby(30, 40, 16, seed=2), blobby(30, 40, 16, seed=3)
    L = capi.lib()
    mask = np.zeros((30, 40), np.uint8)
    with DispEst(*images(40, 30, seed=2), 16) as de:
        h = de.handle
        inject_maps(de, ld, rd)
        de.setLRCheck(2)
        want = speckle(de, FIRST, 6, 1)
        for mode, size, diff in ((-1, 6, 1), (3, 6, 1), (FIRST, 0, 1), (ONLY, -2, 1), (FIRST, 6, -1), (ONLY, 0, -1)):
            assert L.psm_set_speckle_filter(h, mode, size, diff) == capi.PSM_EINVAL and L.psm_last_error(h), (mode, size, diff)
            assert de.PostProcess_GPU() == 0
            assert_same(de.lDisMap, want[0], f"left after rejected ({mode}, {size}, {diff})")
        assert L.psm_set_speckle_filter(None, FIRST, 6, 1) == capi.PSM_EINVAL
        with pytest.raises(capi.PsmError):
            de.setSpeckleFilter(FIRST, 0, 0)
        assert L.psm_set_speckle_filter(h, OFF, 0, -5) == 0                    # sizes are not read while off
        assert_same(speckle(de, OFF, 0, -5)[0], LR.lr_check_fill(ld, rd)[2], "off")
        # the check ran after the removal: removed pixels are invalid
        de.setSpeckleFilter(FIRST, 6, 1); de.PostProcess_GPU()
        sl = SP.filter_speckles(ld, 6, 1)
        assert_same(de.lValid, LR.lr_check(sl, SP.filter_speckles(rd, 6, 1))[0], "mask after the removal")
        # only: no check, no masks (the facade does not read them)
        de.setSpeckleFilter(ONLY, 6, 1)
        assert de.PostProcess_GPU() == 0
        assert L.psm_read_valid_mask(h, 0, ptr(mask), 40) == capi.PSM_ESTATE
    with DispEst(*images(40, 30, seed=2), 16, devices=[0, 0]) as de:     # forwarded to every shard, or to none
        assert L.psm_set_speckle_filter(de.handle, ONLY, 0, 1) == capi.PSM_EINVAL
        de.setSpeckleFilter(ONLY, 6, 1)


def test_torch_stereo_and_held_back_stream():
    import torch
    from primestereomatch_b200.torch_stereo import TorchStereo
    W, H, D = 160, 96, 48
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=13)
    rng = np.random.default_rng(13)
    r8 = np.clip(r8.astype(np.int16) + rng.integers(-40, 41, r8.shape), 0, 255).astype(np.uint8)
    lt, rt = torch.from_numpy(l8).cuda(), torch.from_numpy(r8).cuda()
    with TorchStereo(W, H, D) as ts:
        lm, rm = ts.match(lt, rt)
        ld, rd = lm.cpu().numpy(), rm.cpu().numpy()
        ts.setSpeckleFilter(ONLY, 15, 1)
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)                                   # the frames' stream is held back
            lm, rm = ts.match(lt, rt, post_process=True)
        torch.cuda.synchronize()
        assert_same(lm.cpu().numpy(), SP.filter_speckles(ld, 15, 1), "TorchStereo only left")
        assert_same(rm.cpu().numpy(), SP.filter_speckles(rd, 15, 1), "TorchStereo only right")
        ts.setSpeckleFilter(FIRST, 15, 1); ts.setLRCheck(2)
        lm, rm = ts.match(lt, rt, post_process=True)
        want = LR.lr_check_fill(SP.filter_speckles(ld, 15, 1), SP.filter_speckles(rd, 15, 1))
        assert_same(lm.cpu().numpy(), want[2], "TorchStereo first + fill left")
        with pytest.raises(capi.PsmError):
            ts.setSpeckleFilter(7, 1, 1)


def test_cpp_demo_speckle_flag(tmp_path, scenes, oracle_scene_results):
    exe = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
    if not os.path.exists(exe):
        pytest.skip("dispest_demo not built")
    _, _, l, r = scenes["Cones"]
    H, W, _ = l.shape
    l.tofile(tmp_path / "l.f32"); r.tofile(tmp_path / "r.f32")
    ref = oracle_scene_results["Cones"]
    tail = [str(W), str(H), "64", str(tmp_path / "l.f32"), str(tmp_path / "r.f32"), str(tmp_path / "l.u8"),
            str(tmp_path / "r.u8"), "8", "0.0001", "0.9", "inf", "inf", "9", "25.5", "1", "exp"]
    g = {(e["max_size"], e["max_diff"]): e["sha"] for e in GOLD["scenes"]["Cones"]["l"]}

    def got():
        return [np.fromfile(tmp_path / f, np.uint8).reshape(H, W) for f in ("l.u8", "r.u8")]
    out = subprocess.run([exe, "--speckle", "2", "400", "2"] + tail + ["1"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert SP.sha(got()[0]) == g[(400, 2)]
    out = subprocess.run([exe, "--speckle", "1", "100", "1"] + tail + ["2"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    want = PP.chain(l, r, ref["ld"], ref["rd"], speckle=(FIRST, 100, 1), lr=2)
    assert_same(got()[0], want[0], "demo first + fill left"); assert_same(got()[1], want[1], "demo first + fill right")
    bad = subprocess.run([exe, "--speckle", "1", "0", "1"] + tail, capture_output=True, text=True, timeout=300)
    assert bad.returncode == 1 and "speckle filter" in bad.stderr
