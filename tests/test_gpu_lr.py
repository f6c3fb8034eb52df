"""GPU: the left-right consistency check and occlusion fill (psm_set_lr_check), bit for bit through the C-ABI against the
CPU restatement tests/lr_oracle.py (pinned to the reference's own PP.cpp by golden_lr.json): masks, filled maps and the
post-filtered maps of modes 1 and 2, on both map formats, sharded contexts and the FGF branch.

Maps are injected through the C-ABI: after CostConst / CostFilter, one-hot cost slices (0 at the wanted disparity, 1
elsewhere; +inf everywhere for a wanted 0, which the winner-take-all returns when no cost is below +inf) are written
with psm_write_cost_slice."""
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
import lr_oracle as LR
import pp_chain as PP

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN, "golden_lr.json")) as f:
    GOLD = json.load(f)
CASES = np.load(os.path.join(GOLDEN, "lr_cases.npz"))
DEFAULT = (9, 25.5, 1, "exp")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def posterise(img8, masks=(0xE0, 0xE0, 0xC0)):
    return (img8 & np.array(masks, np.uint8)).astype(np.uint8)


def f32(img):
    return O.u8_to_f32(img) if img.dtype == np.uint8 else img


def assert_same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, f"{what}: shape {a.shape} vs {b.shape}"
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {a.size} differ, first at {list(i)}: {a[i]!r} vs {b[i]!r}")


def inject_maps(de, ld, rd):
    assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
    for d in range(de.maxDis):
        de.write_cost_slice(0, d, np.where(ld == 0, np.inf, ld != d).astype(np.float32))
        de.write_cost_slice(1, d, np.where(rd == 0, np.inf, rd != d).astype(np.float32))
    assert de.DispSelect_GPU() == 0
    assert_same(de.lDisMap, ld, "injected left"); assert_same(de.rDisMap, rd, "injected right")


def device_map(de, what, dtype):
    """psm_device_ptr selector `what` copied to the host (W x H of dtype)"""
    p, pitch = C.c_void_p(), C.c_size_t()
    capi.check(capi.lib().psm_device_ptr(de.handle, what, C.byref(p), C.byref(pitch)), de.handle)
    assert p.value and pitch.value == de.wid
    out = np.empty((de.hei, de.wid), dtype)
    de.sync()
    cudart = C.CDLL("libcudart.so.12")
    assert cudart.cudaMemcpy(ptr(out), p, C.c_size_t(out.nbytes), 2) == 0   # cudaMemcpyDeviceToHost
    return out


def run(de, mode, setting=None):
    """post-process in `mode` (None: keep the context's mode) -> (left, right) copies"""
    if mode is not None:
        assert de.setLRCheck(mode) == 0
    if setting is not None:
        assert de.setPostFilter(*setting) == 0
    assert de.PostProcess_GPU() == 0
    return de.lDisMap.copy(), de.rDisMap.copy()


def check_modes(de, l, r, ld, rd, what, settings=(DEFAULT,)):
    lv, rv, lf, rf = LR.lr_check_fill(ld, rd)
    gl, gr = run(de, 2)
    assert_same(gl, lf, f"{what} mode 2 left"); assert_same(gr, rf, f"{what} mode 2 right")
    assert_same(de.lValid, lv, f"{what} left mask"); assert_same(de.rValid, rv, f"{what} right mask")
    for s in settings:
        gl, gr = run(de, 1, s)
        assert_same(gl, O.post_process(f32(l), lf, *s), f"{what} mode 1 {s} left")
        assert_same(gr, O.post_process(f32(r), rf, *s), f"{what} mode 1 {s} right")
        assert_same(de.lValid, lv, f"{what} mode 1 left mask"); assert_same(de.rValid, rv, f"{what} mode 1 right mask")


def random_pair(W, H, D, seed, dtype=np.uint8, consistent=0.7):
    rng = np.random.default_rng(seed)
    l = rng.integers(0, D, (H, W))
    r = rng.integers(0, D, (H, W))
    for y in range(H):
        for x in np.flatnonzero(rng.random(W) < consistent):
            r[y, (x - l[y, x]) % W] = l[y, x]
    return l.astype(dtype), r.astype(dtype)


def images(W, H, seed, u8=False):
    rng = np.random.default_rng(seed)
    l8 = (rng.integers(0, 4, (H, W, 3)) * 85).astype(np.uint8)
    r8 = np.roll(l8, -1, axis=1).copy()
    return (l8, r8) if u8 else (f32(l8), f32(r8))


# ---- the reference's own results -------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_full_scenes_against_the_golden(scene, scenes, oracle_scene_results):
    l8, r8, l, r = scenes[scene]
    ref = oracle_scene_results[scene]
    g = GOLD["scenes"][scene]["ref"]
    with DispEst(l, r, 64) as de:
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        assert_same(de.lDisMap, ref["ld"], "WTA left")
        gl, gr = run(de, 2)
        assert [sha(de.lValid), sha(de.rValid), sha(gl), sha(gr)] == [g["lValid"], g["rValid"], g["lFill"], g["rFill"]]
        gl, gr = run(de, 1)
        want = PP.chain(l, r, ref["ld"], ref["rd"], lr=1)
        assert_same(gl, want[0], "mode 1 left"); assert_same(gr, want[1], "mode 1 right")
    pl, pr = f32(posterise(l8)), f32(posterise(r8))
    with DispEst(pl, pr, 64) as de:
        inject_maps(de, ref["ld"], ref["rd"])
        for ent in GOLD["processdm"]["settings"]:
            s = (ent["radius"], float.fromhex(ent["sigma"]), ent["iterations"], ent["weight"])
            gl, gr = run(de, 1, s)
            assert sha(gl) == ent["scenes"][scene]["l"]["ref_sha"], (s, "left")
            assert sha(gr) == ent["scenes"][scene]["r"]["ref_sha"], (s, "right")


def test_synthetic_golden_cases():
    """widths 1 .. 256, rows without a valid pixel, rows valid only at the first or last column, wrap-around, 0 and 1"""
    for ent in GOLD["synthetic"]:
        l, r = CASES[ent["key"] + "_l"], CASES[ent["key"] + "_r"]
        H, W = l.shape
        li, ri = images(W, H, seed=W)
        with DispEst(li, ri, 256) as de:
            inject_maps(de, l, r)
            gl, gr = run(de, 2)
            assert [sha(de.lValid), sha(de.rValid), sha(gl), sha(gr)] == \
                [ent["ref"][k] for k in ("lValid", "rValid", "lFill", "rFill")], ent["key"]
            check_modes(de, li, ri, l, r, ent["key"])


# ---- map formats and sizes --------------------------------------------------------------------------------------------
def test_u16_context_at_d64_equals_u8(scenes, oracle_scene_results):
    _, _, l, r = scenes["Cones"]
    ref = oracle_scene_results["Cones"]
    with DispEst(l, r, 64) as a, DispEst(l, r, 64, map_bits=16) as b:
        for de in (a, b):
            de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        for mode in (2, 1):
            ga, gb = run(a, mode), run(b, mode)
            assert gb[0].dtype == np.uint16
            assert_same(gb[0], ga[0].astype(np.uint16), f"mode {mode} left"); assert_same(gb[1], ga[1].astype(np.uint16), f"mode {mode} right")
            assert_same(b.lValid, a.lValid, "left mask"); assert_same(b.rValid, a.rValid, "right mask")
        assert_same(ga[0], PP.chain(l, r, ref["ld"], ref["rd"], lr=1)[0], "u8 mode 1 left")


@pytest.mark.parametrize("W,H,D", [(150, 10, 300), (97, 6, 600)])
def test_wide_u16_narrower_than_d(W, H, D):
    """map values above the width: the Euclidean wrap on both views"""
    ld, rd = random_pair(W, H, D, seed=D, dtype=np.uint16)
    assert (ld.astype(int) > np.arange(W) + W).any()
    l, r = images(W, H, seed=D)
    with DispEst(l, r, D, map_bits=16) as de:
        inject_maps(de, ld, rd)
        check_modes(de, l, r, ld, rd, f"{W}x{H} D={D}", settings=(DEFAULT, (5, 10.0, 2, "iv2")))


@pytest.mark.parametrize("W,H", [(1, 1), (2, 3), (5, 40), (300, 9), (37, 21), (70, 1), (1, 66)])
@pytest.mark.parametrize("u8", [False, True])
def test_ragged_sizes(W, H, u8):
    ld, rd = random_pair(W, H, 16, seed=W * 1000 + H)
    l, r = images(W, H, seed=W + H, u8=u8)
    with DispEst(l, r, 16) as de:
        inject_maps(de, ld, rd)
        check_modes(de, l, r, ld, rd, f"{W}x{H} u8={u8}", settings=(DEFAULT, (3, 25.5, 1, "off")))


@pytest.mark.parametrize("W,bits", [(7681, 8), (9000, 8), (8200, 16)])
def test_rows_wider_than_shared_memory(W, bits):
    H, D = 3, 20
    ld, rd = random_pair(W, H, D, seed=W, dtype=np.uint16 if bits == 16 else np.uint8)
    ld[1] = 1                                                         # a row with no valid pixel
    l, r = images(W, H, seed=1)
    with DispEst(l, r, D, map_bits=bits) as de:
        inject_maps(de, ld, rd)
        check_modes(de, l, r, ld, rd, f"W={W} u{bits}", settings=((2, 25.5, 1, "exp"),))


def test_post_filter_settings_and_iterations():
    ld, rd = random_pair(83, 61, 32, seed=5, consistent=0.5)
    l, r = images(83, 61, seed=5)
    with DispEst(l, r, 32) as de:
        inject_maps(de, ld, rd)
        check_modes(de, l, r, ld, rd, "settings",
                    settings=((16, 25.5, 2, "exp"), (9, 25.5, 16, "exp"), (5, 3.0, 16, "iv1"), (32, 25.5, 1, "iv2"),
                              (9, 25.5, 2, "exp")))


def test_fgf_branch(scenes):
    _, _, l, r = (a[:120, :200].copy() for a in scenes["Teddy"])
    with DispEst(np.ascontiguousarray(l), np.ascontiguousarray(r), 48) as de:
        de.CostConst_GPU(); de.CostFilter_FGF_GPU(); de.DispSelect_GPU()
        ld, rd = de.lDisMap.copy(), de.rDisMap.copy()
        check_modes(de, l, r, ld, rd, "FGF")


# ---- sharded ----------------------------------------------------------------------------------------------------------
def test_sharded_key_path_and_selection_maps_untouched():
    W, H, D, G = 160, 48, 64, 2
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=4)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    L = capi.lib()
    with DispEst(l, r, D) as full:
        full.CostConst_GPU(); full.CostFilter_GPU(); full.DispSelect_GPU()
        ld, rd = full.lDisMap.copy(), full.rDisMap.copy()
        check_modes(full, l, r, ld, rd, "unsharded")
        assert_same(device_map(full, 2, np.uint8), ld, "selection map left after the check")
        assert_same(device_map(full, 3, np.uint8), rd, "selection map right after the check")
        assert_same(device_map(full, 6, np.uint8), full.lValid, "device left mask")
        assert_same(device_map(full, 7, np.uint8), full.rValid, "device right mask")
    import torch
    shards = [DispEst(l, r, D, d_begin=shard_range(D, G, k)[0], d_count=shard_range(D, G, k)[1]) for k in range(G)]
    try:
        keys = [torch.empty((2, W * H), dtype=torch.int64, device="cuda") for _ in range(G)]
        for k, de in enumerate(shards):
            de.CostConst_GPU(); de.CostFilter_GPU()
            capi.check(L.psm_disp_select_keys(de.handle, keys[k][0].data_ptr(), keys[k][1].data_ptr()), de.handle)
            de.sync()
        gathered = torch.stack(keys, 1).contiguous()
        de = shards[0]
        u8 = np.zeros((H, W), np.uint8), np.zeros((H, W), np.uint8)
        capi.check(L.psm_disp_reduce_keys(de.handle, gathered[0].data_ptr(), gathered[1].data_ptr(), G,
                                          ptr(u8[0]), W, ptr(u8[1]), W), de.handle)
        assert_same(u8[0], ld, "keys left")
        check_modes(de, l, r, ld, rd, "key path")
        assert_same(device_map(de, 2, np.uint8), ld, "key-path selection map left")
        assert_same(device_map(de, 3, np.uint8), rd, "key-path selection map right")
    finally:
        for de in shards:
            de.close()


@pytest.mark.parametrize("G", [2, 8])
def test_sharded_p2p_exchange_untouched(G):
    W, H, D = 200, 40, 64
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=21)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    L = capi.lib()
    with DispEst(l, r, D) as full:
        full.CostConst_GPU(); full.CostFilter_GPU(); full.DispSelect_GPU()
        ld, rd = full.lDisMap.copy(), full.rDisMap.copy()
    shards = [DispEst(l, r, D, d_begin=shard_range(D, G, k)[0], d_count=shard_range(D, G, k)[1]) for k in range(G)]
    try:
        bufs = (C.c_void_p * G)()
        for k, de in enumerate(shards):
            de.CostConst_GPU(); de.CostFilter_GPU()
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
            de = shards[k]
            check_modes(de, l, r, ld, rd, f"{G}-way p2p rank {k}")
            xl, xr = np.zeros((H, W), np.uint8), np.zeros((H, W), np.uint8)
            capi.check(L.psm_disp_fetch_p2p(de.handle, ptr(xl), W, ptr(xr), W), de.handle)
            assert_same(xl, ld, f"{G}-way exchange map left after the check"); assert_same(xr, rd, "exchange map right")
    finally:
        for de in shards:
            de.close()


# ---- modes, launches, errors ------------------------------------------------------------------------------------------
def test_switching_modes_between_frames_and_back():
    ld, rd = random_pair(64, 30, 24, seed=9)
    l, r = images(64, 30, seed=9)
    want = {m: PP.chain(l, r, ld, rd, lr=m) for m in (0, 1, 2)}
    with DispEst(l, r, 24) as de:
        inject_maps(de, ld, rd)
        first = run(de, None)
        assert_same(first[0], want[0][0], "default is off")
        for m in (1, 2, 0, 2, 1, 0):
            got = run(de, m)
            assert_same(got[0], want[m][0], f"mode {m} left"); assert_same(got[1], want[m][1], f"mode {m} right")
        # next frame: flipped maps in mode 2, then back to 0
        ld2, rd2 = np.ascontiguousarray(ld[::-1]), np.ascontiguousarray(rd[::-1])
        inject_maps(de, ld2, rd2)
        got = run(de, 2)
        assert_same(got[0], LR.lr_check_fill(ld2, rd2)[2], "frame 2 mode 2")
        got = run(de, 0)
        assert_same(got[0], O.post_process(l, ld2), "frame 2 mode 0")


def test_launch_counts_and_stage_time():
    ld, rd = random_pair(64, 48, 16, seed=11)
    l, r = images(64, 48, seed=11)
    with DispEst(l, r, 16) as de:
        inject_maps(de, ld, rd)
        for mode in (0, 1, 2):
            for it in (1, 3):
                de.setLRCheck(mode); de.setPostFilter(9, 25.5, it, "exp")
                n = de.launch_count()
                assert de.PostProcess_GPU() == 0
                want = {0: 4 * it, 1: 1 + 4 * it, 2: 1}[mode]
                assert de.launch_count() - n == want, (mode, it)
                assert de.stage_ms(5) > 0


def test_invalid_arguments_and_states():
    ld, rd = random_pair(40, 30, 16, seed=2)
    l, r = images(40, 30, seed=2)
    L = capi.lib()
    mask = np.zeros((30, 40), np.uint8)
    with DispEst(l, r, 16) as de:
        h = de.handle
        p = C.c_void_p(1)
        assert L.psm_device_ptr(h, 6, C.byref(p), None) == 0 and not p.value        # no mask before the first check
        assert L.psm_device_ptr(h, 8, C.byref(p), None) == capi.PSM_EINVAL
        assert L.psm_read_valid_mask(h, 0, ptr(mask), 40) == capi.PSM_ESTATE
        inject_maps(de, ld, rd)
        want = run(de, 2)
        for bad in (-1, 3, 4, 100):
            assert L.psm_set_lr_check(h, bad) == capi.PSM_EINVAL and L.psm_last_error(h)
            got = run(de, None)
            assert_same(got[0], want[0], f"left after rejected mode {bad}")
        with pytest.raises(capi.PsmError):
            de.setLRCheck(5)
        assert L.psm_read_valid_mask(h, 0, ptr(mask), 40) == 0
        assert_same(mask, LR.lr_check(ld, rd)[0], "read_valid_mask")
        for view, dst, step in ((2, ptr(mask), 40), (-1, ptr(mask), 40), (0, None, 40), (1, ptr(mask), 39)):
            assert L.psm_read_valid_mask(h, view, dst, step) == capi.PSM_EINVAL, (view, step)
        assert L.psm_read_valid_mask(None, 0, ptr(mask), 40) == capi.PSM_EINVAL
        assert L.psm_set_lr_check(None, 1) == capi.PSM_EINVAL
        de.DispSelect_GPU()                                                   # a new selection: the masks are stale
        assert L.psm_read_valid_mask(h, 1, ptr(mask), 40) == capi.PSM_ESTATE
        run(de, 1)
        assert L.psm_read_valid_mask(h, 1, ptr(mask), 40) == 0
        run(de, 0)                                                            # a post-process without the check
        assert L.psm_read_valid_mask(h, 0, ptr(mask), 40) == capi.PSM_ESTATE
    with DispEst(l, r, 16) as de:                                             # before images / selection
        de.setLRCheck(2)
        assert L.psm_post_process_device(de.handle) == capi.PSM_ESTATE
        assert L.psm_read_valid_mask(de.handle, 0, ptr(mask), 40) == capi.PSM_ESTATE


def test_1080p_row_band():
    W, H, D = 1920, 1080, 64
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=5)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    with DispEst(l, r, D) as de:
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        ld, rd = de.lDisMap.copy(), de.rDisMap.copy()
        lv, rv, lf, rf = LR.lr_check_fill(ld, rd)
        gl, gr = run(de, 2)
        assert_same(gl, lf, "1080p mode 2 left"); assert_same(gr, rf, "1080p mode 2 right")
        assert_same(de.lValid, lv, "1080p left mask"); assert_same(de.rValid, rv, "1080p right mask")
        assert 0.2 < lv.mean() < 1.0
        gl, gr = run(de, 1, DEFAULT)
    band = 64 + 9
    assert_same(gl[:64], O.post_process(l[:band], lf[:band])[:64], "1080p mode 1 left, top 64 rows")
    assert_same(gr[:64], O.post_process(r[:band], rf[:band])[:64], "1080p mode 1 right, top 64 rows")


def test_cpp_demo_mode_argument(tmp_path, scenes, oracle_scene_results):
    exe = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
    if not os.path.exists(exe):
        pytest.skip("dispest_demo not built")
    _, _, l, r = scenes["Cones"]
    H, W, _ = l.shape
    l.tofile(tmp_path / "l.f32"); r.tofile(tmp_path / "r.f32")
    ref = oracle_scene_results["Cones"]
    base = [exe, str(W), str(H), "64", str(tmp_path / "l.f32"), str(tmp_path / "r.f32"), str(tmp_path / "l.u8"),
            str(tmp_path / "r.u8"), "8", "0.0001", "0.9", "inf", "inf", "9", "25.5", "1", "exp"]
    for mode in (1, 2, 0):
        out = subprocess.run(base + [str(mode)], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr
        want = PP.chain(l, r, ref["ld"], ref["rd"], lr=mode)
        assert_same(np.fromfile(tmp_path / "l.u8", np.uint8).reshape(H, W), want[0], f"C++ facade left, mode {mode}")
        assert_same(np.fromfile(tmp_path / "r.u8", np.uint8).reshape(H, W), want[1], f"C++ facade right, mode {mode}")
    bad = subprocess.run(base + ["3"], capture_output=True, text=True, timeout=300)
    assert bad.returncode == 1 and "left-right check mode" in bad.stderr
