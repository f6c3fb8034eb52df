"""GPU: the post-filter at any psm_set_post_filter setting, bit-exact against the CPU restatement tests/pp_oracle.c
(pinned to the reference's JointWMF.h by golden_pp.json).  Every comparison goes through the C-ABI.

Maps are injected through the C-ABI: after CostConst / CostFilter, one-hot cost slices (0 at the wanted disparity, 1
elsewhere) are written with psm_write_cost_slice, and the winner-take-all returns exactly the wanted maps.  The
post-filter then runs on the device maps with the context's own guide planes."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle import oracle as O
from primestereomatch_b200 import DispEst, capi, synth
import pp_oracle as P

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN, "golden_pp.json")) as f:
    GOLD = json.load(f)["settings"]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def posterise(img8, masks=(0xE0, 0xE0, 0xC0)):
    return (img8 & np.array(masks, np.uint8)).astype(np.uint8)


def assert_same(a, b, what):
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {a.size} differ, first at {list(i)}: {a[i]!r} vs {b[i]!r}")


def inject_maps(de, ld, rd):
    """Make the context's disparity maps exactly ld / rd (values in 1 .. de.maxDis - 1: the WTA never selects d = 0,
    DispSel.cpp:96)."""
    assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
    for d in range(de.maxDis):
        de.write_cost_slice(0, d, (ld != d).astype(np.float32))
        de.write_cost_slice(1, d, (rd != d).astype(np.float32))
    assert de.DispSelect_GPU() == 0
    assert np.array_equal(de.lDisMap, ld) and np.array_equal(de.rDisMap, rd)


def post(de, setting):
    """post-process at `setting` (None: never call the setter) -> (left, right) copies"""
    if setting is not None:
        assert de.setPostFilter(*setting) == 0
    assert de.PostProcess_GPU() == 0
    return de.lDisMap.copy(), de.rDisMap.copy()


def f32(img):
    return O.u8_to_f32(img) if img.dtype == np.uint8 else img


def check(de, l, r, ld, rd, setting, what):
    r_, sigma, it, weight = setting
    gl, gr = post(de, setting)
    assert_same(gl, P.post_process(f32(l), ld, r_, sigma, it, weight), f"{what} left")
    assert_same(gr, P.post_process(f32(r), rd, r_, sigma, it, weight), f"{what} right")


def random_case(W, H, D, seed, u8=False):
    rng = np.random.default_rng(seed)
    l8 = (rng.integers(0, 4, (H, W, 3)) * 85).astype(np.uint8)      # few colours: many equal weights and ties
    r8 = np.roll(l8, -1, axis=1).copy()
    # piecewise-constant maps with noise, like real disparity maps
    base = np.repeat(np.repeat(rng.integers(1, D, ((H + 3) // 4, (W + 3) // 4)), 4, 0), 4, 1)[:H, :W]
    noise = rng.integers(1, D, (H, W))
    ld = np.where(rng.random((H, W)) < 0.2, noise, base).astype(np.uint8)
    rd = np.where(rng.random((H, W)) < 0.2, np.roll(noise, 3), base).astype(np.uint8)
    if u8:
        return l8, r8, ld, rd
    return f32(l8), f32(r8), ld, rd


@pytest.fixture(scope="module")
def full_scenes(scenes, oracle, oracle_scene_results):
    out = {}
    for name, (l8, r8, _, _) in scenes.items():
        ref = oracle_scene_results[name]
        out[name] = (oracle.u8_to_f32(posterise(l8)), oracle.u8_to_f32(posterise(r8)), ref["ld"], ref["rd"])
    return out


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_full_scenes_at_every_golden_setting(scene, full_scenes):
    l, r, ld, rd = full_scenes[scene]
    with DispEst(l, r, 64) as de:
        inject_maps(de, ld, rd)
        for ent in GOLD:
            setting = (ent["radius"], float.fromhex(ent["sigma"]), ent["iterations"], ent["weight"])
            gl, gr = post(de, setting)
            assert sha(gl) == ent["scenes"][scene]["l"]["sha"], f"{ent['key']} {scene} left"
            assert sha(gr) == ent["scenes"][scene]["r"]["sha"], f"{ent['key']} {scene} right"


def test_natural_image_at_other_settings(scenes, oracle_scene_results):
    """> 256 colours (no clustering question for the restatement): the real pipeline's maps, both views."""
    _, _, l, r = scenes["Teddy"]
    ref = oracle_scene_results["Teddy"]
    with DispEst(l, r, 64) as de:
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        assert np.array_equal(de.lDisMap, ref["ld"])
        for setting in ((16, 25.5, 1, "exp"), (9, 40.0, 2, "iv1"), (32, 3.0, 1, "iv2")):
            check(de, l, r, ref["ld"], ref["rd"], setting, f"Teddy natural {setting}")


def test_every_radius_on_a_crop(full_scenes):
    l, r, ld, rd = (a[100:172, 150:246] for a in full_scenes["Cones"])
    with DispEst(np.ascontiguousarray(l), np.ascontiguousarray(r), 64) as de:
        inject_maps(de, np.ascontiguousarray(ld), np.ascontiguousarray(rd))
        for radius in range(1, 33):
            check(de, l, r, ld, rd, (radius, 25.5, 1, "exp"), f"radius {radius}")
        check(de, l, r, ld, rd, (9, float(np.nextafter(np.float32(25.5), np.float32(np.inf))), 1, "exp"),
              "generic kernel at the default filter")


@pytest.mark.parametrize("weight", ["exp", "iv1", "iv2", "off"])
def test_weight_types_at_sigma_ends(weight, full_scenes):
    l, r, ld, rd = (np.ascontiguousarray(a[200:260, 40:130]) for a in full_scenes["Teddy"])
    with DispEst(l, r, 64) as de:
        inject_maps(de, ld, rd)
        for sigma in (2.0 ** -16, 1.0, 25.5, 2.0 ** 16):
            for radius in (3, 9, 24):
                check(de, l, r, ld, rd, (radius, sigma, 1, weight), f"{weight} sigma {sigma} radius {radius}")


@pytest.mark.parametrize("radius", [9, 6])
def test_iterations(radius):
    l, r, ld, rd = random_case(83, 61, 32, seed=radius)
    with DispEst(l, r, 32) as de:
        inject_maps(de, ld, rd)
        for it in (1, 2, 5, 16):
            check(de, l, r, ld, rd, (radius, 25.5, it, "exp"), f"radius {radius} iterations {it}")
            check(de, l, r, ld, rd, (radius, 7.0, it, "iv2"), f"radius {radius} iv2 iterations {it}")


@pytest.mark.parametrize("W,H", [(1, 1), (5, 40), (300, 9), (7, 3), (37, 21), (70, 1), (1, 66)])
@pytest.mark.parametrize("u8", [False, True])
def test_ragged_sizes(W, H, u8):
    l, r, ld, rd = random_case(W, H, 16, seed=W * 1000 + H, u8=u8)
    with DispEst(l, r, 16) as de:
        inject_maps(de, ld, rd)
        for setting in ((1, 25.5, 1, "exp"), (9, 25.5, 2, "exp"), (5, 3.0, 1, "iv1"), (32, 25.5, 1, "iv2"),
                        (17, 25.5, 3, "off"), (9, 25.5, 1, "exp")):
            check(de, l, r, ld, rd, setting, f"{W}x{H} u8={u8} {setting}")


def test_1080p_radius_32_row_band():
    W, H, D, r_ = 1920, 1080, 64, 32
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=5)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    with DispEst(l, r, D) as de:
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        ld, rd = de.lDisMap.copy(), de.rDisMap.copy()
        gl, gr = post(de, (r_, 25.5, 1, "exp"))
    band = 64 + r_        # the clipped window of rows [0, 64) lies inside rows [0, 64 + r)
    assert_same(gl[:64], P.post_process(l[:band], ld[:band], r_)[:64], "1080p left, top 64 rows")
    assert_same(gr[:64], P.post_process(r[:band], rd[:band], r_)[:64], "1080p right, top 64 rows")


def test_switching_settings_between_frames(full_scenes):
    l, r, ld, rd = (np.ascontiguousarray(a[:80, :120]) for a in full_scenes["Teddy"])
    with DispEst(l, r, 64) as de:
        inject_maps(de, ld, rd)
        default = post(de, None)
        assert_same(default[0], P.post_process(l, ld), "default before any setter")
        for setting in ((12, 25.5, 1, "exp"), (12, 60.0, 1, "exp"), (12, 60.0, 1, "iv1"), (4, 60.0, 2, "iv1"),
                        (9, 25.5, 1, "exp"), (9, 25.5, 2, "exp"), (9, 25.5, 1, "off"), P.DEFAULT):
            check(de, l, r, ld, rd, setting, f"after switching to {setting}")
        again = post(de, P.DEFAULT)
        assert_same(again[0], default[0], "back to the default")
        # a new frame with the same setting reuses the cached table
        assert de.setPostFilter(20, 5.0, 1, "iv2") == 0
        check(de, l, r, ld, rd, (20, 5.0, 1, "iv2"), "frame 1")
        l2, r2 = np.ascontiguousarray(l[:, ::-1]), np.ascontiguousarray(r[:, ::-1])
        de.setInputImages(l2, r2)
        inject_maps(de, np.ascontiguousarray(ld[:, ::-1]), np.ascontiguousarray(rd[:, ::-1]))
        check(de, l2, r2, ld[:, ::-1], rd[:, ::-1], (20, 5.0, 1, "iv2"), "frame 2")


def test_launch_counts_and_stage_time():
    l, r, ld, rd = random_case(64, 48, 16, seed=11)
    with DispEst(l, r, 16) as de:
        inject_maps(de, ld, rd)
        n = de.launch_count(); post(de, None); base = de.launch_count() - n
        assert base == 4                                   # pack + filter per view, as before
        for setting in ((9, 25.5, 1, "exp"), (9, 25.5, 3, "exp"), (16, 25.5, 1, "exp"), (16, 2.0, 5, "iv2"), (9, 25.5, 16, "off")):
            n = de.launch_count(); post(de, setting)
            assert de.launch_count() - n == 2 * 2 * setting[2], setting
            assert de.stage_ms(5) > 0


def test_invalid_settings_leave_the_context_unchanged():
    l, r, ld, rd = random_case(40, 30, 16, seed=2)
    L = capi.lib()
    with DispEst(l, r, 16) as de:
        inject_maps(de, ld, rd)
        good = (5, 9.0, 2, "iv1")
        want = post(de, good)
        bad = [(0, 25.5, 1, 0), (33, 25.5, 1, 0), (-1, 25.5, 1, 0), (9, 2.0 ** -17, 1, 0), (9, 2.0 ** 17, 1, 0),
               (9, 0.0, 1, 0), (9, -25.5, 1, 0), (9, float("nan"), 1, 0), (9, float("inf"), 1, 0), (9, -float("inf"), 1, 0),
               (9, 25.5, 0, 0), (9, 25.5, 17, 0), (9, 25.5, -3, 0), (9, 25.5, 1, 3), (9, 25.5, 1, 4), (9, 25.5, 1, 6),
               (9, 25.5, 1, -1)]
        for b in bad:
            assert L.psm_set_post_filter(de.handle, *b) == capi.PSM_EINVAL, b
            assert L.psm_last_error(de.handle)
            got = post(de, None)
            assert_same(got[0], want[0], f"left after rejected {b}")
            assert_same(got[1], want[1], f"right after rejected {b}")
        for name in ("cos", "jac", "EXP", "median", 0):
            with pytest.raises(capi.PsmError):
                de.setPostFilter(9, 25.5, 1, name)
        with pytest.raises(capi.PsmError):
            de.setPostFilter(9, float("nan"))
        assert_same(post(de, None)[0], want[0], "after rejected Python calls")
        # both sigma ends are accepted
        assert L.psm_set_post_filter(de.handle, 9, 2.0 ** -16, 1, 0) == 0
        assert L.psm_set_post_filter(de.handle, 9, 2.0 ** 16, 1, 0) == 0
    assert L.psm_set_post_filter(None, 9, 25.5, 1, 0) == capi.PSM_EINVAL


def test_cpp_facade_set_post_filter(tmp_path, scenes, oracle_scene_results):
    exe = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
    if not os.path.exists(exe):
        pytest.skip("dispest_demo not built")
    _, _, l, r = scenes["Cones"]
    H, W, _ = l.shape
    l.tofile(tmp_path / "l.f32"); r.tofile(tmp_path / "r.f32")
    ref = oracle_scene_results["Cones"]
    for setting in (("12", "40", "2", "iv2"), ("9", "25.5", "1", "exp")):
        out = subprocess.run([exe, str(W), str(H), "64", str(tmp_path / "l.f32"), str(tmp_path / "r.f32"),
                              str(tmp_path / "l.u8"), str(tmp_path / "r.u8"), "8", "0.0001", "0.9", "inf", "inf", *setting],
                             capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr
        rad, sig, it, w = int(setting[0]), float(setting[1]), int(setting[2]), setting[3]
        ld = np.fromfile(tmp_path / "l.u8", np.uint8).reshape(H, W)
        rd = np.fromfile(tmp_path / "r.u8", np.uint8).reshape(H, W)
        assert_same(ld, P.post_process(l, ref["ld"], rad, sig, it, w), f"C++ facade left at {setting}")
        assert_same(rd, P.post_process(r, ref["rd"], rad, sig, it, w), f"C++ facade right at {setting}")
    bad = subprocess.run([exe, str(W), str(H), "64", str(tmp_path / "l.f32"), str(tmp_path / "r.f32"),
                          str(tmp_path / "l.u8"), str(tmp_path / "r.u8"), "8", "0.0001", "0.9", "inf", "inf",
                          "9", "25.5", "1", "cos"], capture_output=True, text=True, timeout=300)
    assert bad.returncode == 1 and "weight type" in bad.stderr
