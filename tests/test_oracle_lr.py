"""CPU: the left-right check and fill restatement (tests/lr_oracle.py) against the reference's own compiled PP.cpp
(golden_lr.json, written by tests/golden/make_golden_lr.py), against a direct per-pixel restatement of lrCheck /
fillInv written here, and its properties, including the Euclidean remainder where the reference is undefined."""
import hashlib
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import oracle as O
import lr_oracle as LR
import pp_chain as PP

with open(os.path.join(GOLDEN, "golden_lr.json")) as f:
    GOLD = json.load(f)
CASES = np.load(os.path.join(GOLDEN, "lr_cases.npz"))


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def hashes(arrs):
    return dict(zip(("lValid", "rValid", "lFill", "rFill"), (sha(a) for a in arrs)))


def posterise(img8, masks=(0xE0, 0xE0, 0xC0)):
    return (img8 & np.array(masks, np.uint8)).astype(np.uint8)


def direct(l, r):
    """lrCheck / fillInv pixel by pixel, as PP.cpp:17-143 loops, with Python's (Euclidean) % for the wrap"""
    H, W = l.shape
    lv, rv = np.zeros((H, W), np.uint8), np.zeros((H, W), np.uint8)
    for y in range(H):
        for x in range(W):
            dl, dr = int(l[y, x]), int(r[y, x])
            lv[y, x] = dl == int(r[y, (x - dl) % W]) and dl >= 2
            rv[y, x] = dr == int(l[y, (x + dr) % W]) and dr >= 2
    out = []
    for m, v in ((l, lv), (r, rv)):
        f = m.copy()
        for y in range(H):
            for x in range(W):
                if v[y, x]:
                    continue
                a = next((int(m[y, i]) for i in range(x, -1, -1) if v[y, i]), None)
                b = next((int(m[y, i]) for i in range(x, W) if v[y, i]), None)
                if a is not None or b is not None:
                    f[y, x] = min(c for c in (a, b) if c is not None)
        out.append(f)
    return lv, rv, out[0], out[1]


def random_pair(W, H, D, seed, dtype=np.uint8, consistent=0.7):
    rng = np.random.default_rng(seed)
    l = rng.integers(0, D, (H, W))
    r = rng.integers(0, D, (H, W))
    for y in range(H):
        for x in np.flatnonzero(rng.random(W) < consistent):
            r[y, (x - l[y, x]) % W] = l[y, x]
    return l.astype(dtype), r.astype(dtype)


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_scenes_equal_the_reference(scene, oracle_scene_results):
    ent = GOLD["scenes"][scene]
    assert ent["ref"] == ent["restatement"]
    ref = oracle_scene_results[scene]
    got = LR.lr_check_fill(ref["ld"], ref["rd"])
    assert hashes(got) == ent["ref"]
    assert [int(got[0].sum()), int(got[1].sum())] == ent["valid_pixels"]


def test_synthetic_cases_equal_the_reference():
    assert len(GOLD["synthetic"]) >= 10
    for ent in GOLD["synthetic"]:
        l, r = CASES[ent["key"] + "_l"], CASES[ent["key"] + "_r"]
        assert l.shape == (ent["H"], ent["W"])
        assert (l.astype(int) <= np.arange(ent["W"]) + ent["W"]).all()      # the reference's domain
        assert hashes(LR.lr_check_fill(l, r)) == ent["ref"], ent["key"]


def test_process_dm_with_the_check_equals_the_reference(scenes, oracle_scene_results):
    for ent in GOLD["processdm"]["settings"]:
        setting = (ent["radius"], float.fromhex(ent["sigma"]), ent["iterations"], ent["weight"])
        for scene in ("Cones", "Teddy"):
            l8, r8, _, _ = scenes[scene]
            ref = oracle_scene_results[scene]
            gl, gr, _ = PP.chain(O.u8_to_f32(posterise(l8)), O.u8_to_f32(posterise(r8)), ref["ld"], ref["rd"], lr=1,
                                  setting=setting)
            for v, g in (("l", gl), ("r", gr)):
                e = ent["scenes"][scene][v]
                assert sha(g) == e["sha"], (setting, scene, v)
                assert e["differ"] == 0 and e["ref_sha"] == e["sha"], (setting, scene, v)


@pytest.mark.parametrize("W,H,D,seed", [(1, 4, 3, 0), (2, 3, 5, 1), (3, 5, 4, 2), (7, 6, 9, 3), (33, 4, 20, 4), (40, 3, 64, 5)])
def test_equals_the_direct_restatement(W, H, D, seed):
    l, r = random_pair(W, H, D, seed)
    for a, b in zip(LR.lr_check_fill(l, r), direct(l, r)):
        assert np.array_equal(a, b)


def test_euclidean_remainder_beyond_the_reference():
    """map values above x + W (narrow images, or wide D on u16 maps): the gather wraps with the non-negative remainder"""
    for seed, (W, H, D) in enumerate([(3, 4, 40), (5, 6, 300), (17, 3, 4000), (1, 2, 7)]):
        dtype = np.uint16 if D > 256 else np.uint8
        l, r = random_pair(W, H, D, seed, dtype)
        assert (l.astype(int) > np.arange(W) + W).any()
        got = LR.lr_check_fill(l, r)
        for a, b in zip(got, direct(l, r)):
            assert np.array_equal(a, b)
        # spelled out for one pixel: x = 0, d = 2W + 1 reads column (0 - (2W + 1)) mod W = W - 1
        l2, r2 = np.zeros((1, W), dtype), np.zeros((1, W), dtype)
        l2[0, 0] = 2 * W + 1 if 2 * W + 1 >= 2 else 2
        r2[0, W - 1] = l2[0, 0]
        assert LR.lr_check(l2, r2)[0][0, 0] == 1


def test_properties():
    for seed in range(6):
        l, r = random_pair(50, 8, 30, seed, consistent=0.4)
        l[3] = 1                                          # a row of disparity 1: never valid
        lv, rv, lf, rf = LR.lr_check_fill(l, r)
        for m, v, f in ((l, lv, lf), (r, rv, rf)):
            assert set(np.unique(v)) <= {0, 1}
            assert np.array_equal(f[v == 1], m[v == 1])             # valid pixels unchanged
            assert (v[m < 2] == 0).all()
            for y in range(m.shape[0]):
                idx = np.flatnonzero(v[y])
                if idx.size == 0:
                    assert np.array_equal(f[y], m[y])               # rows without a valid pixel unchanged
                    continue
                for x in np.flatnonzero(v[y] == 0):
                    left, right = idx[idx <= x], idx[idx >= x]
                    cands = ([m[y, left[-1]]] if left.size else []) + ([m[y, right[0]]] if right.size else [])
                    assert f[y, x] == min(cands)
        assert (lv[3] == 0).all() and np.array_equal(lf[3], l[3])


def test_u16_equals_u8_below_256():
    for seed in range(4):
        l, r = random_pair(61, 7, 256, seed)
        a = LR.lr_check_fill(l, r)
        b = LR.lr_check_fill(l.astype(np.uint16), r.astype(np.uint16))
        for x, y in zip(a, b):
            assert np.array_equal(x.astype(np.uint16), y.astype(np.uint16))
        assert b[2].dtype == np.uint16


def test_modes():
    l8 = (np.random.default_rng(0).integers(0, 4, (20, 30, 3)) * 85).astype(np.uint8)
    img = O.u8_to_f32(l8)
    l, r = random_pair(30, 20, 16, 7)
    _, _, lf, rf = LR.lr_check_fill(l, r)
    assert all(np.array_equal(a, b) for a, b in zip(PP.chain(img, img, l, r), (O.post_process(img, l), O.post_process(img, r))))
    assert all(np.array_equal(a, b) for a, b in zip(PP.chain(img, img, l, r, lr=2), (lf, rf)))
    s = (4, 10.0, 2, "iv1")
    assert all(np.array_equal(a, b) for a, b in
               zip(PP.chain(img, img, l, r, lr=1, setting=s), (O.post_process(img, lf, *s), O.post_process(img, rf, *s))))
