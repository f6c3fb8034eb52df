"""CPU: the post-filter restatement at any psm_set_post_filter setting (oracle.post_process, orc_wmf in
oracle/stereo_oracle.c) against the reference's own JointWMF.h as recorded in tests/golden/golden_pp.json
(make_golden_pp.py) and ref_outputs.json, and against hand-checkable cases of the definition (DESIGN.md section 13)."""
import hashlib
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import oracle as O


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def posterise(img8, masks=(0xE0, 0xE0, 0xC0)):
    return (img8 & np.array(masks, np.uint8)).astype(np.uint8)


with open(os.path.join(GOLDEN, "golden_pp.json")) as f:
    GOLD = json.load(f)["settings"]


def setting(ent):
    return ent["radius"], float.fromhex(ent["sigma"]), ent["iterations"], ent["weight"]


@pytest.fixture(scope="module")
def pp_inputs(scenes, oracle, oracle_scene_results):
    """{scene: {view: (posterised f32 feature image, D = 64 WTA map)}} -- the inputs of golden_pp.json"""
    out = {}
    for name, (l8, r8, _, _) in scenes.items():
        ref = oracle_scene_results[name]
        out[name] = {"l": (oracle.u8_to_f32(posterise(l8)), ref["ld"]), "r": (oracle.u8_to_f32(posterise(r8)), ref["rd"])}
    return out


def test_golden_covers_the_settings():
    keys = {(e["radius"], e["sigma"], e["iterations"], e["weight"]) for e in GOLD}
    assert (9, float(25.5).hex(), 1, "exp") in keys
    assert {e["weight"] for e in GOLD} == {"exp", "iv1", "iv2", "off"}
    assert {e["radius"] for e in GOLD} >= {4, 9, 16, 20, 32}
    assert {float.fromhex(e["sigma"]) for e in GOLD} >= {2.0 ** -16, 10.0, 25.5, 80.0, 2.0 ** 16}
    assert max(e["iterations"] for e in GOLD) >= 3


@pytest.mark.parametrize("ent", GOLD, ids=[e["key"] for e in GOLD])
def test_restatement_matches_golden(ent, pp_inputs):
    r, sigma, it, weight = setting(ent)
    assert sha(O.weight_table(sigma, weight)) == ent["table_sha"]
    for name, views in pp_inputs.items():
        for view, (img, disp) in views.items():
            want = ent["scenes"][name][view]
            assert want["colours"] <= 256       # every colour is its own cluster: the reference's result is RNG-free
            got = O.post_process(img, disp, r, sigma, it, weight)
            assert sha(got) == want["sha"], f"{ent['key']} {name}/{view}"
            # the reference's float cut-point search agrees exactly, or differs by the count its float balances give
            assert (want["differ"] == 0) == (want["ref_sha"] == want["sha"])


def test_reference_agreement_counts():
    """The disagreement with the reference is pinned per setting; it is zero at the default and largest for iv2 at the
    smallest sigma, where the weights span 2^36 and the reference's float balance drops the small ones (DESIGN.md)."""
    by = {e["key"]: e for e in GOLD}
    default = by[f"9/{float(25.5).hex()}/1/exp"]
    assert all(v["differ"] == 0 for s in default["scenes"].values() for v in s.values())
    worst = max(GOLD, key=lambda e: sum(v["differ"] for s in e["scenes"].values() for v in s.values()))
    assert (worst["weight"], float.fromhex(worst["sigma"])) == ("iv2", 2.0 ** -16)
    for e in GOLD:
        if e is not worst:
            assert all(v["differ"] <= 25 for s in e["scenes"].values() for v in s.values()), e["key"]


def test_default_equals_reference(pp_inputs):
    """The default call is PP::processDM's filter and gives the reference's own JointWMF results (ref_outputs.json)."""
    with open(os.path.join(GOLDEN, "ref_outputs.json")) as f:
        ref_pp = json.load(f)["pp"]
    for name, views in pp_inputs.items():
        for view, (img, disp) in views.items():
            got = O.post_process(img, disp)
            assert np.array_equal(got, O.post_process(img, disp, 9, 25.5, 1, "exp"))   # PP::processDM's arguments
            assert sha(got) == ref_pp[name][view]["sha"]


def lower_median(disp, y, x, r):
    s = np.sort(disp[max(0, y - r):y + r + 1, max(0, x - r):x + r + 1].ravel())
    return s[(len(s) + 1) // 2 - 1]      # min v with 2 * #(I <= v) >= n


@pytest.mark.parametrize("r", [1, 3, 9, 32])
def test_off_is_the_plain_lower_median_of_the_clipped_window(r):
    rng = np.random.default_rng(r)
    H, W = 23, 41
    img = rng.random((H, W, 3)).astype(np.float32)
    disp = rng.integers(0, 200, (H, W)).astype(np.uint8)
    got = O.post_process(img, disp, r, 25.5, 1, "off")
    for y in range(H):
        for x in range(W):
            assert got[y, x] == lower_median(disp, y, x, r), (y, x)


@pytest.mark.parametrize("weight", ["exp", "iv1", "iv2", "off"])
def test_two_iterations_equal_two_single_passes(weight):
    rng = np.random.default_rng(7)
    img = (rng.integers(0, 4, (40, 57, 3)) / 3.0).astype(np.float32)
    disp = rng.integers(0, 64, (40, 57)).astype(np.uint8)
    once = O.post_process(img, disp, 5, 12.0, 1, weight)
    twice = O.post_process(img, once, 5, 12.0, 1, weight)
    assert np.array_equal(O.post_process(img, disp, 5, 12.0, 2, weight), twice)
    assert not np.array_equal(once, disp)


@pytest.mark.parametrize("weight", ["exp", "iv1", "iv2"])
def test_radius_at_least_the_image_gives_whole_image_windows(weight):
    rng = np.random.default_rng(3)
    H, W = 9, 13
    img = rng.random((H, W, 3)).astype(np.float32)
    disp = rng.integers(0, 30, (H, W)).astype(np.uint8)
    got = O.post_process(img, disp, 13, 25.5, 1, weight)
    assert np.array_equal(got, O.post_process(img, disp, 32, 25.5, 1, weight))
    # direct evaluation over every pixel of the image
    c = (O.to_u8x255(img) >> 2).astype(np.int64).reshape(-1, 3)
    t = O.weight_table(25.5, weight).astype(np.int64)
    d = disp.reshape(-1).astype(np.int64)
    for p in range(H * W):
        diff = c - c[p]
        k = np.abs(diff).sum(1) if weight == "iv1" else (diff * diff).sum(1)
        w = t[k]
        hist = np.zeros(256, np.int64)
        np.add.at(hist, d, w)
        cum = np.cumsum(hist)
        assert got.reshape(-1)[p] == int(np.argmax(2 * cum >= cum[-1])), p


@pytest.mark.parametrize("sigma", [2.0 ** -16, 2.0 ** 16])
@pytest.mark.parametrize("weight", ["exp", "iv1", "iv2", "off"])
def test_tables_at_the_sigma_ends_are_finite_with_unit_centre(sigma, weight):
    t = O.weight_table(sigma, weight)
    assert t[0] == 2 ** 22 and t.max() == 2 ** 22
    # the float weights behind the table: finite, w(0) > 0 and normal
    s = np.float32(sigma) / np.float32(256.0) * np.float32(64)
    k = np.arange(len(t), dtype=np.float32)
    with np.errstate(over="raise", invalid="raise", divide="raise"):
        if weight == "exp":
            w = np.exp(-k * (np.float32(1.0) / ((np.float32(2) * s) * s)))
        elif weight == "iv1":
            w = np.float32(1.0) / (k + s)
        elif weight == "iv2":
            w = np.float32(1.0) / (k + s * s)
        else:
            w = np.ones(1, np.float32)
    assert np.all(np.isfinite(w)) and w[0] >= np.finfo(np.float32).tiny


def test_default_table_is_the_truncated_one():
    """exp at 25.5: the table is zero beyond d^2 = 1295, the prefix the tuned kernel keeps."""
    t = O.weight_table()
    assert len(t) == 11908 and t[1295] > 0 and not t[1296:].any()
    assert O.weight_table(2.0 ** 16, "iv2").min() > 0        # no truncation applies away from the default
