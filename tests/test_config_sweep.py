"""CPU: the all-pairs sweep's generator and oracle composition (tests/config_sweep.py): every allowed pair of levels
occurs, no configuration breaks a constraint, the list is the same on every call, and with every setting at its default
the composition is the oracle's pipeline (and the golden scene hashes)."""
import hashlib

import numpy as np
import pytest

import config_sweep as S
from oracle import oracle as O


@pytest.fixture(scope="module")
def sweep():
    return S.generate()


def levels(c):
    return {f: c[f] for f in S.NAMES}


def test_every_allowed_pair_occurs(sweep, capsys):
    configs, groups = sweep
    allowed = S.allowed_pairs()
    covered = set().union(*(S.pairs_of(levels(c)) for c in configs))
    with capsys.disabled():
        print(f"\nconfig sweep: {len(configs)} configurations on {len(groups)} contexts, "
              f"{len(covered & allowed)} of {len(allowed)} allowed pairs covered")
    assert covered == allowed, sorted(allowed - covered)[:10]
    # every factor's every level is in some allowed pair, so none is dead
    for f, lv in S.FACTORS.items():
        for v in lv:
            assert any((f, v) in p for p in allowed), (f, v)


def test_no_configuration_breaks_a_constraint(sweep):
    configs, groups = sweep
    for c in configs:
        for p in S.CONSTRAINTS:
            assert p(levels(c)), f"configuration {c['group']}.{c['step']} breaks {p.__name__}: {S.describe(c)}"
    # one context per creation group, in order, each reconfigured at least twice
    for gi, g in enumerate(groups):
        seq = [c for c in configs if c["group"] == gi]
        assert len(seq) >= S.MIN_STEPS and [c["step"] for c in seq] == list(range(len(seq)))
        assert all({f: c[f] for f in S.CREATION} == g for c in seq)
    assert [c["group"] for c in configs] == sorted(c["group"] for c in configs)


def test_constraints_judge_what_they_name():
    assert not S.valid({"post": "chain", "outputs": "none"})
    assert not S.valid({"post": "dcheck_only", "outputs": "runner_up"})
    assert S.valid({"post": "dcheck_only", "outputs": "costs"}) and S.valid({"post": "lr2", "outputs": "none"})
    assert not S.valid({"views": "left", "post": "lr2"}) and not S.valid({"views": "left", "post": "generic_wmf_lr1"})
    assert S.valid({"views": "left", "post": "chain"})
    assert not S.valid({"reproject": "post", "post": "off"}) and S.valid({"reproject": "selection", "post": "off"})
    for fmt in S.FORMATS:   # every shape but the narrow one gives the check columns to take part, at every D
        for shape in S.SHAPES:
            W, _, D, _ = S.geometry({"format": fmt, "shape": shape})
            assert (W > D) == (shape != "narrow"), (fmt, shape, W, D)
    assert S.geometry({"format": "u16_d300", "shape": "113x37"})[0] == 337   # (W - 1) a multiple of 112 at D = 300 too


def test_the_generator_is_deterministic(sweep):
    again = S.generate()
    assert again[0] == sweep[0] and again[1] == sweep[1]


def cones_crop(scenes, W, H):
    l8, r8, _, _ = scenes["Cones"]
    return tuple(np.ascontiguousarray(x[120:120 + H, 160:160 + W]) for x in (l8, r8))


def test_defaults_are_the_pipeline(scenes):
    W, H, D, _ = S.geometry(S.DEFAULT)
    src = cones_crop(scenes, W, H)
    fr = {"src": src, "maps": None, "src_size": (W, H)}
    l, r = O.u8_to_f32(src[0]), O.u8_to_f32(src[1])
    ref = O.pipeline(l, r, D, keep_volumes=True)
    got = S.expect(S.DEFAULT, fr)
    assert sorted(got) == [("selection", 0), ("selection", 1)]
    assert np.array_equal(got["selection", 0], ref["lDis"]) and np.array_equal(got["selection", 1], ref["rDis"])
    # every output on: the selection is the pipeline's still, and each output has its shape and type
    full = dict(S.DEFAULT, outputs="both", post="chain", reproject="post")
    got = S.expect(full, fr)
    assert np.array_equal(got["selection", 0], ref["lDis"]) and np.array_equal(got["selection", 1], ref["rDis"])
    for v, vol in ((0, ref["lVol"]), (1, ref["rVol"])):
        assert got["costs", v].shape == (3, H, W) and got["costs", v].dtype == np.uint32
        assert np.array_equal(got["costs", v][1], vol[got["selection", v], np.arange(H)[:, None], np.arange(W)].view(
            np.uint32))
        assert got["runner_up", v].shape == (2, H, W) and got["post", v].dtype == np.uint8
        assert got["valid", v].shape == (H, W) and got["points_post", v].shape == (H, W, 3)
    # 16-bit maps hold the same values
    got16 = S.expect(dict(S.DEFAULT, format="u16_d48"), fr)
    assert got16["selection", 0].dtype == np.uint16 and np.array_equal(got16["selection", 0], ref["lDis"])


def test_defaults_match_the_golden_scene(scenes, golden):
    """the whole Cones scene at the golden D = 64: the maps cv2's build of the reference gave"""
    l8, r8, _, _ = scenes["Cones"]
    H, W = l8.shape[:2]
    got = S.expect(S.DEFAULT, {"src": (l8, r8), "maps": None, "src_size": (W, H)}, D=golden["D"])
    g = golden["scenes"]["Cones"]
    for v, key in ((0, "lDis"), (1, "rDis")):
        assert hashlib.sha256(np.ascontiguousarray(got["selection", v]).tobytes()).hexdigest() == g[key]


def test_rectified_frames_are_the_remap():
    c = dict(S.DEFAULT, entry="rectify", shape="61x15", group=0, step=0)
    fr = S.frames(c, S.step_seed(c))
    W, H, _, _ = S.geometry(c)
    assert fr["src"][0].shape == (H + 2 * S.RECTIFY_MARGIN[1], W + 2 * S.RECTIFY_MARGIN[0], 3)
    l8, r8 = S.ingested(fr)
    assert l8.shape == (H, W, 3) and l8.dtype == np.uint8 and not np.array_equal(l8, r8)
