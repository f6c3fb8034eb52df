"""CPU-only: the rectification restatement (rectify_oracle.py) against cv2's results pinned in golden_rectify.json, the
crop rule, and the argument checks of the Python interfaces that need no GPU."""
import hashlib
import json
import os

import numpy as np
import pytest

import rectify_cases
import rectify_oracle as RO
from primestereomatch_b200 import synth
from primestereomatch_b200.dispest import DispEst, rectify_args

CASES = rectify_cases.load()


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_equals_cv2(case):
    _, srcs, maps, digests = case
    for src, (xy, a), want in zip(srcs, maps, digests):
        if want is not None:
            assert sha(RO.remap(src, xy, a)) == want


def test_golden_covers_the_issue_cases():
    meta = json.load(open(os.path.join(rectify_cases.GOLDEN, "golden_rectify.json")))
    names = {c["name"] for c in meta["cases"]}
    for w, h in ((1344, 376), (640, 480)):
        for alpha in (0, 1):
            for kind in ("zero", "shift"):
                assert f"rig_{w}x{h}_a{alpha}_{kind}" in names
    z = np.load(os.path.join(rectify_cases.GOLDEN, "rectify_cases.npz"))
    assert any((z[k] > 1023).any() for k in z.files if k.startswith("raw") and k.endswith("_a"))
    assert os.path.getsize(os.path.join(rectify_cases.GOLDEN, "rectify_cases.npz")) < 1_200_000


def test_crop_then_remap_equals_remap_then_crop():
    meta = json.load(open(os.path.join(rectify_cases.GOLDEN, "golden_rectify.json")))
    z = np.load(os.path.join(rectify_cases.GOLDEN, "rectify_cases.npz"))
    n = 0
    for c in meta["cases"]:
        if c["kind"] != "rig" or not c["full_maps"]:
            continue
        for v in range(2):
            src = rectify_cases.frame(c["seed"] + v, *c["src"])
            xy, a = z[f"{c['name']}_{v}_xy"], z[f"{c['name']}_{v}_a"]
            box = c["box"]
            assert np.array_equal(RO.remap(src, RO.crop(xy, box), RO.crop(a, box)), RO.crop(RO.remap(src, xy, a), box))
            n += 1
    assert n == 8


def test_crop_box_is_the_reference_rule():
    assert RO.crop_box((17, 40, 1291, 298), (34, 40, 1289, 298)) == (34, 40, 1274, 298)
    assert RO.crop_box((0, 5, 10, 10), (3, 0, 10, 12)) == (3, 5, 7, 7)


def test_oracle_definition_by_hand():
    src = np.array([[[0], [100]], [[200], [255]]], np.uint8)
    xy = np.zeros((1, 1, 2), np.int16)
    for fx, fy in ((0, 0), (16, 0), (0, 16), (16, 16), (31, 31), (5, 27)):
        a = np.array([[fy * 32 + fx]], np.uint16)
        w = np.array([(32 - fx) * (32 - fy), fx * (32 - fy), (32 - fx) * fy, fx * fy]) * 32
        want = (int(w @ np.array([0, 100, 200, 255])) + 16384) >> 15
        assert RO.remap(src, xy, a)[0, 0, 0] == want
        assert RO.remap(src, xy, a | np.uint16(0xFC00))[0, 0, 0] == want   # bits above 10 are ignored
    # taps outside read 0: (-1, -1) with fx = fy = 16 sees only the (0, 0) sample at weight 1/4
    out = RO.remap(np.full((1, 1, 1), 255, np.uint8), np.array([[[-1, -1]]], np.int16), np.array([[16 * 32 + 16]], np.uint16))
    assert out[0, 0, 0] == (255 * 8192 + 16384) >> 15


def test_synthetic_rig_maps():
    xy, a = synth.rectify_maps(64, 40, 80, 50, view=1)
    assert xy.dtype == np.int16 and xy.shape == (40, 64, 2) and a.dtype == np.uint16 and a.shape == (40, 64)
    assert a.max() <= 1023
    assert (xy[..., 0] >= 0).all() and (xy[..., 0] < 80).all() and (xy[..., 1] >= 0).all() and (xy[..., 1] < 50).all()


def maps(w, h):
    return np.zeros((h, w, 2), np.int16), np.zeros((h, w), np.uint16)


def test_rectify_args_accepts_cropped_views_and_off():
    args, keep = rectify_args(None, None, None, 8, 4)
    assert args == (0, 0, None, 0, None, 0, None, 0, None, 0) and keep == ()
    xy, a = maps(20, 10)
    args, keep = rectify_args((xy[2:6, 3:11], a[2:6, 3:11]), maps(8, 4), (30, 12), 8, 4)
    assert args[:2] == (30, 12)
    assert args[3] == 20 * 4 and args[5] == 20 * 2   # a crop of the whole map keeps its row step
    assert args[7] == 8 * 4 and args[9] == 8 * 2
    # a column-strided view is made dense
    args, keep = rectify_args((xy[:4, :16:2], a[:4, :16:2]), maps(8, 4), (30, 12), 8, 4)
    assert keep[0].flags.c_contiguous and args[3] == 8 * 4


@pytest.mark.parametrize("bad, exc", [
    (dict(left=None), ValueError),
    (dict(src=None), ValueError),
    (dict(src=(0, 10)), ValueError),
    (dict(src=(32768, 10)), ValueError),
    (dict(src="big"), TypeError),
    (dict(left=(np.zeros((4, 8, 2), np.int32), np.zeros((4, 8), np.uint16))), ValueError),
    (dict(left=(np.zeros((4, 8, 2), np.int16), np.zeros((4, 8), np.int16))), ValueError),
    (dict(right=(np.zeros((4, 9, 2), np.int16), np.zeros((4, 9), np.uint16))), ValueError),
    (dict(right=(np.zeros((4, 8, 2), np.int16),)), TypeError),
])
def test_rectify_args_rejects(bad, exc):
    kw = dict(left=maps(8, 4), right=maps(8, 4), src=(30, 12))
    kw.update(bad)
    with pytest.raises(exc):
        rectify_args(kw["left"], kw["right"], kw["src"], 8, 4)


def test_dispest_checks_maps_before_the_device():
    img = np.zeros((4, 8, 3), np.uint8)
    de = DispEst(img, img, 16, ocl=False)
    with pytest.raises(ValueError):
        de.setRectify(maps(8, 5), maps(8, 4), (30, 12))
    with pytest.raises(RuntimeError):   # well-formed: it gets as far as the missing GPU context
        de.setRectify(maps(8, 4), maps(8, 4), (30, 12))
    assert de.src_size is None
