"""CPU-only: the demosaicing restatement (bayer_oracle.py) against cv2's results pinned in golden_bayer.json, its two forms
against each other, the layout checks of the Python interfaces (bayer_layout, setInputImagesBayer) and the new C-ABI
symbols, none of which need a GPU."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

import bayer_oracle as BO
import rectify_cases
import rectify_oracle as RO
from primestereomatch_b200 import DispEst, capi
from primestereomatch_b200.dispest import bayer_kind

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
META = json.load(open(os.path.join(GOLDEN, "golden_bayer.json")))
CASES = {c["name"]: c for c in META["cases"]}
KEPT = np.load(os.path.join(GOLDEN, "bayer_cases.npz"))
CODES = [(p, m) for m in BO.METHODS for p in BO.PATTERNS]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def case_frame(c):
    """the raw frame of a golden case, regenerated from its seed"""
    if c["kind"] == "frame":
        return BO.frame(c["seed"], *c["size"])
    if c["kind"] == "side_by_side":
        w, h = c["size"]
        sbs = BO.frame(c["seed"], w, h)
        return np.ascontiguousarray(sbs[:, :w // 2] if c["half"] == "left" else sbs[:, w // 2:])
    f = BO.frame(c["seed"], 64, 48, 3 if c["values"] == "low" else 2)
    return f if c["values"] == "low" else f * np.uint8(255)


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c["kind"] in ("frame", "side_by_side", "ties")])
def test_frames_equal_cv2(name):
    c = CASES[name]
    got = BO.bgr(case_frame(c), c["pattern"], c["method"])
    assert sha(got) == c["sha256"]
    if name in KEPT.files:
        assert np.array_equal(got, KEPT[name])


def test_rectified_frames_equal_cv2():
    rigs = {name: maps for name, _, maps, _ in rectify_cases.load()}
    n = 0
    for c in META["cases"]:
        if c["kind"] != "rectify":
            continue
        xy, a = rigs[c["rig"]][0]
        f = BO.frame(c["seed"], *c["src"])
        assert sha(RO.remap(BO.bgr(f, c["pattern"], c["method"]), xy, a)) == c["sha256"], c["name"]
        n += 1
    assert n == 28


def test_golden_covers_every_code_and_size():
    for kind in ("frame", "side_by_side", "rectify"):
        assert {(c["pattern"], c["method"]) for c in META["cases"] if c["kind"] == kind} == set(CODES), kind
    sizes = {tuple(c["size"]) for c in META["cases"] if c["kind"] == "frame"}
    assert sizes == {(1, 1), (2, 2), (2, 9), (9, 2), (3, 3), (64, 48), (130, 38), (1922, 6)}
    assert {(c["values"], c["pattern"], c["method"]) for c in META["cases"] if c["kind"] == "ties"} == \
        {(v, p, m) for v in ("low", "binary") for p, m in CODES}
    assert os.path.getsize(os.path.join(GOLDEN, "bayer_cases.npz")) < 300_000


@pytest.mark.parametrize("pattern, method", CODES)
@pytest.mark.parametrize("size, high", [((1, 1), 256), ((2, 9), 256), ((9, 2), 256), ((3, 3), 256), ((4, 3), 256),
                                        ((7, 5), 256), ((33, 17), 256), ((20, 12), 3), ((20, 12), 2)])
def test_clamp_form_equals_loop(pattern, method, size, high):
    f = BO.frame(100 * size[0] + size[1] + high, *size, high=high)
    if high == 2:
        f = f * np.uint8(255)
    assert np.array_equal(BO.bgr(f, pattern, method), BO.bgr_loop(f, pattern, method))


def test_definition_by_hand():
    # a 4 x 4 RGGB frame: interior pixels (1, 1) (B site) and (2, 1) (G site on a B row), (1, 2) (G on an R row),
    # (2, 2) (R site)
    raw = np.array([[10, 20, 30, 40],
                    [50, 60, 70, 80],
                    [90, 100, 110, 120],
                    [130, 140, 150, 160]], np.uint8)
    out = BO.bgr(raw, "rggb")
    # B site (1, 1): B = 60, G = (20 + 50 + 70 + 100 + 2) >> 2, R = (10 + 30 + 90 + 110 + 2) >> 2
    assert out[1, 1].tolist() == [60, (20 + 50 + 70 + 100 + 2) >> 2, (10 + 30 + 90 + 110 + 2) >> 2]
    # G site (2, 1) on a B row: B horizontal (60, 80), R vertical (30, 110)
    assert out[1, 2].tolist() == [(60 + 80 + 1) >> 1, 70, (30 + 110 + 1) >> 1]
    # G site (1, 2) on an R row: R horizontal (90, 110), B vertical (60, 140)
    assert out[2, 1].tolist() == [(60 + 140 + 1) >> 1, 100, (90 + 110 + 1) >> 1]
    # borders copy the clamped interior pixel
    assert out[0, 0].tolist() == out[1, 1].tolist() and out[3, 3].tolist() == out[2, 2].tolist()
    # edge-aware at the R site (2, 2): |100 - 120| = 20 <= |70 - 150| = 80, so G is the horizontal pair's
    ea = BO.bgr(raw, "rggb", "ea")
    assert ea[2, 2, 1] == (100 + 120 + 1) >> 1
    # a tie goes horizontal
    tie = np.zeros((3, 3), np.uint8)
    tie[1, 0], tie[1, 2], tie[0, 1], tie[2, 1] = 0, 2, 255, 253   # |0 - 2| == |255 - 253|
    assert BO.bgr(tie, "bggr", "ea")[1, 1, 1] == 1   # (1, 1) is BGGR's R site
    assert BO.bgr(np.zeros((2, 8), np.uint8) + 7, "rggb").max() == 0


def test_from_bgr_keeps_each_sites_colour():
    img = np.random.default_rng(1).integers(0, 256, (6, 8, 3), dtype=np.uint8)
    for pattern in BO.PATTERNS:
        raw = BO.from_bgr(img, pattern)
        rx, ry = BO.red_site(pattern)
        assert raw[ry, rx] == img[ry, rx, 2] and raw[1 - ry, 1 - rx] == img[1 - ry, 1 - rx, 0]
        assert raw[ry, 1 - rx] == img[ry, 1 - rx, 1]


# -- the Python interfaces ----------------------------------------------------------------------------------------------
def test_bayer_kind():
    assert bayer_kind("rggb") == (capi.PSM_BAYER_RGGB, capi.PSM_DEMOSAIC_BILINEAR)
    assert bayer_kind("GBRG", "ea") == (capi.PSM_BAYER_GBRG, capi.PSM_DEMOSAIC_EA)
    for bad in ("bg", "rgb", 1, None):
        with pytest.raises(ValueError):
            bayer_kind(bad)
    for bad in ("vng", "", None):
        with pytest.raises(ValueError):
            bayer_kind("rggb", bad)


def test_dispest_checks_bayer_frames_before_the_device():
    img = np.zeros((4, 8, 3), np.uint8)
    de = DispEst(img, img, 16, ocl=False)
    with pytest.raises(ValueError):
        de.setInputImagesBayer(np.zeros((4, 8), np.uint8), np.zeros((4, 8), np.uint8), "bg")
    with pytest.raises(ValueError):
        de.setInputImagesBayer(np.zeros((4, 8), np.uint8), np.zeros((4, 8), np.uint8), "rggb", "vng")
    with pytest.raises(TypeError):
        de.setInputImagesBayer(np.zeros((4, 8), np.uint16), np.zeros((4, 8), np.uint16), "rggb")
    de.setInputImagesBayer(np.zeros((4, 8), np.uint8), np.zeros((4, 8), np.uint8), "rggb", "ea")
    with pytest.raises(RuntimeError):   # well-formed: it gets as far as the missing GPU context
        de.CostConst_GPU()


@pytest.fixture(scope="module")
def T():
    return pytest.importorskip("torch")


def test_bayer_layout_of_frames_halves_and_batches(T):
    from primestereomatch_b200.torch_stereo import bayer_layout
    H, W = 6, 8
    t = T.zeros(H, W, dtype=T.uint8)
    p = t.data_ptr()
    assert bayer_layout(t, H, W, "rggb") == (capi.PSM_BAYER_RGGB, capi.PSM_DEMOSAIC_BILINEAR, [p], W, 1, False)
    assert bayer_layout(t, H, W, "grbg", "ea")[:2] == (capi.PSM_BAYER_GRBG, capi.PSM_DEMOSAIC_EA)
    sbs = T.zeros(H, 2 * W, dtype=T.uint8)   # one raw frame holding both views side by side
    p = sbs.data_ptr()
    assert bayer_layout(sbs[:, :W], H, W, "bggr") == (capi.PSM_BAYER_BGGR, 1, [p], 2 * W, 1, False)
    assert bayer_layout(sbs[:, W:], H, W, "bggr") == (capi.PSM_BAYER_BGGR, 1, [p + W], 2 * W, 1, False)
    every_other = T.zeros(H, 2 * W, dtype=T.uint8)[:, ::2]   # a column step of 2
    assert bayer_layout(every_other, H, W, "rggb")[3:5] == (2 * W, 2)
    batch = T.zeros(3, H, W, dtype=T.uint8)
    p = batch.data_ptr()
    *_, frames, row, col, batched = bayer_layout(batch, H, W, "gbrg")
    assert batched and frames == [p + b * H * W for b in range(3)] and (row, col) == (W, 1)


@pytest.mark.parametrize("make, pattern, method, exc", [
    (lambda T: T.zeros(6, 8, dtype=T.float32), "rggb", "bilinear", TypeError),     # not uint8
    (lambda T: T.zeros(6, 8, dtype=T.int16), "rggb", "bilinear", TypeError),
    (lambda T: T.zeros(6, 8, 3, dtype=T.uint8), "rggb", "bilinear", ValueError),   # a BGR frame
    (lambda T: T.zeros(6, 9, dtype=T.uint8), "rggb", "bilinear", ValueError),      # another size
    (lambda T: T.zeros(8, dtype=T.uint8), "rggb", "bilinear", ValueError),
    (lambda T: T.zeros(6, 8, dtype=T.uint8), "bg", "bilinear", ValueError),        # unknown pattern
    (lambda T: T.zeros(6, 8, dtype=T.uint8), "rggb", "vng", ValueError),           # unknown method
    (lambda T: T.zeros(6, 1, dtype=T.uint8).expand(6, 8), "rggb", "bilinear", ValueError),   # column stride 0
    (lambda T: T.zeros(8, 6, dtype=T.uint8).t(), "rggb", "bilinear", ValueError),             # rows overlap
    (lambda T: T.zeros(0, 6, 8, dtype=T.uint8), "rggb", "bilinear", ValueError),              # empty batch
    (lambda T: [[0]], "rggb", "bilinear", TypeError),
])
def test_bayer_layout_rejects(T, make, pattern, method, exc):
    from primestereomatch_b200.torch_stereo import bayer_layout
    with pytest.raises(exc):
        bayer_layout(make(T), 6, 8, pattern, method)


def test_match_checks_bayer_frames_before_the_device(T):
    from primestereomatch_b200.torch_stereo import TorchStereo
    ts = TorchStereo.__new__(TorchStereo)   # the checks need the geometry and device alone, not a context
    ts.width, ts.height, ts.device = 8, 6, T.device("cuda", 0)
    ok = T.zeros(6, 8, dtype=T.uint8)
    with pytest.raises(ValueError, match="CUDA tensors"):
        ts._layout(ok, ok, "bgr", bayer="rggb")
    with pytest.raises(ValueError, match="same shape and strides"):
        ts._layout(ok, T.zeros(6, 10, dtype=T.uint8)[:, :8], "bgr", bayer="rggb")
    with pytest.raises(ValueError, match="one or the other"):
        ts._layout(ok, ok, "bgr", yuv="nv12", bayer="rggb")


# -- the C-ABI ---------------------------------------------------------------------------------------------------------
def test_new_symbols_are_declared_bound_and_exported():
    L = capi.lib()
    for name in ("psm_set_images_device_bayer", "psm_set_images_bayer", "psm_set_images_bayer_async"):
        assert name in capi.SYMBOLS
        assert getattr(L, name).restype is C.c_int and getattr(L, name).argtypes
    header = open(os.path.join(os.path.dirname(capi.__file__), "..", "include", "prime_stereo_b200.h")).read()
    for name in ("PSM_BAYER_RGGB = 1", "PSM_BAYER_BGGR = 2", "PSM_BAYER_GRBG = 3", "PSM_BAYER_GBRG = 4",
                 "PSM_DEMOSAIC_BILINEAR = 1", "PSM_DEMOSAIC_EA = 2"):
        assert name in header
    assert [capi.BAYER_PATTERNS[p] for p in BO.PATTERNS] == [1, 2, 3, 4]
    assert [capi.DEMOSAIC_METHODS[m] for m in BO.METHODS] == [1, 2]


def test_null_context_is_einval():
    L = capi.lib()
    buf = np.zeros(64, np.uint8)
    p = buf.ctypes.data_as(C.c_void_p)
    assert L.psm_set_images_bayer(None, capi.PSM_BAYER_RGGB, 1, p, 8, p, 8) == capi.PSM_EINVAL
    assert L.psm_set_images_bayer_async(None, capi.PSM_BAYER_RGGB, 1, p, 8, p, 8) == capi.PSM_EINVAL
    assert L.psm_set_images_device_bayer(None, capi.PSM_BAYER_RGGB, 1, p, p, 8, 1) == capi.PSM_EINVAL
    assert b"null context" in L.psm_last_error(None)
