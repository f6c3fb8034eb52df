"""CPU-only: the YUV-to-BGR restatement (yuv_oracle.py) against cv2's results pinned in golden_yuv.json, the layout checks
of the Python interfaces (yuv_layout, setInputImagesYUV) and the new C-ABI symbols, none of which need a GPU."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

import rectify_cases
import rectify_oracle as RO
import yuv_oracle as YO
from primestereomatch_b200 import DispEst, capi
from primestereomatch_b200.dispest import yuv_format, yuv_shape

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
META = json.load(open(os.path.join(GOLDEN, "golden_yuv.json")))
CASES = {c["name"]: c for c in META["cases"]}
KEPT = np.load(os.path.join(GOLDEN, "yuv_cases.npz"))


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_every_triple_equals_cv2():
    assert sha(YO.all_triples_bgr()) == CASES["triples"]["sha256"]
    assert np.array_equal(YO.bgr(YO.all_triples(), "yuyv"), YO.all_triples_bgr())


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c["kind"] == "frame"])
def test_frames_equal_cv2(name):
    c = CASES[name]
    got = YO.bgr(YO.frame(c["seed"], c["format"], *c["size"]), c["format"])
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
        f = YO.frame(c["seed"], c["format"], *c["src"])
        assert sha(RO.remap(YO.bgr(f, c["format"]), xy, a)) == c["sha256"], c["name"]
        n += 1
    assert n == 28


def test_golden_covers_every_format_and_size():
    sizes = {tuple(c["size"]) for c in META["cases"] if c["kind"] == "frame"}
    assert sizes == {(2, 2), (64, 48), (130, 38), (1922, 6), (2688, 376)}
    for kind in ("frame", "rectify"):
        assert {c["format"] for c in META["cases"] if c["kind"] == kind} == set(YO.FORMATS)
    assert os.path.getsize(os.path.join(GOLDEN, "yuv_cases.npz")) < 300_000


def test_conversion_by_hand():
    # black and white of limited range, and the clamps
    assert YO.convert(16, 128, 128).tolist() == [0, 0, 0]
    assert YO.convert(235, 128, 128).tolist() == [255, 255, 255]
    assert YO.convert(0, 128, 128).tolist() == [0, 0, 0]            # Y below 16 counts as 16
    assert YO.convert(255, 255, 255).tolist()[2] == 255 and YO.convert(0, 0, 0).tolist()[0] == 0
    y, u, v = 100, 90, 200
    yy = (y - 16) * 1220542 + (1 << 19)
    assert YO.convert(y, u, v).tolist() == [max(0, min(255, (yy + 2116026 * (u - 128)) >> 20)),
                                            max(0, min(255, (yy - 852492 * (v - 128) - 409993 * (u - 128)) >> 20)),
                                            max(0, min(255, (yy + 1673527 * (v - 128)) >> 20))]


def test_layout_unpacking_by_hand():
    # a 4 x 2 frame: luma 0..7, chroma pairs (U, V) = (100, 200), (110, 210)
    Y = np.arange(8, dtype=np.uint8).reshape(2, 4)
    nv12 = np.vstack([Y, [[100, 200, 110, 210]]]).astype(np.uint8)
    nv21 = np.vstack([Y, [[200, 100, 210, 110]]]).astype(np.uint8)
    i420 = np.vstack([Y, [[100, 110, 200, 210]]]).astype(np.uint8)
    yv12 = np.vstack([Y, [[200, 210, 100, 110]]]).astype(np.uint8)
    for f, fmt in ((nv12, "nv12"), (nv21, "nv21"), (i420, "i420"), (yv12, "yv12")):
        y, u, v = YO.planes(f, fmt)
        assert np.array_equal(y, Y), fmt
        assert u.tolist() == [[100, 100, 110, 110]] * 2 and v.tolist() == [[200, 200, 210, 210]] * 2, fmt
    yuyv = np.array([[[0, 100], [1, 200], [2, 110], [3, 210]]], np.uint8)
    uyvy = np.array([[[100, 0], [200, 1], [110, 2], [210, 3]]], np.uint8)
    yvyu = np.array([[[0, 200], [1, 100], [2, 210], [3, 110]]], np.uint8)
    for f, fmt in ((yuyv, "yuyv"), (uyvy, "uyvy"), (yvyu, "yvyu")):
        y, u, v = YO.planes(f, fmt)
        assert y.tolist() == [[0, 1, 2, 3]] and u.tolist() == [[100, 100, 110, 110]] and v.tolist() == [[200, 200, 210, 210]]


# -- the Python interfaces ----------------------------------------------------------------------------------------------
def test_yuv_format_and_shape():
    assert yuv_format("nv12") == (capi.PSM_YUV_NV12, True) and yuv_format("YUYV") == (capi.PSM_YUV_YUYV, False)
    assert yuv_shape("i420", 8, 6) == (9, 8) and yuv_shape("uyvy", 8, 5) == (5, 8, 2)
    for bad in ("bgr", "p010", 1, None):
        with pytest.raises(ValueError):
            yuv_format(bad)
    with pytest.raises(ValueError):
        yuv_shape("nv12", 7, 6)
    with pytest.raises(ValueError):
        yuv_shape("nv12", 8, 5)
    with pytest.raises(ValueError):
        yuv_shape("yuyv", 7, 5)


def test_dispest_checks_yuv_frames_before_the_device():
    img = np.zeros((4, 8, 3), np.uint8)
    de = DispEst(img, img, 16, ocl=False)
    with pytest.raises(ValueError):
        de.setInputImagesYUV(np.zeros((6, 8), np.uint8), np.zeros((6, 8), np.uint8), "p010")
    with pytest.raises(TypeError):
        de.setInputImagesYUV(np.zeros((6, 8), np.float32), np.zeros((6, 8), np.float32), "nv12")
    de.setInputImagesYUV(np.zeros((6, 8), np.uint8), np.zeros((6, 8), np.uint8), "nv12")
    with pytest.raises(RuntimeError):   # well-formed: it gets as far as the missing GPU context
        de.CostConst_GPU()


@pytest.fixture(scope="module")
def T():
    return pytest.importorskip("torch")


def test_yuv_layout_of_each_format(T):
    from primestereomatch_b200.torch_stereo import yuv_layout
    H, W = 6, 8
    t = T.zeros(H * 3 // 2, W, dtype=T.uint8)
    p = t.data_ptr()
    assert yuv_layout(t, H, W, "nv12") == (capi.PSM_YUV_420, [(p, p + H * W, p + H * W + 1)], W, 1, W, 2, False)
    assert yuv_layout(t, H, W, "nv21")[1] == [(p, p + H * W + 1, p + H * W)]
    q = (W // 2) * (H // 2)
    assert yuv_layout(t, H, W, "i420") == (capi.PSM_YUV_420, [(p, p + H * W, p + H * W + q)], W, 1, W // 2, 1, False)
    assert yuv_layout(t, H, W, "yv12")[1] == [(p, p + H * W + q, p + H * W)]
    t2 = T.zeros(H, W, 2, dtype=T.uint8)
    p = t2.data_ptr()
    assert yuv_layout(t2, H, W, "yuyv") == (capi.PSM_YUV_422, [(p, p + 1, p + 3)], 2 * W, 2, 2 * W, 4, False)
    assert yuv_layout(t2, H, W, "uyvy")[1] == [(p + 1, p, p + 2)]
    assert yuv_layout(t2, H, W, "yvyu")[1] == [(p, p + 3, p + 1)]


def test_yuv_layout_of_side_by_side_halves_and_batches(T):
    from primestereomatch_b200.torch_stereo import yuv_layout
    H, W = 6, 8
    sbs = T.zeros(H * 3 // 2, 2 * W, dtype=T.uint8)   # one NV12 frame holding both views side by side
    p = sbs.data_ptr()
    assert yuv_layout(sbs[:, W:], H, W, "nv12") == (capi.PSM_YUV_420, [(p + W, p + H * 2 * W + W, p + H * 2 * W + W + 1)],
                                                     2 * W, 1, 2 * W, 2, False)
    sbs2 = T.zeros(H, 2 * W, 2, dtype=T.uint8)
    p = sbs2.data_ptr()
    assert yuv_layout(sbs2[:, W:], H, W, "yuyv") == (capi.PSM_YUV_422, [(p + 2 * W, p + 2 * W + 1, p + 2 * W + 3)],
                                                     4 * W, 2, 4 * W, 4, False)
    batch = T.zeros(3, H, W, 2, dtype=T.uint8)
    p = batch.data_ptr()
    sampling, frames, *_, batched = yuv_layout(batch, H, W, "uyvy")
    assert batched and frames == [(p + b * H * W * 2 + 1, p + b * H * W * 2, p + b * H * W * 2 + 2) for b in range(3)]


@pytest.mark.parametrize("make, fmt, exc", [
    (lambda T: T.zeros(9, 8, dtype=T.float32), "nv12", TypeError),        # not uint8
    (lambda T: T.zeros(6, 8, dtype=T.uint8), "nv12", ValueError),         # the 4:2:2 height for a 4:2:0 format
    (lambda T: T.zeros(9, 8, 2, dtype=T.uint8), "nv12", ValueError),
    (lambda T: T.zeros(6, 8, dtype=T.uint8), "yuyv", ValueError),
    (lambda T: T.zeros(9, 8, dtype=T.uint8), "bgr", ValueError),          # unknown format
    (lambda T: T.zeros(9, 16, dtype=T.uint8)[:, 8:], "i420", ValueError),  # planar chroma: only a contiguous frame
    (lambda T: T.zeros(9, 16, dtype=T.uint8)[:, ::2], "yv12", ValueError),
    (lambda T: T.zeros(9, 1, dtype=T.uint8).expand(9, 8), "nv12", ValueError),   # column stride 0
    (lambda T: T.zeros(8, 9, dtype=T.uint8).t(), "nv12", ValueError),             # rows overlap
    (lambda T: T.zeros(0, 9, 8, dtype=T.uint8), "nv12", ValueError),              # empty batch
    (lambda T: [[0]], "nv12", TypeError),
])
def test_yuv_layout_rejects(T, make, fmt, exc):
    from primestereomatch_b200.torch_stereo import yuv_layout
    with pytest.raises(exc):
        yuv_layout(make(T), 6, 8, fmt)


def test_yuv_layout_rejects_odd_sizes(T):
    from primestereomatch_b200.torch_stereo import yuv_layout
    with pytest.raises(ValueError):
        yuv_layout(T.zeros(6, 7, 2, dtype=T.uint8), 6, 7, "yuyv")
    with pytest.raises(ValueError):
        yuv_layout(T.zeros(7, 8, dtype=T.uint8), 5, 8, "nv12")


# -- the C-ABI ---------------------------------------------------------------------------------------------------------
def test_new_symbols_are_declared_bound_and_exported():
    L = capi.lib()
    for name in ("psm_set_images_device_yuv", "psm_set_images_yuv", "psm_set_images_yuv_async"):
        assert name in capi.SYMBOLS
        assert getattr(L, name).restype is C.c_int and getattr(L, name).argtypes
    assert (capi.PSM_YUV_420, capi.PSM_YUV_422) == (1, 2)
    assert [capi.YUV_FORMATS[f] for f in YO.FORMATS] == list(range(1, 8))
    assert set(capi.YUV_420) == set(YO.FORMATS_420)


def test_null_context_is_einval():
    L = capi.lib()
    buf = np.zeros(64, np.uint8)
    p = buf.ctypes.data_as(C.c_void_p)
    ptrs = (C.c_void_p * 3)(p, p, p)
    assert L.psm_set_images_yuv(None, capi.PSM_YUV_NV12, p, 8, p, 8) == capi.PSM_EINVAL
    assert L.psm_set_images_yuv_async(None, capi.PSM_YUV_NV12, p, 8, p, 8) == capi.PSM_EINVAL
    assert L.psm_set_images_device_yuv(None, capi.PSM_YUV_420, ptrs, ptrs, 8, 1, 8, 2) == capi.PSM_EINVAL
    assert b"null context" in L.psm_last_error(None)


@pytest.mark.parametrize("fmt", YO.FORMATS)
def test_pack_inverts_planes(fmt):
    rng = np.random.default_rng(5)
    f = YO.frame(11, fmt, 10, 6)
    assert np.array_equal(YO.pack(*(p[::2 if fmt in YO.FORMATS_420 else 1, ::2] if k else p
                                    for k, p in enumerate(YO.planes(f, fmt))), fmt), f)
    img = rng.integers(0, 256, (6, 10, 3), dtype=np.uint8)
    assert YO.from_bgr(img, fmt).shape == YO.shape(fmt, 10, 6)
