"""Seeded inputs for the Fast Guided Filter numerics tests (test_fgf_numerics.py on the CPU, test_gpu_fgf_numerics.py on
the device): costs whose fp64 box sums are not exact, non-finite and signed-zero costs, exact ties between slices, and a
guide pair with a near-black background.  Special voxels sit on the NN sample points of the low-resolution grid (the
only full-resolution pixels the low-resolution stages read), near the start of a 32 x 16 low-resolution tile row."""
import numpy as np

F32 = np.float32
COST_KINDS = ("wide12", "wide40", "outlier", "posinf", "neginf", "nan", "mixed", "ties")
SPECIAL = {"outlier": 1e30, "posinf": np.inf, "neginf": -np.inf, "nan": np.nan}


def sample_points(W, H, s):
    """-> (xs, ys): the full-resolution column / row that low-resolution column / row i samples (cv::resize INTER_NN)"""
    w2, h2 = W // s, H // s
    xs = np.minimum(np.floor(np.arange(w2) * (1.0 / (w2 / W))).astype(np.int64), W - 1)
    ys = np.minimum(np.floor(np.arange(h2) * (1.0 / (h2 / H))).astype(np.int64), H - 1)
    return xs, ys


def dark_pair(W, H, seed, shift=2):
    """float BGR pair in [0, 1]: a near-black background (1e-7 .. 1e-6) with textured O(1) rectangles; the right view
    is the left one shifted by `shift` columns"""
    rng = np.random.default_rng(seed)
    l = rng.uniform(1e-7, 1e-6, (H, W, 3)).astype(F32)
    for _ in range(max(2, W * H // 800)):
        h, w = int(rng.integers(1, max(2, H // 2) + 1)), int(rng.integers(1, max(2, W // 3) + 1))
        y0, x0 = int(rng.integers(0, H)), int(rng.integers(0, W))
        l[y0:y0 + h, x0:x0 + w] = rng.random((min(h, H - y0), min(w, W - x0), 3), dtype=F32)
    return l, np.ascontiguousarray(np.roll(l, -shift, axis=1))


def to_u8(img):
    """the pair as 8-bit images (the background becomes 0)"""
    return np.clip(np.rint(np.asarray(img, F32) * F32(255)), 0, 255).astype(np.uint8)


def costs(kind, D, W, H, s, seed):
    """one raw cost volume [D, H, W] of the given kind (D >= 4)"""
    rng = np.random.default_rng(seed)
    shape = (D, H, W)
    if kind in ("wide12", "wide40"):
        lo, hi = (-12, 3) if kind == "wide12" else (-40, 10)
        return (np.abs(rng.standard_normal(shape)) * np.exp(rng.uniform(lo, hi, shape))).astype(F32)
    if kind in SPECIAL:
        v = rng.random(shape, dtype=F32)
        xs, ys = sample_points(W, H, s)
        cols = [c for c in (1, 33) if c < len(xs)] or [0]
        rows = [min(2, len(ys) - 1), len(ys) // 2]
        for d in (1, D - 1):
            for c, y in zip(cols, rows):
                v[d, ys[y], xs[c]] = SPECIAL[kind]
        return v
    if kind == "mixed":
        v = rng.standard_normal(shape).astype(F32)
        v[rng.random(shape) < 0.1] = -0.0
        v[2] = -0.0
        return v
    if kind == "ties":
        v = (rng.random(shape, dtype=F32) + F32(1))
        v[1] = v[3] = rng.random((H, W), dtype=F32) * F32(0.5)
        v[2] = v[D - 1] = rng.random((H, W), dtype=F32) * F32(0.5)
        return v
    raise ValueError(kind)


# full-resolution W, H and rate s: low-resolution sizes of one column or row, at and around the 32 x 16 tile edges, and
# below half the box, where the reflections wrap more than once
GEOMETRY = [
    (4, 37, 4), (8, 8, 8), (1, 23, 1), (2, 3, 2),           # w2 = 1 (and h2 = 1)
    (57, 6, 4), (200, 15, 8),                               # h2 = 1
    (62, 30, 2), (64, 32, 2), (67, 35, 2),                  # low-res 31 x 15, 32 x 16, 33 x 17: the tile edges
    (128, 30, 2), (131, 34, 2), (260, 68, 4),               # 64 x 15, 65 x 17, 65 x 17
    (33, 17, 1), (65, 16, 1), (31, 15, 1),
    (3, 5, 1), (5, 7, 2), (12, 9, 4), (17, 9, 8),           # low-res sizes below K / 2: reflections wrap more than once
]


def differ(a, b):
    """mask of elements whose bits differ; two NaNs count as equal whatever their payloads"""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype != np.float32:
        return a != b
    na, nb = np.isnan(a), np.isnan(b)
    return (na != nb) | (~na & ~nb & (a.view(np.uint32) != b.view(np.uint32)))


def assert_same(a, b, what):
    """bit-for-bit equality (NaN at the same places); on failure the count and the first differing element"""
    assert a.shape == b.shape, f"{what}: shape {a.shape} vs {b.shape}"
    bad = np.argwhere(differ(a, b))
    if len(bad):
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {a.size} differ, first at {list(i)}: {a[i]!r} vs {b[i]!r}")
