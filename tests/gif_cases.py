"""Seeded inputs for the guided-filter numerics tests (test_gif_numerics.py on the CPU, test_gpu_gif_numerics.py on the
device): non-finite costs, costs of 2^63 and more, a band of large costs above small ones, costs over wide ranges, mixed
signs with -0.0, exact ties between slices, and guide images outside the u8 domain (a near-black float background, NaN
and inf pixels).  Special voxels sit on the seams of the streaming filter's decomposition (psm_cvf_plan at 132 SMs, with
and without a forced segment height): the first row of a segment and the row before it, the strip seams every 112
columns, the packed remainder columns, the first and last rows and columns, and the warm-up rows at the top."""
import numpy as np

from fgf_cases import assert_same, dark_pair, differ, to_u8  # noqa: F401  (shared helpers)

F32 = np.float32
W, H = 240, 136            # two full strips and a 16-column packed remainder; several row segments
SMS = 132                  # H100 SXM
FORCED_ROWS = 24           # option 101: rows per segment
EXACT_KINDS = ("posinf", "neginf", "nan", "outlier", "mixed", "ties")   # the device must equal the oracle bit for bit
INEXACT_KINDS = ("band", "wide40")                                       # finite, fp64 sums not exact: a derived bound
COST_KINDS = EXACT_KINDS + INEXACT_KINDS
SPECIAL = {"outlier": 1e30, "posinf": np.inf, "neginf": -np.inf, "nan": np.nan}


def plan_segments(H, target):
    """the row segmentation of psm_capi.cu (plan_segments) -> (nseg, seg_rows)"""
    n = max(1, H // target)
    for n in range(n, 1, -1):
        rows = ((H + n - 1) // n + 7) & ~7
        if rows >= 16 and H - (n - 1) * rows >= 8:
            return n, rows
    return 1, (H + 7) & ~7


def seams(W=W, H=H, D=5):
    """-> (rows, cols): the rows and columns where the decomposition changes hands"""
    from primestereomatch_b200 import capi
    plan = capi.cvf_plan(W, H, D, SMS)
    rows = {0, 1, 2, 3, 4, H - 1, H - 2}
    for nseg, seg in ((plan["nseg"], plan["seg_rows"]), plan_segments(H, FORCED_ROWS)):
        for k in range(1, nseg):
            rows |= {k * seg - 1, k * seg}
    cols = {0, 1, W - 1, W - 2}
    for s in range(1, W // 112 + 1):
        if s * 112 < W:
            cols |= {s * 112 - 1, s * 112}
    if plan["pack_gl"]:
        cols |= {plan["pack_x0"], plan["pack_x0"] + 5}
    return sorted(r for r in rows if 0 <= r < H), sorted(c for c in cols if 0 <= c < W)


def costs(kind, D, seed, W=W, H=H):
    """one raw cost volume [D, H, W] of the given kind (D >= 4)"""
    rng = np.random.default_rng(seed)
    shape = (D, H, W)
    if kind == "wide40":
        return (np.abs(rng.standard_normal(shape)) * np.exp(rng.uniform(-40, 10, shape))).astype(F32)
    if kind == "band":
        v = (rng.random(shape) * 2e-3).astype(F32)
        v[:, 10:14] = F32(1e15) * (F32(1) + rng.random((D, 4, W), dtype=F32))
        return v
    if kind in SPECIAL:
        v = rng.random(shape, dtype=F32)
        rows, cols = seams(W, H, D)
        for i, d in enumerate((1, D - 1)):
            # a few seam voxels per slice, different ones in the two slices
            for j, (y, x) in enumerate(zip(rows[i::2], cols[(i + 1) % 2::2])):
                if j < 4:
                    v[d, y, x] = SPECIAL[kind]
        return v
    if kind == "mixed":
        v = rng.standard_normal(shape).astype(F32)
        v[rng.random(shape) < 0.1] = -0.0
        v[2] = -0.0
        return v
    if kind == "ties":
        v = rng.random(shape, dtype=F32) + F32(1)
        v[1] = v[3] = rng.random((H, W), dtype=F32) * F32(0.5)
        v[2] = v[D - 1] = rng.random((H, W), dtype=F32) * F32(0.5)
        return v
    raise ValueError(kind)


def nan_pair(W=W, H=H, seed=21, shift=2):
    """a float pair in [0, 1] with a few NaN and inf pixels on the seams"""
    rng = np.random.default_rng(seed)
    l = rng.random((H, W, 3), dtype=F32)
    rows, cols = seams(W, H)
    l[rows[3], cols[2], 0] = np.nan
    l[rows[-2], cols[-3], 1] = np.inf
    l[rows[5], cols[4], 2] = np.nan
    return l, np.ascontiguousarray(np.roll(l, -shift, axis=1))


IMAGE_KINDS = ("dark_f32", "dark_u8", "nan_f32")


def images(kind):
    """-> (left, right) as the device takes them (float or u8), and the float pair the oracle takes"""
    if kind == "nan_f32":
        l, r = nan_pair()
        return (l, r), (l, r)
    l, r = dark_pair(W, H, seed=11)
    if kind == "dark_u8":
        from oracle import oracle as O
        l8, r8 = to_u8(l), to_u8(r)
        return (l8, r8), (O.u8_to_f32(l8), O.u8_to_f32(r8))
    return (l, r), (l, r)


# ---- how far two summation orders can drift apart --------------------------------------------------------------------
_U = 2.0 ** -53     # fp64 unit roundoff
_F = 2.0 ** -24     # fp32 unit roundoff


def _sum_error(x, K=8):
    """Per pixel: the largest rounding error that the fp64 box sum of the plane x (K x K, reflected, anchor K/2) can carry
    in either order.  OpenCV (orc_box): one running sum per row (2 roundings per step, W + K steps) whose magnitude is at
    most the largest K-wide row window of |x| it has passed (columns <= x), then one running sum per column (2 (H + K)
    roundings) of magnitude at most the largest box of |x| it has passed (centres <= y).  The tuned kernels: running column
    sums of single columns within a row segment (the 8 columns x - 4 .. x + 3, each at most such a box) and 8-wide row sums
    of those.  The error is the sum of the two."""
    from scipy.ndimage import maximum_filter1d
    a = np.abs(np.asarray(x, np.float64))
    h, w = a.shape
    k0 = K // 2

    def window_sums(t, axis):
        """sums over the K reflected taps -k0 .. K-1-k0 along an axis (numpy's "reflect" is BORDER_REFLECT_101)"""
        pad = np.pad(t, [(k0, K - 1 - k0) if ax == axis else (0, 0) for ax in range(2)], mode="reflect")
        return sum(np.take(pad, np.arange(t.shape[axis]) + i, axis=axis) for i in range(K))

    rows = window_sums(a, 1)                                                                   # row windows of |x|
    boxes = window_sums(rows, 0)                                                               # box windows of |x|
    row_err = 2 * (w + K) * _U * np.maximum.accumulate(rows, axis=1)
    col_m = maximum_filter1d(np.maximum.accumulate(boxes, axis=0), size=K + 1, axis=1, mode="nearest")
    return window_sums(row_err, 0) + (K + 1) * 2 * (h + K) * _U * col_m + 2 * K * _U * boxes, boxes


def carried_error_bound(img, p, K=8, eps=1e-4):
    """Per voxel: the largest |q_a - q_b| between two evaluations of GuidedFilter_cv (K x K box, eps) of the slice p that
    add the same fp64 values in different orders (OpenCV's running sums against the tuned kernels' segment / strip sums).

    A running sum keeps the rounding of every operation, each at most U = 2^-53 times the magnitude of its result, and
    that magnitude is at most the window sum of |x| of some window the sum has passed through (_sum_error).  So a box mean
    of a plane x differs by at most that carried error / K^2, plus one float rounding.  The difference is carried through cov, a, b (CVF.cpp:92-155) with this voxel's own mean_I, adjugate and
    1/det, through the second box (whose inputs a, b now differ as well) and q = box(b) + sum_c box(a_c) I_c; every float
    operation on the way adds at most 2^-24 of the magnitudes involved.  Non-finite voxels of the reference get inf."""
    from oracle import oracle as O
    img = np.asarray(img, np.float32)
    p = np.asarray(p, np.float32)
    with np.errstate(all="ignore"):
        rgb, mean, var = O.cvf_preprocess(img, window=K)
        q, a, b = O.guided_filter(rgb, mean, var, p, want_ab=True, window=K, eps=eps)
        f64 = lambda t: np.asarray(t, np.float64)
        I, mI, v = f64(rgb), f64(mean), f64(var)
        a, b, q = f64(a), f64(b), f64(q)

        def mean_err(x, dx=None):
            """|box mean of x computed two ways| where the inputs themselves may differ by dx"""
            m = np.abs(f64(O.box(np.asarray(x, np.float32), K)))
            xa = np.abs(f64(x)) if dx is None else np.abs(f64(x)) + dx
            e = _sum_error(xa, K)[0] / (K * K)
            if dx is not None:
                e = e + _sum_error(dx, K)[1] / (K * K)
            return e + 2 * _F * (m + e), m

        ep, mp = mean_err(p)
        eIp, mIp = zip(*(mean_err(f64(rgb[c]) * f64(p)) for c in range(3)))
        e_ = float(eps)
        a11, a22, a33 = v[0] + e_, v[3] + e_, v[5] + e_
        a12, a13, a23 = v[1], v[2], v[4]
        M = np.array([[a33 * a22 - a23 * a23, a13 * a23 - a33 * a12, a12 * a23 - a22 * a13],
                      [a13 * a23 - a33 * a12, a33 * a11 - a13 * a13, a13 * a12 - a23 * a11],
                      [a12 * a23 - a22 * a13, a13 * a12 - a23 * a11, a22 * a11 - a12 * a12]])
        idet = np.abs(1.0 / (a11 * M[0, 0] + a12 * M[1, 0] + a13 * M[2, 0]))
        M = np.abs(M) * (1 + 8 * _F) + 8 * _F * np.abs(M).max(axis=(0, 1))   # the float adjugate is within this of the real one
        cov = [np.abs(mIp[j]) + np.abs(mI[j]) * mp for j in range(3)]
        dcov = [eIp[j] + np.abs(mI[j]) * ep + 4 * _F * cov[j] for j in range(3)]
        da = [idet * (1 + 8 * _F) * sum(M[j, c] * dcov[j] for j in range(3))
              + 12 * _F * idet * sum(M[j, c] * cov[j] for j in range(3)) for c in range(3)]
        db = ep + sum(da[c] * np.abs(mI[c]) for c in range(3)) + 12 * _F * (mp + sum(np.abs(a[c] * mI[c]) for c in range(3)))
        emb, mb = mean_err(b, db)
        ema = [mean_err(a[c], da[c]) for c in range(3)]
        dq = emb + sum(ema[c][0] * np.abs(I[c]) for c in range(3)) \
            + 14 * _F * (mb + sum(ema[c][1] * np.abs(I[c]) for c in range(3)))
        bound = dq * 1.01 + 2.0 ** -140
    return np.where(np.isfinite(q) & np.isfinite(bound), bound, np.inf)


def beyond_bound(dev, ref, bound):
    """mask of voxels where dev and ref differ by more than the bound (NaN at different places counts as beyond)"""
    dev, ref = np.asarray(dev, np.float64), np.asarray(ref, np.float64)
    nd, nr = np.isnan(dev), np.isnan(ref)
    with np.errstate(invalid="ignore"):
        far = np.abs(dev - ref) > bound
    return (nd != nr) | (~nd & ~nr & far & (dev != ref))
