"""CPU restatement of the uniqueness test (psm_set_uniqueness_check, OpenCV StereoSGBM's uniquenessRatio).  Test
infrastructure.

Definition, per pixel of one view's selection map m, with q(m) = plane 1 of PSM_OPT_COSTS and q(r) = plane 1 of
PSM_OPT_RUNNER_UP: a pixel with m != 0 becomes 0 when (double)q(r) * (100 - ratio) < (double)q(m) * 100; every other
pixel keeps its value.

Two forms:
  - check: the runner-up form above, which the device computes;
  - check_loop: computeDisparitySGBM's own loop, `Sp[d]*(100 - uniquenessRatio) < minS*100 && abs(bestDisp - d) > 1`
    over every candidate d of the filtered volume, [max(1, min_disp), max_disp), in fp64.
They agree because the runner-up is the lowest candidate with |d - m| >= 2 and multiplying by a constant >= 0 keeps the
order; the CPU tests hold check to check_loop rather than assume it.
"""
import numpy as np

MAX_RATIO = 100   # the largest ratio psm_set_uniqueness_check takes


def _ratio(ratio):
    assert isinstance(ratio, (int, np.integer)) and 0 <= ratio <= MAX_RATIO, ratio
    return int(ratio)


def check(m, qm, qr, ratio):
    """m (u8 / u16 [H, W]), q(m) and q(r) (float32 [H, W]) -> the tested map, of m's dtype"""
    ratio = _ratio(ratio)
    m = np.asarray(m)
    assert m.ndim == 2 and m.dtype in (np.uint8, np.uint16), (m.shape, m.dtype)
    qm, qr = np.asarray(qm, np.float32), np.asarray(qr, np.float32)
    assert qm.shape == m.shape and qr.shape == m.shape
    with np.errstate(invalid="ignore", over="ignore"):
        reject = (m != 0) & (qr.astype(np.float64) * (100 - ratio) < qm.astype(np.float64) * 100)
    return np.where(reject, 0, m).astype(m.dtype)


def check_loop(m, vol, ratio, min_disp=0):
    """m (u8 / u16 [H, W]) selected from vol (float32 [D, H, W], the slices of the whole range [0, D), of which the
    context searched [min_disp, D)) -> the tested map: OpenCV's loop over every candidate d"""
    ratio = _ratio(ratio)
    m = np.asarray(m)
    f = np.asarray(vol, np.float32)
    mi = m.astype(np.int64)
    minS = np.take_along_axis(f, np.clip(mi, 0, f.shape[0] - 1)[None], 0)[0].astype(np.float64) * 100
    reject = np.zeros(m.shape, bool)
    for d in range(max(1, min_disp), f.shape[0]):
        with np.errstate(invalid="ignore", over="ignore"):
            reject |= (f[d].astype(np.float64) * (100 - ratio) < minS) & (np.abs(d - mi) > 1)
    return np.where((m != 0) & reject, 0, m).astype(m.dtype)
