"""CPU restatement of the median step (psm_set_median_blur, OpenCV's medianBlur).  Test infrastructure; pinned to
cv2.medianBlur itself by tests/golden/golden_median.json (tests/golden/make_golden_median.py).

Definition, per view: out(x, y) = the median of the ksize x ksize map values around (x, y), rows and columns clamped to
the map (BORDER_REPLICATE); zeros take part as values.
"""
import numpy as np

KSIZES = (3, 5)


def median(m, ksize):
    """m (u8 / u16 [H, W]) -> the ksize x ksize edge-replicated median, of m's dtype"""
    m = np.asarray(m)
    assert m.ndim == 2 and m.dtype in (np.uint8, np.uint16) and ksize in KSIZES, (m.shape, m.dtype, ksize)
    R = ksize // 2
    H, W = m.shape
    p = np.pad(m, R, mode="edge")
    win = np.stack([p[j:j + H, i:i + W] for j in range(ksize) for i in range(ksize)])
    return np.sort(win, axis=0)[ksize * ksize // 2].astype(m.dtype)


def seeded(H, W, u16, seed):
    """a map of constant rows and noise with a quarter zeros, u8 up to 255 or u16 up to 4095: the seeded inputs of the
    median's golden cases"""
    rng = np.random.default_rng(seed)
    top = 4096 if u16 else 256
    m = rng.integers(0, top, (H, W))
    m = np.where(rng.random((H, W)) < 0.5, np.repeat(rng.integers(0, top, (H, 1)), W, axis=1), m)
    m = np.where(rng.random((H, W)) < 0.25, 0, m)
    return m.astype(np.uint16 if u16 else np.uint8)
