"""CPU restatement of the YUV-to-BGR conversion ingest applies to YUV frames (DESIGN.md section 27): OpenCV's
cvtColor(frame, COLOR_YUV2BGR_<FORMAT>), BT.601 limited range in fixed point, and the unpacking of each of cv2's seven
layouts.  golden_yuv.json pins it to cv2's own results.  With rectification the frame is
rectify_oracle.remap(bgr(frame, fmt), xy, a), in the reference's order (convert, then remap).

Every value is an integer, so each output is exact."""
import numpy as np

FORMATS = ("nv12", "nv21", "i420", "yv12", "yuyv", "uyvy", "yvyu")
FORMATS_420 = FORMATS[:4]


def convert(Y, U, V):
    """integer arrays of equal shape -> uint8 (..., 3) B, G, R, each clamped to 0..255"""
    y = np.maximum(np.asarray(Y, np.int64) - 16, 0) * 1220542 + (1 << 19)
    u = np.asarray(U, np.int64) - 128
    v = np.asarray(V, np.int64) - 128
    b = (y + 2116026 * u) >> 20
    g = (y - 852492 * v - 409993 * u) >> 20
    r = (y + 1673527 * v) >> 20
    return np.clip(np.stack([b, g, r], -1), 0, 255).astype(np.uint8)


def shape(fmt, width, height):
    """cv2's shape of a frame of width x height: (H * 3 / 2, W) for 4:2:0, (H, W, 2) for 4:2:2"""
    return (height * 3 // 2, width) if fmt in FORMATS_420 else (height, width, 2)


def size(frame, fmt):
    """(width, height) of a frame in cv2's layout"""
    return (frame.shape[1], frame.shape[0] * 2 // 3) if fmt in FORMATS_420 else (frame.shape[1], frame.shape[0])


def planes(frame, fmt):
    """a frame in cv2's layout -> (Y, U, V), each (H, W): the chroma sample of pixel (x, y) is the one at
    (x >> 1, y >> 1) for 4:2:0 and (x >> 1, y) for 4:2:2"""
    frame = np.asarray(frame, np.uint8)
    W, H = size(frame, fmt)
    if fmt in FORMATS_420:
        Y = frame[:H]
        if fmt in ("nv12", "nv21"):
            uv = frame[H:].reshape(H // 2, W // 2, 2)
            U, V = (uv[..., 0], uv[..., 1]) if fmt == "nv12" else (uv[..., 1], uv[..., 0])
        else:   # two planes of W / 2 x H / 2, packed into the rows after the luma
            q = (W // 2) * (H // 2)
            flat = frame[H:].ravel()
            first, second = flat[:q].reshape(H // 2, W // 2), flat[q:2 * q].reshape(H // 2, W // 2)
            U, V = (first, second) if fmt == "i420" else (second, first)
        U = np.repeat(np.repeat(U, 2, 0), 2, 1)
        V = np.repeat(np.repeat(V, 2, 0), 2, 1)
        return Y, U, V
    pairs = frame.reshape(H, W // 2, 4)   # one macropixel of two pixels: 4 bytes
    order = {"yuyv": (0, 2, 1, 3), "uyvy": (1, 3, 0, 2), "yvyu": (0, 2, 3, 1)}[fmt]   # Y0, Y1, U, V
    Y = np.stack([pairs[..., order[0]], pairs[..., order[1]]], -1).reshape(H, W)
    U = np.repeat(pairs[..., order[2]], 2, 1)
    V = np.repeat(pairs[..., order[3]], 2, 1)
    return Y, U, V


def bgr(frame, fmt):
    """cv2.cvtColor(frame, COLOR_YUV2BGR_<FMT>): uint8 (H, W, 3)"""
    return convert(*planes(frame, fmt))


def frame(seed, fmt, width, height):
    """a seeded frame of width x height in cv2's layout (every byte uniform)"""
    return np.random.default_rng(seed).integers(0, 256, shape(fmt, width, height), dtype=np.uint8)


def all_triples():
    """a YUYV frame of 4096 x 4096 that holds each (Y, U, V) triple once: pixel t = y * 4096 + x holds Y = t & 255,
    U = (t >> 8) & 255, V = t >> 16 (the two pixels of a macropixel share U and V)"""
    t = np.arange(1 << 24, dtype=np.uint32).reshape(4096, 2048, 2)
    out = np.empty((4096, 2048, 4), np.uint8)
    out[..., 0] = t[..., 0] & 255
    out[..., 2] = t[..., 1] & 255
    out[..., 1] = (t[..., 0] >> 8) & 255
    out[..., 3] = t[..., 0] >> 16
    return out.reshape(4096, 4096, 2)


def all_triples_bgr():
    """bgr(all_triples(), "yuyv"), from the triples directly: (4096, 4096, 3)"""
    t = np.arange(1 << 24, dtype=np.int64)
    return convert(t & 255, (t >> 8) & 255, t >> 16).reshape(4096, 4096, 3)


def pack(Y, U, V, fmt):
    """luma (H, W) and chroma at its own resolution -- (H / 2, W / 2) for 4:2:0, (H, W / 2) for 4:2:2 -> a frame in
    cv2's layout for fmt (the inverse of planes on the chroma samples it keeps)"""
    Y, U, V = (np.asarray(p, np.uint8) for p in (Y, U, V))
    H, W = Y.shape
    if fmt in ("nv12", "nv21"):
        uv = np.stack([U, V] if fmt == "nv12" else [V, U], -1).reshape(H // 2, W)
        return np.vstack([Y, uv])
    if fmt in ("i420", "yv12"):
        first, second = (U, V) if fmt == "i420" else (V, U)
        return np.concatenate([Y.ravel(), first.ravel(), second.ravel()]).reshape(H * 3 // 2, W)
    order = {"yuyv": (0, 2, 1, 3), "uyvy": (1, 3, 0, 2), "yvyu": (0, 2, 3, 1)}[fmt]
    out = np.empty((H, W // 2, 4), np.uint8)
    out[..., order[0]], out[..., order[1]] = Y[:, 0::2], Y[:, 1::2]
    out[..., order[2]], out[..., order[3]] = U, V
    return out.reshape(H, W, 2)


def from_bgr(img, fmt):
    """a frame of fmt that looks like the BGR image img (even sides): BT.601 limited range, chroma of the top-left pixel
    of each block.  Any frame is a valid input; this one gives the matcher a real scene."""
    b, g, r = (img[..., k].astype(np.float64) for k in range(3))
    Y = np.clip(np.rint(16 + (65.481 * r + 128.553 * g + 24.966 * b) / 255), 0, 255)
    U = np.clip(np.rint(128 + (-37.797 * r - 74.203 * g + 112.0 * b) / 255), 0, 255)
    V = np.clip(np.rint(128 + (112.0 * r - 93.786 * g - 18.214 * b) / 255), 0, 255)
    step = 2 if fmt in FORMATS_420 else 1
    return pack(Y, U[::step, 0::2], V[::step, 0::2], fmt)
