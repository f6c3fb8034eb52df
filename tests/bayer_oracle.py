"""CPU restatement of the demosaicing ingest applies to Bayer frames (DESIGN.md section 28): OpenCV's
cvtColor(frame, COLOR_Bayer<PATTERN>2BGR) (bilinear) and COLOR_Bayer<PATTERN>2BGR_EA (edge-aware) for the four colour
filter patterns.  golden_bayer.json pins it to cv2's own results.  With rectification the frame is
rectify_oracle.remap(bgr(frame, pattern, method), xy, a), in the reference's order (demosaic, then remap).

Two restatements: bgr, the vectorised clamp form, and bgr_loop, the definition written out pixel by pixel.  Every value
is an integer, so each output is exact.

Definition, for a frame raw of Wf x Hf whose 2 x 2 cell at (0, 0) has the pattern's colours in reading order:
  - interior pixel (1 <= x <= Wf - 2, 1 <= y <= Hf - 2) of colour c: channel c is raw(x, y).  At an R or B site
    G = (n4 + 2) >> 2 and the opposite colour = (d4 + 2) >> 2 (n4: the four edge neighbours' sum, d4: the four
    diagonal ones').  At a G site the colour of the horizontal neighbours is their (a + b + 1) >> 1, the other colour
    the vertical neighbours'.
  - edge-aware: G at an R or B site is the horizontal pair's (a + b + 1) >> 1 when |left - right| <= |up - down|
    (ties go horizontal), the vertical pair's otherwise.  R and B are the bilinear values.
  - border: pixel (x, y) is interior pixel (clamp(x, 1, Wf - 2), clamp(y, 1, Hf - 2)); every pixel is 0 when Wf < 3 or
    Hf < 3."""
import numpy as np

PATTERNS = ("rggb", "bggr", "grbg", "gbrg")
METHODS = ("bilinear", "ea")
# cv2's code of each pattern: its four-letter names (COLOR_BayerRGGB2BGR = COLOR_BayerBG2BGR = 46, ...)
CV2_CODE = {"rggb": 46, "bggr": 48, "grbg": 47, "gbrg": 49}
CV2_CODE_EA = {"rggb": 135, "bggr": 137, "grbg": 136, "gbrg": 138}


def red_site(pattern):
    """(rx, ry): the parity of the red site's column and row"""
    return {"rggb": (0, 0), "bggr": (1, 1), "grbg": (1, 0), "gbrg": (0, 1)}[pattern]


def bgr(raw, pattern, method="bilinear"):
    """cv2.cvtColor(raw, COLOR_Bayer<PATTERN>2BGR[_EA]): uint8 (Hf, Wf, 3), the vectorised clamp form"""
    raw = np.asarray(raw, np.uint8)
    H, W = raw.shape
    out = np.zeros((H, W, 3), np.uint8)
    if W < 3 or H < 3:
        return out
    r = raw.astype(np.int32)
    xs, ys = np.clip(np.arange(W), 1, W - 2), np.clip(np.arange(H), 1, H - 2)

    def at(dx, dy):   # raw(cx + dx, cy + dy) at each pixel's clamped position (cx, cy)
        return r[(ys + dy)[:, None], (xs + dx)[None, :]]

    c, le, ri, up, dn = at(0, 0), at(-1, 0), at(1, 0), at(0, -1), at(0, 1)
    d4 = at(-1, -1) + at(1, -1) + at(-1, 1) + at(1, 1)
    hor, ver = (le + ri + 1) >> 1, (up + dn + 1) >> 1
    if method == "ea":
        g_rb = np.where(np.abs(le - ri) <= np.abs(up - dn), hor, ver)
    else:
        g_rb = (le + ri + up + dn + 2) >> 2
    diag = (d4 + 2) >> 2
    rx, ry = red_site(pattern)
    px, py = ((xs[None, :] ^ rx) & 1), ((ys[:, None] ^ ry) & 1)   # 0 on the red site's columns / rows
    red, blue = (px == 0) & (py == 0), (px == 1) & (py == 1)
    red_row = np.broadcast_to(py == 0, c.shape)
    R = np.where(red, c, np.where(blue, diag, np.where(red_row, hor, ver)))
    B = np.where(blue, c, np.where(red, diag, np.where(red_row, ver, hor)))
    G = np.where(red | blue, g_rb, c)
    out[...] = np.stack([B, G, R], -1)
    return out


def bgr_loop(raw, pattern, method="bilinear"):
    """the definition pixel by pixel; equals bgr"""
    raw = np.asarray(raw, np.uint8)
    H, W = raw.shape
    out = np.zeros((H, W, 3), np.uint8)
    if W < 3 or H < 3:
        return out
    rx, ry = red_site(pattern)
    for y in range(H):
        for x in range(W):
            cx, cy = min(max(x, 1), W - 2), min(max(y, 1), H - 2)

            def p(dx, dy):
                return int(raw[cy + dy, cx + dx])

            le, ri, up, dn = p(-1, 0), p(1, 0), p(0, -1), p(0, 1)
            hor, ver = (le + ri + 1) >> 1, (up + dn + 1) >> 1
            red_row, red_col = (cy - ry) % 2 == 0, (cx - rx) % 2 == 0
            if red_row == red_col:   # an R or B site
                if method == "ea":
                    g = hor if abs(le - ri) <= abs(up - dn) else ver
                else:
                    g = (le + ri + up + dn + 2) >> 2
                opp = (p(-1, -1) + p(1, -1) + p(-1, 1) + p(1, 1) + 2) >> 2
                R, B = (p(0, 0), opp) if red_row else (opp, p(0, 0))
                G = g
            else:   # a G site: its row's other colour is horizontal
                G = p(0, 0)
                R, B = (hor, ver) if red_row else (ver, hor)
            out[y, x] = (B, G, R)
    return out


def frame(seed, width, height, high=256):
    """a seeded raw frame of width x height, every sample uniform in 0 .. high - 1"""
    return np.random.default_rng(seed).integers(0, high, (height, width), dtype=np.uint8)


def from_bgr(img, pattern):
    """the raw frame a camera with the pattern would take of the BGR image img: each pixel keeps its site's colour.  Any
    frame is a valid input; this one gives the matcher a real scene."""
    img = np.asarray(img, np.uint8)
    H, W = img.shape[:2]
    rx, ry = red_site(pattern)
    px, py = (np.arange(W)[None, :] ^ rx) & 1, (np.arange(H)[:, None] ^ ry) & 1
    ch = np.where((px == 0) & (py == 0), 2, np.where((px == 1) & (py == 1), 0, 1))
    return np.take_along_axis(img, ch[..., None], 2)[..., 0].copy()
