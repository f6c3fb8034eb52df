"""CPU restatements of speckle removal (psm_set_speckle_filter, OpenCV's cv::filterSpeckles(m, 0, max_size, max_diff)),
which the device runs as union-find labelling.  Test infrastructure; pinned to cv2.filterSpeckles itself by
tests/golden/golden_speckle.json (tests/golden/make_golden_speckle.py).

Definition: pixels of value 0 belong to no blob; two 4-neighbours p, q, both non-zero, are in the same blob when
|m(p) - m(q)| <= max_diff (as int); every pixel of a blob of at most max_size pixels becomes 0, every other pixel keeps
its value.

filter_speckles labels the blobs with scipy's connected components of that graph (fast enough for full-size maps);
filter_speckles_flood is a raster-order flood fill written from the definition, for small maps, that the tests hold
the first one to.
"""
import hashlib
from collections import deque

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components


def _check(m, max_size, max_diff):
    m = np.asarray(m)
    assert m.ndim == 2 and m.dtype in (np.uint8, np.uint16, np.int16), (m.shape, m.dtype)
    assert max_size >= 1 and max_diff >= 0
    return m


def blob_sizes(m, max_diff):
    """-> (component label per pixel, pixels per component) of the blob graph; zero pixels are singletons"""
    H, W = m.shape
    v = m.astype(np.int64)
    idx = np.arange(H * W, dtype=np.int64).reshape(H, W)
    nz = v != 0
    eh = nz[:, :-1] & nz[:, 1:] & (np.abs(v[:, :-1] - v[:, 1:]) <= max_diff)
    ev = nz[:-1, :] & nz[1:, :] & (np.abs(v[:-1, :] - v[1:, :]) <= max_diff)
    src = np.concatenate([idx[:, :-1][eh], idx[:-1, :][ev]])
    dst = np.concatenate([idx[:, 1:][eh], idx[1:, :][ev]])
    g = coo_matrix((np.ones(src.size, np.int8), (src, dst)), shape=(H * W, H * W))
    _, comp = connected_components(g, directed=False)
    return comp.reshape(H, W), np.bincount(comp)


def filter_speckles(m, max_size, max_diff):
    """-> the filtered map, of m's dtype"""
    m = _check(m, max_size, max_diff)
    comp, size = blob_sizes(m, max_diff)
    return np.where((m != 0) & (size[comp] <= max_size), 0, m).astype(m.dtype)


def filter_speckles_flood(m, max_size, max_diff):
    """raster-order flood fill of every unlabelled non-zero pixel (cv::filterSpeckles' own visiting order) -> the
    filtered map"""
    m = _check(m, max_size, max_diff)
    H, W = m.shape
    v = m.astype(np.int64).tolist()
    out = m.copy()
    seen = [[False] * W for _ in range(H)]
    for y0 in range(H):
        for x0 in range(W):
            if v[y0][x0] == 0 or seen[y0][x0]:
                continue
            seen[y0][x0] = True
            blob, todo = [], deque([(y0, x0)])
            while todo:
                y, x = todo.popleft()
                blob.append((y, x))
                for yy, xx in ((y, x + 1), (y + 1, x), (y, x - 1), (y - 1, x)):
                    if 0 <= yy < H and 0 <= xx < W and not seen[yy][xx] and v[yy][xx] != 0 \
                            and abs(v[yy][xx] - v[y][x]) <= max_diff:
                        seen[yy][xx] = True
                        todo.append((yy, xx))
            if len(blob) <= max_size:
                for y, x in blob:
                    out[y, x] = 0
    return out


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
