"""CPU oracle of the texture post-processing of NeRFRenderer._export_obj (nerf/renderer.py:374-402), restated literally with the libraries
the reference uses (scipy.ndimage dilation / erosion, an sklearn KD-tree, cv2.resize), plus the closed forms the device kernels use
(csrc/texture.cu): the L1-ball classification, the separable +-32 windowed nearest-neighbour search and the 2x2 rounded mean."""
import numpy as np


def reference_inpaint(feats, mask):
    """renderer.py:378-394 verbatim -> (inpainted feats, inpaint_region, search_region, squared distance of every inpaint texel (in
    np.nonzero order) to the search texel the KD-tree chose).  An empty mask returns the input (the reference's fit fails there)."""
    from scipy.ndimage import binary_dilation, binary_erosion
    from sklearn.neighbors import NearestNeighbors
    feats = feats.copy()
    mask = mask.astype(bool)
    inpaint_region = binary_dilation(mask, iterations=32)
    inpaint_region[mask] = 0
    search_region = mask.copy()
    not_search_region = binary_erosion(search_region, iterations=3)
    search_region[not_search_region] = 0
    if not mask.any():
        return feats, inpaint_region, search_region, np.zeros(0, dtype=np.int64)
    search_coords = np.stack(np.nonzero(search_region), axis=-1)
    inpaint_coords = np.stack(np.nonzero(inpaint_region), axis=-1)
    if len(inpaint_coords) == 0:
        return feats, inpaint_region, search_region, np.zeros(0, dtype=np.int64)
    knn = NearestNeighbors(n_neighbors=1, algorithm="kd_tree").fit(search_coords)
    _, indices = knn.kneighbors(inpaint_coords)
    src = search_coords[indices[:, 0]]
    feats[tuple(inpaint_coords.T)] = feats[tuple(src.T)]
    d2 = ((src - inpaint_coords) ** 2).sum(-1).astype(np.int64)
    return feats, inpaint_region, search_region, d2


def reference_resize(img, w0, h0):
    """cv2.resize(img, (w0, h0), INTER_LINEAR) (renderer.py:400-402)"""
    import cv2
    return cv2.resize(img, (w0, h0), interpolation=cv2.INTER_LINEAR)


def _windowed_min(a, radius, axis, big):
    """out[i] = min over |d| <= radius of (a[i + d] + d^2) along `axis` (in-image d only)"""
    out = np.full(a.shape, big, dtype=np.int64)
    n = a.shape[axis]
    for d in range(-radius, radius + 1):
        lo, hi = max(0, -d), min(n, n - d)
        if hi <= lo:
            continue
        src = np.take(a, np.arange(lo + d, hi + d), axis=axis)
        idx = [slice(None)] * a.ndim
        idx[axis] = slice(lo, hi)
        idx = tuple(idx)
        out[idx] = np.minimum(out[idx], src + d * d)
    return out


def l1_distance_le(mask, radius):
    """L1 distance to the nearest True texel <= radius (the closed form of binary_dilation(mask, iterations=radius))"""
    big = 1 << 30
    col = np.where(mask, 0, big).astype(np.int64)
    g = np.full(mask.shape, big, dtype=np.int64)
    for d in range(-radius, radius + 1):                       # column pass: min |dy|
        n = mask.shape[0]
        lo, hi = max(0, -d), min(n, n - d)
        if hi > lo:
            g[lo:hi] = np.minimum(g[lo:hi], col[lo + d:hi + d] + abs(d))
    out = np.full(mask.shape, big, dtype=np.int64)
    for d in range(-radius, radius + 1):                       # row pass: min |dx| + g
        n = mask.shape[1]
        lo, hi = max(0, -d), min(n, n - d)
        if hi > lo:
            out[:, lo:hi] = np.minimum(out[:, lo:hi], g[:, lo + d:hi + d] + abs(d))
    return out <= radius


def closed_form_regions(mask):
    """(inpaint, search) by the L1 rules: dilation = L1 distance to the mask <= 32; erosion (border 0) = every texel within L1 3 in the
    image and in the mask"""
    mask = mask.astype(bool)
    inpaint = l1_distance_le(mask, 32) & ~mask
    padded = np.pad(~mask, 3, constant_values=True)
    near_outside = l1_distance_le(padded, 3)[3:-3, 3:-3]
    search = mask & near_outside
    return inpaint, search


def windowed_min_d2(search, radius=32):
    """the separable exact search: g(x, y) = min dy^2 over the search texels of column x within the window, then min dx^2 + g(x + dx, y)"""
    big = 1 << 40
    g = _windowed_min(np.where(search, 0, big).astype(np.int64), radius, 0, big)
    return _windowed_min(g, radius, 1, big)


def down2(feats):
    """(a + b + c + d + 2) >> 2 over each 2x2 block"""
    f = feats.astype(np.uint32)
    s = f[0::2, 0::2] + f[0::2, 1::2] + f[1::2, 0::2] + f[1::2, 1::2]
    return ((s + 2) >> 2).astype(np.uint8)


def grid_atlas(F, gutter=0.18):
    """a per-triangle UV atlas (xatlas stands in the caller's place): triangle i gets its own right triangle in cell i of a
    ceil(sqrt(F))^2 grid, inset by `gutter` of a cell -> vt [3F,2] float32, ft [F,3] int32"""
    n = int(np.ceil(np.sqrt(F)))
    c = 1.0 / n
    i = np.arange(F)
    x0, y0 = (i % n) * c, (i // n) * c
    g = gutter * c
    vt = np.stack([np.stack([x0 + g, y0 + g], 1), np.stack([x0 + c - g, y0 + g], 1), np.stack([x0 + g, y0 + c - g], 1)], 1)
    return vt.reshape(-1, 2).astype(np.float32), np.arange(3 * F, dtype=np.int32).reshape(F, 3)


def sample_masks():
    """(name, mask) cases for the inpaint: random blobs, blobs touching every border, single texels, empty, full"""
    h, w = 300, 260
    out = [("blobs", blob_mask(h, w, 14, seed=1)), ("sparse_blobs", blob_mask(h, w, 5, seed=2, rmax=9))]
    m = blob_mask(h, w, 6, seed=3)
    yy, xx = np.mgrid[0:h, 0:w]
    for cy, cx in ((0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1), (0, w // 2), (h // 2, 0), (h - 1, w // 3), (h // 3, w - 1)):
        m |= (yy - cy) ** 2 + (xx - cx) ** 2 <= 15 ** 2
    out.append(("touches_every_border", m))
    s = np.zeros((90, 70), dtype=bool); s[40, 31] = True
    out.append(("single_texel", s))
    c = np.zeros((64, 64), dtype=bool); c[0, 0] = True
    out.append(("single_corner_texel", c))
    out.append(("empty", np.zeros((50, 40), dtype=bool)))
    out.append(("full", np.ones((40, 50), dtype=bool)))
    return out


def blob_mask(h, w, n, seed, rmax=20):
    """union of random discs (some touching the border)"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    m = np.zeros((h, w), dtype=bool)
    for _ in range(n):
        cy, cx, r = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(2, rmax)
        m |= (yy - cy) ** 2 + (xx - cx) ** 2 <= r * r
    return m
