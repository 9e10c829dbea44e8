"""oracle/raster_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT.  PARITY UNPINNED (see below).

CPU (numpy, float64) restatement of the two nvdiffrast operators the reference's stage 1 calls
(`dr.rasterize`, `dr.interpolate`; call sites nerf/renderer.py:860-863, consumers :890 `rast[..., 2]` as depth and :894
`rast[..., -1] - 1` as triangle id).  nvdiffrast is a third-party dependency of the reference that is NOT vendored under
the reference tree and not installed in this image; the reference pins no version (readme.md:28-29 installs the git head).  Its published
output convention (nvdiffrast documentation, "rasterize" / "interpolate"):

    rast[n, y, x] = (u, v, z/w, triangle_id + 1), all zero where no triangle covers the pixel centre;
    pixel (x, y) has its centre at NDC ((x + 0.5) / W * 2 - 1, (y + 0.5) / H * 2 - 1)  (row 0 = y_ndc -1, OpenGL orientation);
    (u, v) are PERSPECTIVE-CORRECT barycentrics of vertices 0 and 1 (vertex 2 has 1 - u - v);  z/w is the NDC depth, linear in
    screen space; the nearest fragment with -1 <= z/w <= 1 wins (GL depth test LESS);
    interpolate: attr = u * a0 + v * a1 + (1 - u - v) * a2, zero where triangle_id == 0.

"Parity unpinned": the reference's tests hold no golden vectors at this boundary (it has no tests at all) and the library cannot be
run here, so this oracle is anchored on the documented convention and on the reference's call sites only; exact fill-rule ties
(a pixel centre exactly on an edge) follow OpenGL rules in the library and are NOT reproduced: an edge hit counts as covered.  The
tests avoid them and allow id mismatches only on pixels whose smallest screen-space barycentric is within 1e-5 of zero.
Near / far clipping: triangles in front of the camera plane (all w > 0) are tested per pixel against -1 <= z/w <= 1; triangles that
cross the camera plane (some w <= 0) are rasterised in homogeneous coordinates (`_rasterize_homogeneous`), which yields exactly the part
in front of the near plane without constructing clipped polygons -- the result the library's clipper produces.
"""
import numpy as np


def rasterize(pos, tri, H, W):
    """pos [V,4] clip space (float), tri [F,3] int -> rast [H,W,4] float64 = (u, v, z/w, id+1)."""
    pos = np.asarray(pos, np.float64); tri = np.asarray(tri, np.int64)
    rast = np.zeros((H, W, 4))
    zbuf = np.full((H, W), np.inf)
    idbuf = np.zeros((H, W), np.int64)
    w = pos[:, 3]
    ndc = pos[:, :3] / np.where(w == 0, 1.0, w)[:, None]
    sx = (ndc[:, 0] * 0.5 + 0.5) * W          # continuous pixel coordinates: centre of pixel x is at x + 0.5
    sy = (ndc[:, 1] * 0.5 + 0.5) * H
    for f in range(tri.shape[0]):
        i0, i1, i2 = tri[f]
        if w[i0] <= 0 or w[i1] <= 0 or w[i2] <= 0:
            if not (w[i0] <= 0 and w[i1] <= 0 and w[i2] <= 0):
                _rasterize_homogeneous(pos, f, i0, i1, i2, H, W, rast, zbuf, idbuf)
            continue
        x0, y0, x1, y1, x2, y2 = sx[i0], sy[i0], sx[i1], sy[i1], sx[i2], sy[i2]
        area = (x1 - x0) * (y2 - y0) - (x2 - x0) * (y1 - y0)
        if area == 0:
            continue
        xa = int(max(np.floor(min(x0, x1, x2) - 0.5), 0)); xb = int(min(np.ceil(max(x0, x1, x2) - 0.5), W - 1))
        ya = int(max(np.floor(min(y0, y1, y2) - 0.5), 0)); yb = int(min(np.ceil(max(y0, y1, y2) - 0.5), H - 1))
        if xa > xb or ya > yb:
            continue
        px = np.arange(xa, xb + 1) + 0.5
        py = np.arange(ya, yb + 1) + 0.5
        PX, PY = np.meshgrid(px, py)
        # screen-space barycentrics (sum to 1)
        b0 = ((x1 - PX) * (y2 - PY) - (x2 - PX) * (y1 - PY)) / area
        b1 = ((x2 - PX) * (y0 - PY) - (x0 - PX) * (y2 - PY)) / area
        b2 = 1.0 - b0 - b1
        inside = (b0 >= 0) & (b1 >= 0) & (b2 >= 0)
        if not inside.any():
            continue
        z = b0 * ndc[i0, 2] + b1 * ndc[i1, 2] + b2 * ndc[i2, 2]
        ok = inside & (z >= -1) & (z <= 1)
        sub_z = zbuf[ya:yb + 1, xa:xb + 1]
        sub_id = idbuf[ya:yb + 1, xa:xb + 1]
        win = ok & ((z < sub_z) | ((z == sub_z) & (f + 1 < sub_id)))
        if not win.any():
            continue
        p0, p1, p2 = b0 / w[i0], b1 / w[i1], b2 / w[i2]
        ps = p0 + p1 + p2
        sub = rast[ya:yb + 1, xa:xb + 1]
        sub[win, 0] = (p0 / ps)[win]; sub[win, 1] = (p1 / ps)[win]; sub[win, 2] = z[win]; sub[win, 3] = f + 1
        sub_z[win] = z[win]; sub_id[win] = f + 1
    return rast


def near_clip_bbox(p0, p1, p2, H, W):
    """pixel bounding box (xa, xb, ya, yb, inclusive, clamped; None if empty) of a triangle clipped against the near plane z >= -w"""
    poly = [np.asarray(p, np.float64) for p in (p0, p1, p2)]
    out = []
    for k in range(3):
        a, b = poly[k], poly[(k + 1) % 3]
        da, db = a[2] + a[3], b[2] + b[3]
        if da >= 0:
            out.append(a)
        if (da >= 0) != (db >= 0):
            t = da / (da - db)
            out.append(a + t * (b - a))
    if not out:
        return None
    xs, ys = [], []
    for q in out:
        ww = max(q[3], 1e-30)
        xs.append((q[0] / ww * 0.5 + 0.5) * W); ys.append((q[1] / ww * 0.5 + 0.5) * H)
    xa = int(max(np.floor(min(min(xs), W + 1.0) - 0.5), 0)); xb = int(min(np.ceil(max(max(xs), -1.0) - 0.5), W - 1))
    ya = int(max(np.floor(min(min(ys), H + 1.0) - 0.5), 0)); yb = int(min(np.ceil(max(max(ys), -1.0) - 0.5), H - 1))
    if xa > xb or ya > yb:
        return None
    return xa, xb, ya, yb


def _rasterize_homogeneous(pos, f, i0, i1, i2, H, W, rast, zbuf, idbuf):
    """a triangle with one or two vertices at w <= 0 (it crosses the camera plane): 2-D homogeneous rasterization (Olano & Greer 1997).
    For pixel NDC (X, Y) solve  sum_i b'_i (x_i, y_i, w_i) = (X, Y, 1): the pixel is covered iff all b'_i >= 0 (the point then lies in
    the triangle and in front of the camera), z/w = sum_i b'_i z_i (tested against [-1, 1]: the near / far clip, per pixel),
    (u, v) = (b'_0, b'_1) / sum b'."""
    p = [pos[i0], pos[i1], pos[i2]]
    box = near_clip_bbox(p[0], p[1], p[2], H, W)
    if box is None:
        return
    xa, xb, ya, yb = box
    M = np.array([[p[0][0], p[1][0], p[2][0]], [p[0][1], p[1][1], p[2][1]], [p[0][3], p[1][3], p[2][3]]], np.float64)
    det = np.linalg.det(M)
    if det == 0 or not np.isfinite(det):
        return
    Mi = np.linalg.inv(M)
    px = (np.arange(xa, xb + 1) + 0.5) / W * 2 - 1
    py = (np.arange(ya, yb + 1) + 0.5) / H * 2 - 1
    PX, PY = np.meshgrid(px, py)
    b = [Mi[k, 0] * PX + Mi[k, 1] * PY + Mi[k, 2] for k in range(3)]
    inside = (b[0] >= 0) & (b[1] >= 0) & (b[2] >= 0)
    if not inside.any():
        return
    z = b[0] * p[0][2] + b[1] * p[1][2] + b[2] * p[2][2]
    ok = inside & (z >= -1) & (z <= 1)
    sub_z = zbuf[ya:yb + 1, xa:xb + 1]; sub_id = idbuf[ya:yb + 1, xa:xb + 1]
    win = ok & ((z < sub_z) | ((z == sub_z) & (f + 1 < sub_id)))
    if not win.any():
        return
    bs = b[0] + b[1] + b[2]
    sub = rast[ya:yb + 1, xa:xb + 1]
    sub[win, 0] = (b[0] / bs)[win]; sub[win, 1] = (b[1] / bs)[win]; sub[win, 2] = z[win]; sub[win, 3] = f + 1
    sub_z[win] = z[win]; sub_id[win] = f + 1


def edge_distance(pos, tri, rast):
    """per covered pixel: the smallest screen-space barycentric of the winning triangle (how close the centre is to an edge)"""
    pos = np.asarray(pos, np.float64)
    H, W = rast.shape[:2]
    w = pos[:, 3]
    ndc = pos[:, :3] / w[:, None]
    sx = (ndc[:, 0] * 0.5 + 0.5) * W; sy = (ndc[:, 1] * 0.5 + 0.5) * H
    out = np.full((H, W), np.inf)
    ys, xs = np.nonzero(rast[..., 3] > 0)
    f = rast[ys, xs, 3].astype(np.int64) - 1
    i0, i1, i2 = tri[f, 0], tri[f, 1], tri[f, 2]
    PX, PY = xs + 0.5, ys + 0.5
    area = (sx[i1] - sx[i0]) * (sy[i2] - sy[i0]) - (sx[i2] - sx[i0]) * (sy[i1] - sy[i0])
    b0 = ((sx[i1] - PX) * (sy[i2] - PY) - (sx[i2] - PX) * (sy[i1] - PY)) / area
    b1 = ((sx[i2] - PX) * (sy[i0] - PY) - (sx[i0] - PX) * (sy[i2] - PY)) / area
    out[ys, xs] = np.minimum(np.minimum(b0, b1), 1 - b0 - b1)
    return out


def interpolate(attr, rast, tri):
    """attr [V,A], rast [H,W,4], tri [F,3] -> [H,W,A]"""
    attr = np.asarray(attr, np.float64)
    H, W = rast.shape[:2]
    out = np.zeros((H, W, attr.shape[1]))
    ys, xs = np.nonzero(rast[..., 3] > 0)
    f = rast[ys, xs, 3].astype(np.int64) - 1
    u, v = rast[ys, xs, 0][:, None], rast[ys, xs, 1][:, None]
    out[ys, xs] = u * attr[tri[f, 0]] + v * attr[tri[f, 1]] + (1 - u - v) * attr[tri[f, 2]]
    return out


def interpolate_backward(grad_out, attr_shape, rast, tri):
    """d loss / d attr [V,A] for grad_out [H,W,A]"""
    g = np.zeros(attr_shape)
    ys, xs = np.nonzero(rast[..., 3] > 0)
    f = rast[ys, xs, 3].astype(np.int64) - 1
    u, v = rast[ys, xs, 0][:, None], rast[ys, xs, 1][:, None]
    go = np.asarray(grad_out, np.float64)[ys, xs]
    np.add.at(g, tri[f, 0], u * go); np.add.at(g, tri[f, 1], v * go); np.add.at(g, tri[f, 2], (1 - u - v) * go)
    return g


# ---- synthetic closed meshes / projections: input synthesis shared with the bench lives in the product package ----
from nerf2mesh_b200.synthetic import icosphere, perspective_mvp  # noqa: E402,F401  (re-exported: the tests build their scenes through this module)
