"""oracle/antialias_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT.  PARITY UNPINNED (see below).

CPU (numpy, float64, plain loops) restatement of the third nvdiffrast operator of the reference's stage 1, `dr.antialias`
(call sites nerf/renderer.py:886-887: `dr.antialias(alphas | rgbs, rast, vertices_clip, self.triangles, pos_gradient_boost=...)`,
the only differentiable path from the image loss to `vertices_offsets` when `enable_offset_nerf_grad` is off).  nvdiffrast is not
vendored in the reference tree, not installed here, and the reference pins no version, so the library cannot be run: this file
restates the PUBLISHED algorithm (Laine et al., "Modular Primitives for High-Performance Differentiable Rendering", section 3.4
"Antialiasing"; nvdiffrast documentation, "antialias") and is anchored on the reference's call sites and on hand-computable
cases (tests/test_antialias_oracle.py).  The reference's tests hold no vectors at this boundary: PARITY UNPINNED.

Algorithm (per pair of horizontally or vertically adjacent pixels with different triangle ids in `rast[..., 3]`):
  1. the FOREGROUND pixel P is the one whose surface is closer: the covered one if the other is background, else the smaller z/w
     (ties: the second pixel of the pair); Q is the other pixel;
  2. the first edge (order v0v1, v1v2, v2v0) of P's triangle whose screen-space segment crosses the segment between the two pixel
     centres strictly inside (0 < t < 1, t measured from P's centre) is the candidate;
  3. it must be a SILHOUETTE edge: it belongs to one triangle only, or the two triangles that share it lie on the same side of it in
     screen space (one folds behind the other);
  4. alpha = t - 0.5: the foreground surface covers (0.5 + t) of the pair's span.  alpha > 0: it reaches into Q,
         out[Q] += alpha * (in[P] - in[Q]);      alpha <= 0: it leaves part of P uncovered,   out[P] += alpha * (in[P] - in[Q]).
Gradients: to both colours (+-alpha) and, through t, to the clip-space x, y, w of the edge's two vertices (multiplied by
`pos_gradient_boost`).  Vertices with w <= 0 disable the pair.  Edges shared by more than two triangles keep the first two (the CUDA
hash keeps an arbitrary two; tests use manifold meshes).
"""
import numpy as np


def build_topology(tri):
    """edge (min, max) -> list of opposing vertices (first two triangles that use the edge, in triangle order)"""
    topo = {}
    for f in range(len(tri)):
        i0, i1, i2 = (int(x) for x in tri[f])
        for a, b, o in ((i0, i1, i2), (i1, i2, i0), (i2, i0, i1)):
            lst = topo.setdefault((min(a, b), max(a, b)), [])
            if len(lst) < 2:
                lst.append(o)
    return topo


def _screen(pos, H, W):
    pos = np.asarray(pos, np.float64)
    w = pos[:, 3]
    ws = np.where(w > 0, w, 1.0)
    return (pos[:, 0] / ws * 0.5 + 0.5) * W, (pos[:, 1] / ws * 0.5 + 0.5) * H, w


def analyze_pair(px, py, d, rast, sx, sy, w, tri, topo):
    """None, or dict(P, Q, dst (flat pixel indices), alpha, va, vb, s, d, g = d t / d (sx[a], sy[a], sx[b], sy[b]))"""
    H, W = rast.shape[:2]
    qx, qy = (px + 1, py) if d == 0 else (px, py + 1)
    if qx >= W or qy >= H:
        return None
    id0, id1 = int(rast[py, px, 3]), int(rast[qy, qx, 3])
    if id0 == id1:
        return None
    if id0 == 0:
        fg = 1
    elif id1 == 0:
        fg = 0
    else:
        fg = 0 if rast[py, px, 2] < rast[qy, qx, 2] else 1
    (Px, Py), (Qx, Qy) = ((px, py), (qx, qy)) if fg == 0 else ((qx, qy), (px, py))
    s = 1.0 if (Qx - Px + Qy - Py) > 0 else -1.0
    f = (id0 if fg == 0 else id1) - 1
    i0, i1, i2 = (int(x) for x in tri[f])
    if w[i0] <= 0 or w[i1] <= 0 or w[i2] <= 0:
        return None
    cx, cy = Px + 0.5, Py + 0.5
    for a, b, o in ((i0, i1, i2), (i1, i2, i0), (i2, i0, i1)):
        ax, ay, bx, by = sx[a] - cx, sy[a] - cy, sx[b] - cx, sy[b] - cy       # relative to P's centre
        if d == 0:
            if (ay < 0) == (by < 0):
                continue
            u = -ay / (by - ay)
            cross = ax + (bx - ax) * u
            t = s * cross
            g = (s * (1 - u), -s * (bx - ax) * (1 - u) / (by - ay), s * u, -s * (bx - ax) * u / (by - ay))
        else:
            if (ax < 0) == (bx < 0):
                continue
            u = -ax / (bx - ax)
            cross = ay + (by - ay) * u
            t = s * cross
            g = (-s * (by - ay) * (1 - u) / (bx - ax), s * (1 - u), -s * (by - ay) * u / (bx - ax), s * u)
        if not (0.0 < t < 1.0):
            continue
        # silhouette test
        lst = list(topo[(min(a, b), max(a, b))])
        lst.remove(o)
        if lst:
            o2 = lst[0]
            if w[o2] <= 0:
                return None
            ex, ey = bx - ax, by - ay
            s1 = ex * (sy[o] - cy - ay) - ey * (sx[o] - cx - ax)
            s2 = ex * (sy[o2] - cy - ay) - ey * (sx[o2] - cx - ax)
            if not (s1 * s2 > 0):
                return None
        alpha = t - 0.5
        P, Q = Py * W + Px, Qy * W + Qx
        return dict(P=P, Q=Q, dst=Q if alpha > 0 else P, alpha=alpha, va=a, vb=b, g=g)
    return None


def pairs(rast, pos, tri, topo=None):
    H, W = rast.shape[:2]
    tri = np.asarray(tri, np.int64)
    topo = topo or build_topology(tri)
    sx, sy, w = _screen(pos, H, W)
    out = []
    for py in range(H):
        for px in range(W):
            for d in (0, 1):
                r = analyze_pair(px, py, d, rast, sx, sy, w, tri, topo)
                if r is not None:
                    out.append(r)
    return out


def antialias(color, rast, pos, tri, topo=None):
    """color [H,W,C], rast [H,W,4], pos [V,4] clip space, tri [F,3] -> [H,W,C] float64"""
    color = np.asarray(color, np.float64)
    H, W, C = color.shape
    flat = color.reshape(-1, C)
    out = flat.copy()
    for r in pairs(np.asarray(rast, np.float64), pos, tri, topo):
        out[r["dst"]] += r["alpha"] * (flat[r["P"]] - flat[r["Q"]])
    return out.reshape(H, W, C)


def antialias_backward(grad_out, color, rast, pos, tri, topo=None, pos_gradient_boost=1.0):
    """-> (grad_color [H,W,C], grad_pos [V,4]) for grad_out [H,W,C]"""
    color = np.asarray(color, np.float64); grad_out = np.asarray(grad_out, np.float64)
    pos = np.asarray(pos, np.float64)
    H, W, C = color.shape
    flat, go = color.reshape(-1, C), grad_out.reshape(-1, C)
    gc = go.copy()
    gp = np.zeros((pos.shape[0], 4))
    for r in pairs(np.asarray(rast, np.float64), pos, tri, topo):
        g = go[r["dst"]]
        gc[r["P"]] += r["alpha"] * g
        gc[r["Q"]] -= r["alpha"] * g
        dt = float(np.dot(g, flat[r["P"]] - flat[r["Q"]])) * pos_gradient_boost
        for v, (gx, gy) in ((r["va"], r["g"][0:2]), (r["vb"], r["g"][2:4])):
            x, y, ww = pos[v, 0], pos[v, 1], pos[v, 3]
            dsx, dsy = dt * gx, dt * gy                    # d loss / d screen x, y of the vertex
            gp[v, 0] += dsx * 0.5 * W / ww
            gp[v, 1] += dsy * 0.5 * H / ww
            gp[v, 3] += -(dsx * 0.5 * W * x + dsy * 0.5 * H * y) / (ww * ww)
    return gc.reshape(H, W, C), gp
