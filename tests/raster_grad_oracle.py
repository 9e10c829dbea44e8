"""float64 restatement of the gradients of dr.rasterize and dr.interpolate (csrc/raster_grad.cuh) and of contract()'s backward
(n2m_common.cuh: contract_linf_backward), for the CPU tests and the GPU tests of the colour-field vertex gradient.

rast (u, v) at pixel NDC (X, Y) of a triangle with clip-space vertices p_k = (x_k, y_k, z_k, w_k): with p'_k = (x_k - X w_k, y_k - Y w_k)
and the edge functions a_k = p'_{k+1} x p'_{k+2}, u = a_0 / sum a, v = a_1 / sum a -- the perspective-correct barycentrics in 2-D
homogeneous form, for triangles in front of the camera and for triangles that cross it."""
import numpy as np


def _cross(a, b):
    return a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]


def pixel_ndc(x, y, H, W):
    return (x + 0.5) / W * 2.0 - 1.0, (y + 0.5) / H * 2.0 - 1.0


def uv(P, X, Y):
    """closed-form (u, v) of the triangle P [3,4] (float64 clip space) at NDC (X, Y)"""
    P = np.asarray(P, np.float64)
    q = P[:, :2] - np.array([X, Y]) * P[:, 3:4]
    a = np.array([_cross(q[1], q[2]), _cross(q[2], q[0]), _cross(q[0], q[1])])
    return a[0] / a.sum(), a[1] / a.sum()


def rasterize_backward(P, X, Y, du, dv):
    """d loss / d P [3,4] from d loss / d (u, v), the arithmetic of rasterize_uv_backward; column 2 (clip z) is zero"""
    P = np.asarray(P, np.float64)
    q = P[:, :2] - np.array([X, Y]) * P[:, 3:4]
    a = np.array([_cross(q[(k + 1) % 3], q[(k + 2) % 3]) for k in range(3)])
    s = a.sum()
    G = du * a[0] / s + dv * a[1] / s
    ga = np.array([du - G, dv - G, -G]) / s
    g = np.zeros((3, 4))
    for k in range(3):
        k1, k2 = (k + 1) % 3, (k + 2) % 3
        gx = ga[k2] * q[k1, 1] - ga[k1] * q[k2, 1]
        gy = ga[k1] * q[k2, 0] - ga[k2] * q[k1, 0]
        g[k] = (gx, gy, 0.0, -(X * gx + Y * gy))
    return g


def interpolate_backward_rast(g, a0, a1, a2):
    """d loss / d (u, v) of out = u a0 + v a1 + (1 - u - v) a2 from d loss / d out = g (vectors over the attributes)"""
    g, a0, a1, a2 = (np.asarray(t, np.float64) for t in (g, a0, a1, a2))
    return float(np.dot(g, a0 - a2)), float(np.dot(g, a1 - a2))


def contract_backward(x, g):
    """J(x)^T g of contract() (renderer.py:25-32) at the uncontracted point x, ties of |x_k| split evenly (torch's amax backward)"""
    x, g = np.asarray(x, np.float64), np.asarray(g, np.float64)
    ax = np.abs(x)
    m = ax.max()
    if not m > 1:
        return g.copy()
    s = (2 - 1 / m) / m
    ds = 2 * (1 - m) / m ** 3
    tie = ax == m
    dm = np.where(tie, np.sign(x) / tie.sum(), 0.0)
    return s * g + np.dot(g, x) * ds * dm
