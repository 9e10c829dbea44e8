"""float64 restatement of the two pytorch3d regularisers of the reference's stage-1 loss (nerf/utils.py:759-769), written from their
definitions for one mesh (the reference's `Meshes([v + offsets], [triangles])`):

  mesh_edge_loss(target_length=0)  mean over the unique undirected edges of |v_a - v_b|^2
  mesh_normal_consistency          mean over every unordered pair of faces sharing an edge (a, b), a < b, with opposite vertices c, d
                                   of 1 - cosine_similarity(n_c, -n_d), n_c = (v_b - v_a) x (v_c - v_a), n_d likewise; 0 without pairs

`regularisers` evaluates them with torch ops (torch.cosine_similarity, eps 1e-8), so autograd gives the gradient torch gives;
`closed_form` is the per-pair expression csrc/stage1.cu's k_s1_mesh_reg evaluates (|u + w|^2 / 2 with both norms >= eps, the clamped
branch otherwise) with its hand-derived gradient, in numpy float64."""
from collections import defaultdict

import numpy as np
import torch

EPS = 1e-8


def edge_faces(faces):
    """{(a, b), a < b: [opposite vertex of every face on the edge]} of faces [F,3] (faces with a repeated index are not handled)"""
    out = defaultdict(list)
    for f in np.asarray(faces, np.int64).tolist():
        for e in range(3):
            a, b, o = f[e], f[(e + 1) % 3], f[(e + 2) % 3]
            out[(min(a, b), max(a, b))].append(o)
    return out


def pairs(faces):
    """[K,4] int64 rows (a, b, c, d): every unordered pair of faces on every edge"""
    rows = []
    for (a, b), opp in edge_faces(faces).items():
        for i in range(len(opp)):
            for j in range(i + 1, len(opp)):
                rows.append((a, b, opp[i], opp[j]))
    return np.array(rows, np.int64).reshape(-1, 4)


def regularisers(v, faces):
    """(normal consistency, edge loss) of vertices v [V,3] (a float64 tensor, may require grad) and faces [F,3]"""
    ef = edge_faces(faces)
    e = torch.tensor(sorted(ef), dtype=torch.long, device=v.device).reshape(-1, 2)
    edge = ((v[e[:, 0]] - v[e[:, 1]]) ** 2).sum(1).mean() if e.shape[0] else v.sum() * 0
    p = torch.from_numpy(pairs(faces)).to(v.device)
    if p.shape[0] == 0:
        return v.sum() * 0, edge
    va, vb, vc, vd = (v[p[:, k]] for k in range(4))
    nc = torch.cross(vb - va, vc - va, dim=1)
    nd = torch.cross(vb - va, vd - va, dim=1)
    normal = (1 - torch.cosine_similarity(nc, -nd, dim=1, eps=EPS)).mean()
    return normal, edge


def total(v, faces, lambda_normal, lambda_edgelen):
    normal, edge = regularisers(v, faces)
    return lambda_normal * normal + lambda_edgelen * edge


def loss_and_grad(v, faces, lambda_normal, lambda_edgelen):
    """float64 (loss, d loss / d v [V,3]) by autograd"""
    x = torch.as_tensor(v, dtype=torch.float64).detach().clone().requires_grad_(True)
    loss = total(x, faces, lambda_normal, lambda_edgelen)
    loss.backward()
    return float(loss.detach()), x.grad.detach()


def closed_form(v, faces, lambda_normal, lambda_edgelen):
    """the kernel's per-edge / per-pair expressions and gradient (numpy float64): (loss, grad [V,3])"""
    v = np.asarray(v, np.float64)
    ef = edge_faces(faces)
    E = len(ef)
    pr = pairs(faces)
    P = pr.shape[0]
    wn = lambda_normal / P if P else 0.0
    we = lambda_edgelen / E if E else 0.0
    g = np.zeros_like(v)
    loss = 0.0
    for a, b in ef:
        d = v[b] - v[a]
        loss += we * d @ d
        g[a] -= 2 * we * d
        g[b] += 2 * we * d
    for a, b, c, d in pr.tolist():
        e, qc, qd = v[b] - v[a], v[c] - v[a], v[d] - v[a]
        nc, nd = np.cross(e, qc), np.cross(e, qd)
        lc, ld = np.linalg.norm(nc), np.linalg.norm(nd)
        u, w = nc / max(lc, EPS), nd / max(ld, EPS)
        if lc >= EPS and ld >= EPS:
            s = u + w
            L = 0.5 * s @ s
            gc, gd = (s - L * u) / lc, (s - L * w) / ld
        else:
            dp = u @ w
            L = 1 + dp
            gc = (w - (dp if lc >= EPS else 0.0) * u) / max(lc, EPS)
            gd = (u - (dp if ld >= EPS else 0.0) * w) / max(ld, EPS)
        loss += wn * L
        gc, gd = wn * gc, wn * gd
        ge = np.cross(qc, gc) + np.cross(qd, gd)
        gqc, gqd = np.cross(gc, e), np.cross(gd, e)
        g[b] += ge
        g[c] += gqc
        g[d] += gqd
        g[a] -= ge + gqc + gqd
    return loss, g


# ---- meshes ----
def grid(n=4, z=None):
    """an open (n+1) x (n+1) grid of 2 n^2 triangles in the plane z = 0, or at heights z [(n+1)^2]"""
    xs, ys = np.meshgrid(np.arange(n + 1, dtype=np.float64), np.arange(n + 1, dtype=np.float64), indexing="ij")
    v = np.stack([xs.ravel(), ys.ravel(), np.zeros(xs.size) if z is None else z], 1)
    f = []
    for i in range(n):
        for j in range(n):
            p = i * (n + 1) + j
            f += [[p, p + n + 1, p + n + 2], [p, p + n + 2, p + 1]]
    return v, np.array(f, np.int64)


def cube():
    """the unit cube as 12 consistently oriented triangles: 12 cube edges (90 degrees) and 6 face diagonals (0 degrees)"""
    v = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float64)
    quads = [[0, 1, 3, 2], [4, 6, 7, 5], [0, 4, 5, 1], [2, 3, 7, 6], [0, 2, 6, 4], [1, 5, 7, 3]]
    f = []
    for a, b, c, d in quads:
        f += [[a, b, c], [a, c, d]]
    return v, np.array(f, np.int64)


def hinge(phi):
    """two triangles on the edge (0, 1) bent by phi from flat: normal consistency 1 - cos(phi)"""
    th = np.pi - phi
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0.3, np.cos(th), np.sin(th)]], np.float64)
    return v, np.array([[0, 1, 2], [1, 0, 3]], np.int64)
