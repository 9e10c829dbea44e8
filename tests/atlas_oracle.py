"""numpy restatement of the UV atlas rule of nerf2mesh_b200/texture.py uv_unwrap (csrc/atlas.cu), bit for bit: every float64 step is one
numpy operation on float64 arrays or Python floats (IEEE, one rounding each, no FMA), and every decision is a minimum, a maximum, a count
or a sort, so the order the device's atomics run in does not reach the result.

    vt, ft, vmapping = unwrap(vertices, triangles, resolution, ssaa=2, info=None)
"""
import itertools
import math

import numpy as np

SMALL_CHART, MERGE_ROUNDS, ANGLES, PAD, BISECT_STEPS, MERGE_COS = 8, 3, 16, 2, 24, 0.5


def tables():
    """(axes [26,3], basis [26,6], rot [ANGLES,2]): the 26 directions, a right-handed in-plane basis per direction, (cos, sin) of the angles"""
    dirs = np.array([d for d in itertools.product((-1.0, 0.0, 1.0), repeat=3) if any(d)], np.float64)
    axes = dirs / np.sqrt((dirs * dirs).sum(1))[:, None]
    basis = np.empty((26, 6), np.float64)
    for i, a in enumerate(axes):
        h = np.array([1.0, 0.0, 0.0]) if abs(a[2]) == 1.0 else np.array([0.0, 0.0, 1.0])
        e1 = np.cross(h, a)
        e1 = e1 / np.sqrt(e1 @ e1)
        basis[i, :3], basis[i, 3:] = e1, np.cross(a, e1)
    t = np.arange(ANGLES, dtype=np.float64) * (math.pi / 2) / ANGLES
    return axes, basis, np.stack([np.cos(t), np.sin(t)], 1)


def dot3(x, y):
    """(x0 y0 + x1 y1) + x2 y2 along the last axis, as the kernels' dot3"""
    return (x[..., 0] * y[..., 0] + x[..., 1] * y[..., 1]) + x[..., 2] * y[..., 2]


def faces(v, f, axes):
    """1. -> (unit normals [F,3], bucket [F] (-1: degenerate))"""
    p = v.astype(np.float64)[f]
    e1, e2 = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    ln = np.sqrt(dot3(n, n))
    deg = (f[:, 0] == f[:, 1]) | (f[:, 1] == f[:, 2]) | (f[:, 0] == f[:, 2]) | ~(ln > 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        u = n / np.where(deg, 1.0, ln)[:, None]
    u[deg] = 0.0
    bucket = np.argmax(dot3(u[:, None, :], axes[None, :, :]), axis=1).astype(np.int64)       # first maximum: the lowest index
    bucket[deg] = -1
    return u, bucket


def mates(f, keep):
    """mate [3F]: the other face-edge of an edge with exactly two face-edges among the kept faces, -1 elsewhere"""
    F = len(f)
    e = np.arange(3 * F)
    a, b = f.reshape(-1), np.roll(f, -1, axis=1).reshape(-1)
    live = keep[e // 3]
    key = np.minimum(a, b).astype(np.int64) << 32 | np.maximum(a, b)
    el, kl = e[live], key[live]
    o = np.lexsort((el, kl))
    el, kl = el[o], kl[o]
    _, first, cnt = np.unique(kl, return_index=True, return_counts=True)
    two = first[cnt == 2]
    mate = np.full(3 * F, -1, np.int64)
    mate[el[two]], mate[el[two + 1]] = el[two + 1], el[two]
    return mate


def components(F, pairs):
    """label [F] = the lowest face of each connected component of the pairs"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    g = coo_matrix((np.ones(len(pairs)), (pairs[:, 0], pairs[:, 1])), shape=(F, F)) if len(pairs) else coo_matrix((F, F))
    _, comp = connected_components(g, directed=False)
    low = np.full(F, F, np.int64)
    np.minimum.at(low, comp, np.arange(F))
    return low[comp]


def merge_round(label, fax, nrm, bucket, mate, axes):
    """3. one round -> (label, fax)"""
    F = len(label)
    count = np.bincount(label, minlength=F)
    e = np.nonzero(mate >= 0)[0]
    a, b = label[e // 3], label[mate[e] // 3]
    sel = (a != b) & (count[a] < SMALL_CHART) & (bucket[a] >= 0)
    a, b = a[sel], b[sel]
    propose = np.full(F, -1, np.int64)
    if len(a):
        pairs, cnt = np.unique(np.stack([a, b], 1), axis=0, return_counts=True)
        o = np.lexsort((pairs[:, 1], -cnt, pairs[:, 0]))                    # per chart: most shared edges, then the lowest id
        pairs = pairs[o]
        first = np.r_[True, pairs[1:, 0] != pairs[:-1, 0]]
        best = np.full(F, -1, np.int64)
        best[pairs[first, 0]] = pairs[first, 1]
        fb = best[label]
        ok = np.ones(F, bool)
        has = fb >= 0
        ok[has] = dot3(nrm[has], axes[fax[fb[has]]]) >= MERGE_COS
        bad = np.zeros(F, bool)
        bad[label[~ok]] = True
        good = (best >= 0) & ~bad
        propose[good] = best[good]
    tb = propose[label]
    acc = (tb >= 0) & (propose[np.maximum(tb, 0)] < 0)
    label, fax0 = label.copy(), fax.copy()
    label[acc] = tb[acc]
    fax = fax0.copy()
    fax[acc] = fax0[tb[acc]]
    return label, fax


def chart_index(label):
    F = len(label)
    incl = np.cumsum(label == np.arange(F))
    return incl[label] - 1, int(incl[-1])


def rotated(p, B, rot):
    """[n,3] points, [n,6] bases -> x, y [n,K] before the turn"""
    u, w = dot3(p, B[:, :3]), dot3(p, B[:, 3:])
    c, s = rot[:, 0][None, :], rot[:, 1][None, :]
    return c * u[:, None] - s * w[:, None], s * u[:, None] + c * w[:, None]


def dkey(x):
    """float64 -> uint64 in value order, -0 below +0 (the kernels' min / max order)"""
    u = np.ascontiguousarray(x, np.float64).view(np.uint64)
    return np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))


def dkey_inv(k):
    return np.where(k >> np.uint64(63), k & np.uint64((1 << 63) - 1), ~k).view(np.float64)


def orient(v, f, ci, C, fax, basis, rot):
    """4. -> (angle k [C], turn [C], org [C,2], ext [C,2])"""
    e = np.arange(3 * len(f))
    x, y = rotated(v.astype(np.float64)[f.reshape(-1)], basis[fax[e // 3]], rot)
    c = ci[e // 3]
    o = np.argsort(c, kind="stable")
    starts = np.r_[0, np.nonzero(np.diff(c[o]))[0] + 1]
    kx, ky = dkey(x[o]), dkey(y[o])
    x0, x1 = dkey_inv(np.minimum.reduceat(kx, starts)), dkey_inv(np.maximum.reduceat(kx, starts))
    y0, y1 = dkey_inv(np.minimum.reduceat(ky, starts)), dkey_inv(np.maximum.reduceat(ky, starts))
    k = np.argmin((x1 - x0) * (y1 - y0), axis=1)
    r = np.arange(C)
    x0, x1, y0, y1 = x0[r, k], x1[r, k], y0[r, k], y1[r, k]
    w, h = x1 - x0, y1 - y0
    turn = h > w
    org = np.stack([np.where(turn, -y1, x0), np.where(turn, x0, y0)], 1)
    ext = np.stack([np.where(turn, h, w), np.where(turn, w, h)], 1)
    return k, turn, org, ext


def layout(W, H, s, res, pad=PAD):
    """next-fit decreasing height over charts already in order -> offsets [C,2] or None"""
    w = np.maximum(1, np.ceil(s * W)).astype(np.int64)
    h = np.maximum(1, np.ceil(s * H)).astype(np.int64)
    P = np.r_[0, np.cumsum(w + pad)]
    nxt = np.searchsorted(P, P[:-1] + (res - pad), side="right") - 1
    off = np.zeros((len(W), 2), np.int64)
    a, y = 0, pad
    while a < len(W):
        e = int(nxt[a])
        if e == a or y + h[a] + pad > res:
            return None
        off[a:e, 0] = pad + P[a:e] - P[a]
        off[a:e, 1] = y
        y += int(h[a]) + pad
        a = e
    return off


def pack(ext, res):
    """5. -> (s, off [C,2]) or raise ValueError"""
    C = len(ext)
    order = np.lexsort((np.arange(C), -ext[:, 1]))
    W, H = ext[order, 0], ext[order, 1]
    m = float(ext[:, 0].max())
    hi = float(res - 2 * PAD) / m if m > 0 else float(res)
    lo = hi * 2.0 ** -20
    if layout(W, H, lo, res) is None:
        raise ValueError(f"{C} charts do not fit")
    if layout(W, H, hi, res) is not None:
        lo = hi
    else:
        for _ in range(BISECT_STEPS):
            mid = math.sqrt(lo * hi)
            if layout(W, H, mid, res) is not None:
                lo = mid
            else:
                hi = mid
    off = np.empty((C, 2), np.int64)
    off[order] = layout(W, H, lo, res)
    return lo, off


def corner_vt(p, B, rot_k, turn, org, off, s, res):
    """vt [n,2] float32 of points p [n,3] float64 in their charts"""
    u, w = dot3(p, B[:, :3]), dot3(p, B[:, 3:])
    c, sn = rot_k[:, 0], rot_k[:, 1]
    x, y = c * u - sn * w, sn * u + c * w
    x, y = np.where(turn, -y, x), np.where(turn, x, y)
    return np.stack([(off[:, 0] + s * (x - org[:, 0])) / float(res), (off[:, 1] + s * (y - org[:, 1])) / float(res)], 1).astype(np.float32)


def face_vt(v, f, ci, fax, basis, rot, k, turn, org, off, s, res):
    c = np.repeat(ci, 3)
    return corner_vt(v.astype(np.float64)[f.reshape(-1)], basis[np.repeat(fax, 3)], rot[k[c]], turn[c], org[c], off[c], s, res).reshape(-1, 3, 2)


def inside_pairs(fvt, faces_idx, R, chunk=1 << 22):
    """(face, texel) for every bake-raster texel centre strictly inside a face (float64 edge functions > 0), in chunks"""
    P = fvt.astype(np.float64) * R
    x0, x1 = P[:, :, 0].min(1), P[:, :, 0].max(1)
    y0, y1 = P[:, :, 1].min(1), P[:, :, 1].max(1)
    i0 = np.maximum(0, np.ceil(x0 - 0.5)).astype(np.int64); i1 = np.minimum(R - 1, np.floor(x1 - 0.5)).astype(np.int64)
    j0 = np.maximum(0, np.ceil(y0 - 0.5)).astype(np.int64); j1 = np.minimum(R - 1, np.floor(y1 - 0.5)).astype(np.int64)
    nw, nh = np.maximum(0, i1 - i0 + 1), np.maximum(0, j1 - j0 + 1)
    n = nw * nh
    fs, ts = [], []
    start = 0
    cum = np.cumsum(n)
    while start < len(n):
        stop = int(np.searchsorted(cum, (cum[start - 1] if start else 0) + chunk, side="right"))
        stop = max(stop, start + 1)
        idx = np.arange(start, stop)
        cnt = n[idx]
        fi = np.repeat(idx, cnt)
        q = np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        i = i0[fi] + q % nw[fi]
        j = j0[fi] + q // nw[fi]
        px, py = i + 0.5, j + 0.5
        A, B, Cc = P[fi, 0], P[fi, 1], P[fi, 2]

        def edge(a, b):
            return (b[:, 0] - a[:, 0]) * (py - a[:, 1]) - (b[:, 1] - a[:, 1]) * (px - a[:, 0])
        ins = (edge(A, B) > 0) & (edge(B, Cc) > 0) & (edge(Cc, A) > 0)
        fs.append(faces_idx[fi[ins]]); ts.append(j[ins] * R + i[ins])
        start = stop
    return (np.concatenate(fs), np.concatenate(ts)) if fs else (np.zeros(0, np.int64), np.zeros(0, np.int64))


def conflicts(fvt, keep, R):
    """6. -> (faces over a texel centre a lower face also covers strictly, one entry per such pair)"""
    idx = np.nonzero(keep)[0]
    fs, ts = inside_pairs(fvt[idx], idx, R)
    if len(ts) == 0:
        return fs
    o = np.lexsort((fs, ts))
    fs, ts = fs[o], ts[o]
    first = np.r_[True, ts[1:] != ts[:-1]]
    owner = fs[np.maximum.accumulate(np.where(first, np.arange(len(ts)), 0))]
    return fs[owner != fs]


def unwrap(v, f, resolution, ssaa=2, info=None, trace=None):
    """-> (vt [Nt,2] float32, ft [F,3] int64, vmapping [Nt] int64); `trace` (a list) receives the chart count of every packing"""
    v = np.asarray(v, np.float32); f = np.asarray(f, np.int64).reshape(-1, 3)
    F, R = len(f), int(resolution) * int(ssaa)
    if F == 0:
        if info is not None:
            info.update(charts=0, texels_per_unit=0.0, utilization=0.0, split_rounds=0)
        return np.zeros((0, 2), np.float32), np.zeros((0, 3), np.int64), np.zeros(0, np.int64)
    axes, basis, rot = tables()
    nrm, bucket = faces(v, f, axes)
    keep = bucket >= 0
    mate = mates(f, keep)
    e = np.nonzero(mate >= 0)[0]
    g = mate[e] // 3
    same = bucket[e // 3] == bucket[g]
    base = components(F, np.stack([e[same] // 3, g[same]], 1))
    label, fax = base.copy(), np.maximum(bucket, 0)
    for _ in range(MERGE_ROUNDS):
        label, fax = merge_round(label, fax, nrm, bucket, mate, axes)
    splits = 0
    while True:
        ci, C = chart_index(label)
        if trace is not None:
            trace.append(C)
        k, turn, org, ext = orient(v, f, ci, C, fax, basis, rot)
        s, off = pack(ext, resolution)
        fvt = face_vt(v, f, ci, fax, basis, rot, k, turn, org, off, s, resolution)
        bad = conflicts(fvt, keep, R)
        if len(bad) == 0:
            break
        conf = np.zeros(C, bool); conf[ci[bad]] = True
        merged = np.zeros(C, bool); merged[ci[base != label]] = True
        hit = conf[ci]
        label = np.where(hit, np.where(merged[ci], base, np.arange(F)), label)
        fax = np.where(hit, np.maximum(bucket, 0), fax)
        splits += 1
    keys = ci.repeat(3).astype(np.int64) << 32 | f.reshape(-1)
    uk, first, inv = np.unique(keys, return_index=True, return_inverse=True)
    ft = inv.reshape(F, 3).astype(np.int64)
    vt = fvt.reshape(-1, 2)[first]
    if info is not None:
        info.update(charts=C, texels_per_unit=s, utilization=uv_area(vt, ft), split_rounds=splits)
    return vt, ft, (uk & 0xFFFFFFFF).astype(np.int64)


def uv_area(vt, ft):
    t = np.asarray(vt, np.float64)[np.asarray(ft)]
    d1, d2 = t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]
    return float(np.abs(0.5 * (d1[:, 0] * d2[:, 1] - d1[:, 1] * d2[:, 0])).sum())
