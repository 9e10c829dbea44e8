"""Test infrastructure, not product: a numpy / scipy restatement of the parallel quadric edge collapse of csrc/decimate.cu, the checker of
those kernels, and a plain sequential greedy collapse with the same quadrics, validity and placement as a quality yardstick.

    decimate(v, f, target, optimal_placement=True, info=None)    the library's rule, round by round (bit-exact with the kernels)
    decimate_greedy(v, f, target, optimal_placement=True)        one collapse at a time, cheapest key first, from a heap

Vertices are float32 [V,3], faces int [F,3]; results are float32 / int32.  Every float64 value the kernels compute is written out here
in the kernels' order, one rounded operation at a time (numpy does not contract a * b + c into an FMA, and the kernels use the explicit
__d*_rn intrinsics); no pairwise np.sum touches a value that must be bit-exact.  The rule is the library's reading of pymeshlab's
meshing_decimation_quadric_edge_collapse (VCG) with its defaults; pymeshlab is not run, so agreement with it is not claimed.

Validity adds one check to the link condition of an edge with one face: the collapse may not delete a lone triangle (a face whose three
edges are all boundary edges), which would remove a component and change the Euler characteristic."""
import heapq

import numpy as np
from scipy.sparse import coo_matrix

DET_REL = 1e-6          # the solve is taken when det(A) > DET_REL * trace(A)^3 (every eigenvalue of A above DET_REL * trace)
NONE = np.uint64(0xFFFFFFFFFFFFFFFF)


def fkey(x):
    """float32 -> u32 key whose unsigned order is the float order"""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000).astype(np.uint64)


def _cross(pa, pb, pc):
    """float64 cross(b - a, c - a), one rounding per operation (meshclean.cu's face_cross)"""
    e1, e2 = pb - pa, pc - pa
    return (e1[..., 1] * e2[..., 2] - e1[..., 2] * e2[..., 1],
            e1[..., 2] * e2[..., 0] - e1[..., 0] * e2[..., 2],
            e1[..., 0] * e2[..., 1] - e1[..., 1] * e2[..., 0])


def face_quadrics(p, tri):
    """[n,10] float64 plane quadrics (a00 a01 a02 a11 a12 a22 b0 b1 b2 c) of the faces tri [n,3] over positions p [V,3] float32:
    unit normal u = cross / |cross| with |cross| = sqrt((x*x + y*y) + z*z), d = -((ux*ax + uy*ay) + uz*az), K = [u u^T, d u, d^2];
    a face whose |cross| is 0 gives the zero quadric"""
    q = np.asarray(p, np.float64)
    a, b, c = q[tri[:, 0]], q[tri[:, 1]], q[tri[:, 2]]
    nx, ny, nz = _cross(a, b, c)
    ln = np.sqrt((nx * nx + ny * ny) + nz * nz)
    ok = ln > 0
    s = np.where(ok, ln, 1.0)
    ux, uy, uz = nx / s, ny / s, nz / s
    d = -((ux * a[:, 0] + uy * a[:, 1]) + uz * a[:, 2])
    K = np.stack([ux * ux, ux * uy, ux * uz, uy * uy, uy * uz, uz * uz, d * ux, d * uy, d * uz, d * d], 1)
    K[~ok] = 0.0
    return K


def vertex_quadrics(p, tri, fkeep):
    """Q_v = the sum of K_f over the live faces containing v, in ascending face index, left to right, from +0"""
    fid = np.nonzero(fkeep)[0]
    K = face_quadrics(p, tri[fid])
    vert = tri[fid].reshape(-1)
    face = np.repeat(np.arange(len(fid)), 3)
    order = np.lexsort((face, vert))                          # face index order within each vertex (fid ascending = face ascending)
    vert, face = vert[order], face[order]
    first = np.searchsorted(vert, vert, "left")
    rank = np.arange(len(vert)) - first
    Q = np.zeros((len(p), 10))
    for r in range(int(rank.max()) + 1 if len(rank) else 0):
        m = rank == r
        Q[vert[m]] = Q[vert[m]] + K[face[m]]
    return Q


def quadric_cost(Q, x, y, z):
    """x^T A x + 2 b.x + c as ((((x*Ax + y*Ay) + z*Az) + 2*bx) + c), Ax = (a00*x + a01*y) + a02*z, ..., bx = (b0*x + b1*y) + b2*z"""
    a00, a01, a02, a11, a12, a22, b0, b1, b2, c = (Q[..., i] for i in range(10))
    Ax = (a00 * x + a01 * y) + a02 * z
    Ay = (a01 * x + a11 * y) + a12 * z
    Az = (a02 * x + a12 * y) + a22 * z
    bx = (b0 * x + b1 * y) + b2 * z
    return (((x * Ax + y * Ay) + z * Az) + 2.0 * bx) + c


def placement(Q, pa, pb, optimal):
    """the merged vertex's float32 position and the float64 cost there, for quadrics Q [n,10] and endpoints pa, pb [n,3] float32 (pa the
    lower index).  optimal: A p = -b by cofactors when det > DET_REL * tr^3, else the cheapest of pa, pb, midpoint (ties in that order);
    not optimal: the midpoint (pa + pb) * 0.5 in float64.  Every candidate is rounded once to float32 and costed there."""
    a64, b64 = pa.astype(np.float64), pb.astype(np.float64)
    mid = ((a64 + b64) * 0.5).astype(np.float32)

    def cost(p32):
        p = p32.astype(np.float64)
        return quadric_cost(Q, p[:, 0], p[:, 1], p[:, 2])

    cm = cost(mid)
    if not optimal:
        return mid, cm
    a00, a01, a02, a11, a12, a22, b0, b1, b2 = (Q[:, i] for i in range(9))
    C00 = a11 * a22 - a12 * a12
    C01 = a02 * a12 - a01 * a22
    C02 = a01 * a12 - a11 * a02
    C11 = a00 * a22 - a02 * a02
    C12 = a01 * a02 - a00 * a12
    C22 = a00 * a11 - a01 * a01
    det = (a00 * C00 + a01 * C01) + a02 * C02
    tr = (a00 + a11) + a22
    ok = det > DET_REL * ((tr * tr) * tr)
    s = np.where(ok, det, 1.0)
    opt = np.stack([-(((C00 * b0 + C01 * b1) + C02 * b2) / s),
                    -(((C01 * b0 + C11 * b1) + C12 * b2) / s),
                    -(((C02 * b0 + C12 * b1) + C22 * b2) / s)], 1)
    opt = np.where(ok[:, None], opt, 0.0).astype(np.float32)
    ca, cb, co = cost(pa), cost(pb), cost(opt)
    best, cbest = pa.copy(), ca.copy()
    m = cb < cbest
    best[m], cbest[m] = pb[m], cb[m]
    m = cm < cbest
    best[m], cbest[m] = mid[m], cm[m]
    best[ok], cbest[ok] = opt[ok], co[ok]
    return best, cbest


def _csr(tri, fid, V):
    """vertex -> live face lists: (start [V+1], faces)"""
    vert = tri[fid].reshape(-1)
    order = np.argsort(vert, kind="stable")
    start = np.zeros(V + 1, np.int64)
    np.cumsum(np.bincount(vert, minlength=V), out=start[1:])
    return start, np.repeat(fid, 3)[order]


def _gather(start, faces, verts):
    """for every entry of verts: its faces, flattened, with the entry's index"""
    n = start[verts + 1] - start[verts]
    owner = np.repeat(np.arange(len(verts)), n)
    base = np.repeat(start[verts] - np.concatenate([[0], np.cumsum(n)[:-1]]), n)
    return owner, faces[base + np.arange(int(n.sum()))]


def evaluate(P, Q, tri, fkeep, optimal):
    """every edge of the live faces: (lo, hi, edge id, face count, key, position); key = NONE where the collapse is not valid"""
    V = len(P)
    fid = np.nonzero(fkeep)[0]
    T = tri[fid]
    e = (3 * fid[:, None] + np.arange(3)).reshape(-1)
    x, y = T.reshape(-1), np.roll(T, -1, axis=1).reshape(-1)
    lo, hi = np.minimum(x, y), np.maximum(x, y)
    _, first, inv, cnt = np.unique(lo * V + hi, return_index=True, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    eid = np.full(len(cnt), np.iinfo(np.int64).max); np.minimum.at(eid, inv, e)
    emax = np.full(len(cnt), -1); np.maximum.at(emax, inv, e)
    lo, hi = lo[first], hi[first]
    n = len(cnt)
    opp = lambda ee: tri[ee // 3, (ee % 3 + 2) % 3]
    c = opp(eid)
    d = np.where(cnt == 2, opp(emax), -1)
    cand = (cnt == 1) | (cnt == 2)
    # link condition: the common neighbours of lo and hi are exactly the opposite vertices
    pairs = np.stack([T[:, [0, 1, 2, 1, 2, 0]].reshape(-1), T[:, [1, 2, 0, 0, 1, 2]].reshape(-1)])
    A = coo_matrix((np.ones(pairs.shape[1]), (pairs[0], pairs[1])), shape=(V, V)).tocsr()
    A.data[:] = 1.0
    common = np.asarray((A @ A)[lo, hi]).reshape(-1)
    nopp = np.where(cnt == 2, np.where(c == d, 1, 2), 1)
    valid = cand & (common == nopp)
    # boundary: an interior edge may not join two boundary vertices, a boundary edge may not take the last face of a lone triangle
    bnd = np.zeros(V, bool)
    bnd[lo[cnt == 1]] = True; bnd[hi[cnt == 1]] = True
    valid &= (cnt == 1) | ~(bnd[lo] & bnd[hi])
    ecnt = np.zeros(3 * len(tri), np.int64)
    ecnt[e] = cnt[inv]
    f0, k0 = eid // 3, eid % 3
    lone = (ecnt[3 * f0 + (k0 + 1) % 3] == 1) & (ecnt[3 * f0 + (k0 + 2) % 3] == 1)
    valid &= ~((cnt == 1) & lone)
    # tetrahedron
    s = np.sort(T, 1)
    fk = set(((s[:, 0] * V + s[:, 1]) * V + s[:, 2]).tolist())

    def has(u, w, z):
        t = np.sort(np.stack([u, w, z], 1), 1)
        return np.array([k in fk for k in ((t[:, 0] * V + t[:, 1]) * V + t[:, 2]).tolist()], bool)

    two = np.nonzero(valid & (cnt == 2))[0]
    if len(two):
        tet = has(lo[two], c[two], d[two]) & has(hi[two], c[two], d[two])
        valid[two[tet]] = False
    # placement and cost
    Qs = Q[lo] + Q[hi]
    pos, cost = placement(Qs, P[lo], P[hi], optimal)
    # flip / degeneracy of the surviving faces around lo and hi
    start, faces = _csr(tri, fid, V)
    idx = np.nonzero(valid)[0]
    ends = np.concatenate([lo[idx], hi[idx]])
    owner, g = _gather(start, faces, ends)
    edge = np.concatenate([idx, idx])[owner]
    moved = ends[owner]
    G = tri[g]
    both = ((G == lo[edge][:, None]).any(1)) & ((G == hi[edge][:, None]).any(1))
    edge, moved, G = edge[~both], moved[~both], G[~both]
    p64 = P.astype(np.float64)
    old = p64[G]
    new = old.copy()
    k = G == moved[:, None]
    new[k] = pos[edge].astype(np.float64)             # one corner per face is the moved endpoint
    n0 = _cross(old[:, 0], old[:, 1], old[:, 2])
    n1 = _cross(new[:, 0], new[:, 1], new[:, 2])
    dot = (n0[0] * n1[0] + n0[1] * n1[1]) + n0[2] * n1[2]
    bad = np.zeros(n, bool)
    bad[edge[dot <= 0]] = True
    valid &= ~bad
    key = np.where(valid, (fkey(cost.astype(np.float32)) << np.uint64(32)) | eid.astype(np.uint64), NONE)
    return lo, hi, eid, cnt, key, pos


def budget_threshold(key, cnt, need):
    """K*: the least key at which the valid edges in key order, each weighted by its face count, reach `need`; every valid key when they
    do not"""
    m = key != NONE
    if not m.any():
        return None
    order = np.argsort(key[m])
    ks, cum = key[m][order], np.cumsum(cnt[m][order])
    if cum[-1] < need:
        return ks[-1]
    return ks[np.searchsorted(cum, need, "left")]


def _round(P, Q, tri, fkeep, flive, target, optimal, trace=None):
    lo, hi, eid, cnt, key, pos = evaluate(P, Q, tri, fkeep, optimal)
    K = budget_threshold(key, cnt, flive - target)
    if K is None:
        return 0, 0
    elig = (key != NONE) & (key <= K)
    V = len(P)
    vmin = np.full(V, NONE)
    np.minimum.at(vmin, lo[elig], key[elig]); np.minimum.at(vmin, hi[elig], key[elig])
    T = tri[fkeep]
    r1 = vmin.copy()
    for i in range(3):
        for j in range(3):
            np.minimum.at(r1, T[:, i], vmin[T[:, j]])
    sel = elig & (key == r1[lo]) & (key == r1[hi])
    if trace is not None:
        trace.append(dict(key=key, eid=eid, lo=lo, hi=hi, K=K, selected=eid[sel]))
    a, b = lo[sel], hi[sel]
    Q[a] = Q[a] + Q[b]
    P[a] = pos[sel]
    t = np.arange(V)
    t[b] = a
    live = np.nonzero(fkeep)[0]
    tri[live] = t[tri[live]]
    L = tri[live]
    fkeep[live[(L[:, 0] == L[:, 1]) | (L[:, 1] == L[:, 2]) | (L[:, 0] == L[:, 2])]] = False
    return int(sel.sum()), int(cnt[sel].sum())


def compact(v, f, fkeep):
    f = f[fkeep]
    vkeep = np.zeros(len(v), bool)
    vkeep[f.reshape(-1)] = True
    new = np.cumsum(vkeep) - 1
    return v[vkeep], new[f].reshape(-1, 3)


def _start(v, f, target):
    if target < 1:
        raise ValueError("decimate: target must be at least 1")
    v = np.asarray(v, np.float32).reshape(-1, 3).copy()
    f = np.asarray(f, np.int64).reshape(-1, 3).copy()
    fkeep = (f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])
    return v, f, fkeep


def decimate(v, f, target, optimal_placement=True, info=None, trace=None):
    """the library's rule (nerf2mesh_b200/mesh.py decimate_mesh): rounds while live faces > target; `info` gets rounds, stalled and the
    live faces after each round; `trace` (a list) gets each round's keys, K* and selected edge ids"""
    v, f, fkeep = _start(v, f, target)
    info = {} if info is None else info
    info.update(rounds=0, stalled=False, faces=[])
    if len(f) <= target:
        out_v, out_f = compact(v, f, np.ones(len(f), bool))
        return out_v.astype(np.float32), out_f.astype(np.int32)
    Q = vertex_quadrics(v, f, fkeep)
    flive = int(fkeep.sum())
    while flive > target:
        nsel, removed = _round(v, Q, f, fkeep, flive, target, optimal_placement, trace)
        if nsel == 0:
            info["stalled"] = True
            break
        flive -= removed
        assert flive == int(fkeep.sum())
        info["rounds"] += 1
        info["faces"].append(flive)
    out_v, out_f = compact(v, f, fkeep)
    return out_v.astype(np.float32), out_f.astype(np.int32)


# ---- the sequential yardstick --------------------------------------------------------------------------------------------------------
def decimate_greedy(v, f, target, optimal_placement=True):
    """one valid collapse at a time, the least key first (a heap; an entry is re-checked when popped), with the same quadrics, validity,
    placement and key as `decimate`.  After a collapse the edges at the survivor are re-keyed.  Quality yardstick only."""
    v, f, fkeep = _start(v, f, target)
    if len(f) <= target:
        out_v, out_f = compact(v, f, np.ones(len(f), bool))
        return out_v.astype(np.float32), out_f.astype(np.int32)
    Q = vertex_quadrics(v, f, fkeep).tolist()                # plain Python floats and lists from here: scalar IEEE doubles, no FMA
    P = v.astype(np.float64).tolist()
    T = f.tolist()
    vf = [set() for _ in range(len(v))]
    for i in np.nonzero(fkeep)[0].tolist():
        for x in T[i]:
            vf[x].add(i)
    flive = int(fkeep.sum())
    f32 = lambda x: float(np.float32(x))

    def nbrs(x):
        return {w for g in vf[x] for w in T[g]} - {x}

    def boundary(x):
        seen = {}
        for g in vf[x]:
            for w in T[g]:
                if w != x:
                    seen[w] = seen.get(w, 0) + 1
        return any(n == 1 for n in seen.values())

    def cross(p, q, r):
        e1 = (q[0] - p[0], q[1] - p[1], q[2] - p[2]); e2 = (r[0] - p[0], r[1] - p[1], r[2] - p[2])
        return (e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0])

    def cost(q, p):
        x, y, z = p
        Ax = (q[0] * x + q[1] * y) + q[2] * z
        Ay = (q[1] * x + q[3] * y) + q[4] * z
        Az = (q[2] * x + q[4] * y) + q[5] * z
        bx = (q[6] * x + q[7] * y) + q[8] * z
        return (((x * Ax + y * Ay) + z * Az) + 2.0 * bx) + q[9]

    def place(q, pa, pb):
        """`placement` for one edge, in scalars"""
        mid = [f32((pa[i] + pb[i]) * 0.5) for i in range(3)]
        if not optimal_placement:
            return mid, cost(q, mid)
        a00, a01, a02, a11, a12, a22, b0, b1, b2 = q[:9]
        C00 = a11 * a22 - a12 * a12
        C01 = a02 * a12 - a01 * a22
        C02 = a01 * a12 - a11 * a02
        det = (a00 * C00 + a01 * C01) + a02 * C02
        tr = (a00 + a11) + a22
        if det > DET_REL * ((tr * tr) * tr):
            C11 = a00 * a22 - a02 * a02
            C12 = a01 * a02 - a00 * a12
            C22 = a00 * a11 - a01 * a01
            p = [f32(-(((C00 * b0 + C01 * b1) + C02 * b2) / det)), f32(-(((C01 * b0 + C11 * b1) + C12 * b2) / det)),
                 f32(-(((C02 * b0 + C12 * b1) + C22 * b2) / det))]
            return p, cost(q, p)
        best, cb = pa, cost(q, pa)
        for c in (pb, mid):
            cc = cost(q, c)
            if cc < cb:
                best, cb = c, cc
        return list(best), cb

    def valid(a, b, p):
        """the validity of collapsing (a, b) to p on the current mesh"""
        shared = vf[a] & vf[b]
        if len(shared) not in (1, 2):
            return False
        opp = {w for g in shared for w in T[g]} - {a, b}
        if nbrs(a) & nbrs(b) != opp:
            return False
        if len(shared) == 2 and boundary(a) and boundary(b):
            return False
        if len(shared) == 1 and all(len(vf[x] & vf[w]) == 1 for x in (a, b) for w in opp):
            return False
        if len(shared) == 2 and len(opp) == 2:
            c, d = opp
            if any(set(T[g]) == {a, c, d} for g in vf[a]) and any(set(T[g]) == {b, c, d} for g in vf[b]):
                return False
        for x in (a, b):
            for g in vf[x] - shared:
                old = [P[w] for w in T[g]]
                n0, n1 = cross(*old), cross(*[p if w == x else P[w] for w in T[g]])
                if (n0[0] * n1[0] + n0[1] * n1[1]) + n0[2] * n1[2] <= 0:
                    return False
        return True

    heap, cur = [], {}

    def push(edges):
        """key every valid edge; the entry keeps the position, which changes only with Q or P at an end (and then the edge is re-keyed)"""
        for a, b in edges:
            q = [Q[a][i] + Q[b][i] for i in range(10)]
            p, c = place(q, P[a], P[b])
            if valid(a, b, p):
                k = int(fkey(np.float32(c))) << 32
                cur[(a, b)] = (k, p)
                heapq.heappush(heap, (k, (a, b)))

    push({(min(x, y), max(x, y)) for g in np.nonzero(fkeep)[0].tolist() for x, y in zip(T[g], T[g][1:] + T[g][:1])})
    while flive > target and heap:
        k, (a, b) = heapq.heappop(heap)
        entry = cur.get((a, b))
        if entry is None or entry[0] != k:
            continue
        del cur[(a, b)]
        p = entry[1]
        if not valid(a, b, p):
            continue
        shared = vf[a] & vf[b]
        for g in shared:
            fkeep[g] = False
            for w in T[g]:
                vf[w].discard(g)
        flive -= len(shared)
        for g in vf[b]:
            T[g] = [a if w == b else w for w in T[g]]
            vf[a].add(g)
        vf[b] = set()
        P[a] = p
        Q[a] = [Q[a][i] + Q[b][i] for i in range(10)]
        push([(min(a, w), max(a, w)) for w in nbrs(a)])
    out_v, out_f = compact(np.array(P, np.float32), np.array(T, np.int64), fkeep)
    return out_v.astype(np.float32), out_f.astype(np.int32)
