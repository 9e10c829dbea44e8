"""Test infrastructure, not product: a numpy / scipy restatement of the stage-0 mesh clean-up of csrc/meshclean.cu, the checker of those
kernels.  It shares no code with them: components and fans come from scipy.sparse.csgraph, the greedy close-vertex merge and the
non-manifold edge repair are plain sequential loops, and every step compacts the mesh as it goes (the kernels keep flags and compact once).

    remove_masked_faces(v, f, mask, dilation)     remove_masked_trigs (meshutils.py:63-93)
    clean_mesh(v, f, v_pct, min_f, min_d, repair)  clean_mesh(..., remesh=False) (meshutils.py:146-188)

Vertices are float32 [V,3], faces int [F,3]; results are float32 / int32.  Surviving vertices and faces keep their order.  The rules are
those of the library's specification (nerf2mesh_b200/mesh.py); pymeshlab is not run, so agreement with it is not claimed."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components
from scipy.spatial import cKDTree


def bbox_diag(v):
    """diagonal of the float32 bounding box, float64: sqrt((dx*dx + dy*dy) + dz*dz); 0 for no vertices"""
    if len(v) == 0:
        return 0.0
    lo, hi = v.min(0).astype(np.float64), v.max(0).astype(np.float64)
    d = hi - lo
    return float(np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]))


def merge_radius(diag, v_pct):
    """PercentageValue(v_pct) of meshing_merge_close_vertices read against its parameter range [0, diag / 10]"""
    return v_pct / 100.0 * diag / 10.0


def min_component_diag(diag, min_d):
    """PercentageValue(min_d) of meshing_remove_connected_component_by_diameter read against the whole diagonal"""
    return min_d / 100.0 * diag


def compact(v, f, fkeep):
    """keep the flagged faces and the vertices they reference, in order, re-indexed"""
    f = f[fkeep]
    vkeep = np.zeros(len(v), bool)
    vkeep[f.reshape(-1)] = True
    new = np.cumsum(vkeep) - 1
    return v[vkeep], new[f].reshape(-1, 3)


def _edges(f):
    """[3F] sorted (lo, hi) keys of the face edges (edge k of face i runs from corner k to corner k+1) and their group ids"""
    a, b = f.reshape(-1), np.roll(f, -1, axis=1).reshape(-1)
    keys = np.stack([np.minimum(a, b), np.maximum(a, b)], 1)
    _, inv, counts = np.unique(keys, axis=0, return_inverse=True, return_counts=True)
    return a, b, inv.reshape(-1), counts


def _cross(v, f):
    p = v.astype(np.float64)
    a, b, c = p[f[:, 0]], p[f[:, 1]], p[f[:, 2]]
    e1, e2 = b - a, c - a
    return np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1],
                     e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                     e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)


def face_area(v, f):
    n = _cross(v, f)
    return 0.5 * np.sqrt(n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2])


def remove_masked_faces(v, f, mask, dilation):
    v = np.asarray(v, np.float32).reshape(-1, 3)
    f = np.asarray(f, np.int64).reshape(-1, 3)
    kept = np.asarray(mask).reshape(-1) == 0
    for _ in range(int(dilation)):
        sel = np.zeros(len(v), bool)
        sel[f[kept].reshape(-1)] = True
        kept = sel[f].any(1)
    v, f = compact(v, f, kept)
    return v, f.astype(np.int32)


def merge_close_vertices(v, f, v_pct, stats):
    """greedy in index order: i is a leader unless a leader j < i lies within r; a non-leader takes the lowest such leader's index"""
    r = merge_radius(bbox_diag(v), v_pct)
    r2 = r * r
    p = v.astype(np.float64)
    near = cKDTree(p).query_ball_point(p, np.nextafter(r * 1.001, np.inf))
    target = np.arange(len(v))
    for i in range(len(v)):
        for j in sorted(near[i]):
            if j >= i:
                break
            if target[j] != j:
                continue
            dx, dy, dz = p[i, 0] - p[j, 0], p[i, 1] - p[j, 1], p[i, 2] - p[j, 2]
            if dx * dx + dy * dy + dz * dz <= r2:
                target[i] = j
                break
    stats["merged"] = int((target != np.arange(len(v))).sum())
    f = target[f]
    ok = (f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])
    return compact(v, f, ok)


def remove_duplicate_faces(v, f, stats):
    _, first = np.unique(np.sort(f, 1), axis=0, return_index=True)
    keep = np.zeros(len(f), bool)
    keep[first] = True
    stats["duplicates"] = int(len(f) - keep.sum())
    return compact(v, f, keep)


def remove_null_faces(v, f, stats):
    keep = (_cross(v, f) != 0).any(1)
    stats["null"] = int(len(f) - keep.sum())
    return compact(v, f, keep)


def remove_small_components(v, f, min_f, min_d, stats):
    """edge-connected components; drop those whose bounding-box diagonal < min_component_diag or whose face count < min_f"""
    F = len(f)
    _, _, inv, _ = _edges(f)
    face = np.repeat(np.arange(F), 3)
    first = np.full(inv.max() + 1, F)
    np.minimum.at(first, inv, face)
    g = coo_matrix((np.ones(3 * F), (face, first[inv])), shape=(F, F))
    n, label = connected_components(g, directed=False)
    count = np.bincount(label, minlength=n)
    lo = np.full((n, 3), np.inf, np.float32); hi = np.full((n, 3), -np.inf, np.float32)
    for k in range(3):
        np.minimum.at(lo, label, v[f[:, k]]); np.maximum.at(hi, label, v[f[:, k]])
    d = hi.astype(np.float64) - lo.astype(np.float64)
    cdiag = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
    drop = np.zeros(n, bool)
    if min_d > 0:
        drop |= cdiag < min_component_diag(bbox_diag(v), min_d)
    if min_f > 0:
        drop |= count < min_f
    stats["components_removed"] = int(drop.sum())
    return compact(v, f, ~drop[label])


def repair_non_manifold_edges(v, f, stats):
    """faces with an edge of > 2 faces, by ascending float64 area then index; delete one whose edge still has > 2 live faces"""
    _, _, inv, counts = _edges(f)
    inv = inv.reshape(-1, 3)
    cand = np.nonzero((counts[inv] > 2).any(1))[0]
    area = face_area(v, f[cand])
    order = cand[np.lexsort((cand, area))]
    cnt = counts.copy()
    keep = np.ones(len(f), bool)
    for i in order:
        if (cnt[inv[i]] > 2).any():
            keep[i] = False
            cnt[inv[i]] -= 1
    stats["nm_edge_faces"] = int((~keep).sum())
    return compact(v, f, keep)


def repair_non_manifold_vertices(v, f, stats):
    """split a vertex whose faces form k > 1 fans (joined through an edge at the vertex): the fan with the lowest face keeps it, the
    others get copies appended in (vertex, lowest face of the fan) order"""
    F = len(f)
    a, b, inv, _ = _edges(f)
    e = np.arange(3 * F)
    corner_a = e                                       # edge k of face i starts at corner 3i + k ...
    corner_b = 3 * (e // 3) + (e % 3 + 1) % 3          # ... and ends at corner 3i + (k+1) % 3
    c_lo = np.where(a < b, corner_a, corner_b)         # the corner at the edge's lower vertex
    c_hi = np.where(a < b, corner_b, corner_a)
    first = np.full(inv.max() + 1, 3 * F)
    np.minimum.at(first, inv, e)                       # each edge's first face-edge
    fe = first[inv]
    f_lo = np.where(a[fe] < b[fe], fe, 3 * (fe // 3) + (fe % 3 + 1) % 3)
    f_hi = np.where(a[fe] < b[fe], 3 * (fe // 3) + (fe % 3 + 1) % 3, fe)
    rows = np.concatenate([c_lo, c_hi]); cols = np.concatenate([f_lo, f_hi])
    _, label = connected_components(coo_matrix((np.ones(len(rows)), (rows, cols)), shape=(3 * F, 3 * F)), directed=False)
    fan_face = np.full(label.max() + 1, F)
    np.minimum.at(fan_face, label, e // 3)
    vert = f.reshape(-1)
    lowest = fan_face[label]                           # per corner: the lowest face of its fan
    primary = np.full(len(v), F)
    np.minimum.at(primary, vert, lowest)
    extra = lowest != primary[vert]
    pairs = np.unique(np.stack([vert[extra], lowest[extra]], 1), axis=0)        # sorted by (vertex, lowest face)
    stats["split_copies"] = len(pairs)
    out = vert.copy()
    if len(pairs):
        key = vert[extra] * (F + 1) + lowest[extra]
        out[extra] = len(v) + np.searchsorted(pairs[:, 0] * (F + 1) + pairs[:, 1], key)
        v = np.concatenate([v, v[pairs[:, 0]]])
    return v, out.reshape(-1, 3)


def clean_mesh(v, f, v_pct=1, min_f=8, min_d=5, repair=True, stats=None):
    """steps 1-8 of the specification; `stats` (a dict) receives how many vertices / faces each step removed or added"""
    stats = {} if stats is None else stats
    v = np.asarray(v, np.float32).reshape(-1, 3)
    f = np.asarray(f, np.int64).reshape(-1, 3)
    v, f = compact(v, f, np.ones(len(f), bool))                                     # 1. unreferenced vertices
    if len(f) and v_pct > 0:
        v, f = merge_close_vertices(v, f, v_pct, stats)                             # 2.
    if len(f):
        v, f = remove_duplicate_faces(v, f, stats)                                  # 3.
    if len(f):
        v, f = remove_null_faces(v, f, stats)                                       # 4.
    if len(f) and (min_d > 0 or min_f > 0):
        v, f = remove_small_components(v, f, min_f, min_d, stats)                   # 5. + 6.
    if len(f) and repair:
        v, f = repair_non_manifold_edges(v, f, stats)                               # 7.
        if len(f):
            v, f = repair_non_manifold_vertices(v, f, stats)                        # 8.
    return v.astype(np.float32), f.astype(np.int32)
