"""Test infrastructure, not product: a numpy float64 restatement of the outer-cascade mesh chain of export_stage0 (nerf/renderer.py:631-649)
after marching cubes, the checker of csrc/cascade.cu's selection and vertex-removal kernels.

    normalise          p = idx / (R - 1) * 2 - 1                                               (float64, as PyMCubes returns it)
    centre box         remove_selected_verts where every |p_c| <= 0.45
    scale              p * (bound - half), half = bound / R
    AABB               remove_selected_verts where x <= xmn + half or x >= xmx - half (each axis)
    -> float32 vertices, int32 faces

remove_selected_verts (meshutils.py:122-144, pymeshlab's meshing_remove_selected_vertices) drops the flagged vertices and every face that
touches one, keeps the other vertices in order even when no face uses them any more, and re-indexes the faces."""
import numpy as np


def remove_selected_verts(v, f, flag):
    keep = ~np.asarray(flag, bool)
    new_index = np.cumsum(keep) - 1
    fkeep = keep[f].all(axis=1) if len(f) else np.zeros(0, bool)
    return v[keep], new_index[f[fkeep]].astype(np.int64).reshape(-1, 3)


def outer_chain(vidx, f, R, bound, aabb):
    """vidx [V,3] index coordinates, f [F,3] -> (vertices [V',3] float32, faces [F',3] int32); aabb (xmn, ymn, zmn, xmx, ymx, zmx)"""
    v = np.asarray(vidx, np.float64)
    f = np.asarray(f, np.int64).reshape(-1, 3)
    v = v / (R - 1.0) * 2 - 1
    r = 0.45
    v, f = remove_selected_verts(v, f, ((v <= r) & (v >= -r)).all(axis=1))
    half = bound / R
    v = v * (bound - half)
    lo = np.array(aabb[:3], np.float64) + half
    hi = np.array(aabb[3:], np.float64) - half
    v, f = remove_selected_verts(v, f, ((v <= lo) | (v >= hi)).any(axis=1))
    return v.astype(np.float32), f.astype(np.int32)
