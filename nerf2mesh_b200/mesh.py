"""Stage-0 -> stage-1 mesh hand-off on the device: marching cubes over the density volume + PLY writer.

Replaces the `mcubes.marching_cubes(sigmas, density_thresh)` call of NeRFRenderer.export_stage0 (nerf/renderer.py:526-529; PyMCubes is a
third-party CPU library) with the kernels of csrc/mcubes.cu (C ABI include/n2m_b200_mesh.h):

    vertices, triangles = marching_cubes(volume, isovalue)      # volume [X,Y,Z] float32 CUDA tensor
    # vertices [V,3] float32 in index coordinates (0 .. X-1), triangles [F,3] int32 -- the form PyMCubes returns (as tensors)

`export_stage0_mesh(trainer, path, resolution)` is the reference's export: density volume (Stage0Trainer.density_volume ==
renderer.py:480-524) -> marching cubes -> `vertices / (resolution - 1) * 2 - 1` (:531) -> with `clean=CleanOptions(...)` the visibility
test, remove_masked_faces and clean_mesh -> with `decimate_target=` decimate_mesh -> `mesh_0.ply`.  No CPU fallback: the volume must
live on a CUDA device.

The reference's pymeshlab post-processing (meshutils.py) is restated as exact rules in csrc/meshclean.cu: `remove_masked_faces`
(remove_masked_trigs: the faces a mask keeps, dilated along shared vertices) and `clean_mesh` (clean_mesh(..., remesh=False): close-vertex
merge, duplicate and null faces, small components, non-manifold edges and vertices).  `decimate_mesh` (csrc/decimate.cu) restates
meshing_decimation_quadric_edge_collapse as rounds of independent quadric edge collapses, this library's own deterministic rule.  The mesh
stays on the device from marching cubes to the PLY writer; the host reads back output sizes, the merge's round flags and one face count
per decimation round only.

Unbounded scenes (bound > 1, C = 1 + ceil(log2(bound)) cascades) also get one mesh per outer cascade (csrc/cascade.cu):
`export_outer_meshes(trainer, path, env_reso)` is the non-SDF branch of export_stage0 for cas = 1 .. C-1 (renderer.py:606-672) --
occupancy volume of density_grid[cas] -> marching cubes at 0.5 -> world coordinates (float64, rounded once) -> removal of the centre box
and of what lies outside the training AABB -> with `clean=` clean_mesh -> with `decimate_target=` decimate_mesh to half of it -> with
`clean=` the visibility test -> `mesh_{cas}.ply`.
`mark_unseen_triangles` is the reference's visibility test on those meshes, `load_stage0_meshes` picks every cascade's mesh up again for
stage 1.
"""
import ctypes
import os
import struct

import numpy as np
import torch

from . import _lib
from . import mc_table
from . import raster as dr
from ._lib import F, P, U, call, ptr, stream

D = ctypes.c_double

_lib.register({
    "n2m_mc_count": [P, U, U, U, F, P, P, P, P],
    "n2m_mc_emit": [P, U, U, U, F, P, P, P, P, P, P, P],
    "n2m_outer_occupancy": [P, U, U, F, P, P],
    "n2m_outer_select": [P, U, U, D, D, D, D, D, D, D, P, P, P],
    "n2m_rsv_count": [P, U, P, U, P, P, P],
    "n2m_rsv_emit": [P, U, P, U, P, P, P, P, P, P, P],
    "n2m_mark_seen_faces": [P, U, U, P, P],
    "n2m_clean_mark_verts": [P, U, P, P, P],
    "n2m_clean_dilate": [P, U, P, P, P],
    "n2m_clean_bbox": [P, U, P, P, P],
    "n2m_clean_merge_bin": [P, U, P, P, D, U, P, P, P],
    "n2m_clean_merge_fill": [U, P, P, P, P, P],
    "n2m_clean_merge_round": [P, U, P, P, D, U, P, P, ctypes.c_int32, P, P, P, P],
    "n2m_clean_merge_apply": [P, U, P, P, P],
    "n2m_clean_dup_null": [P, P, U, P, U, P, P, P],
    "n2m_clean_edge_table": [P, U, P, U, P, P, P],
    "n2m_clean_components": [P, P, U, P, P, P, P, D, U, P, P, P, P, P, P],
    "n2m_clean_nm_edges": [P, P, U, P, P, U, P, P, P, P, U, P],
    "n2m_clean_nm_verts_find": [P, U, U, P, P, U, P, P, P, P, P, P, P, P, U, P],
    "n2m_clean_nm_verts_apply": [P, U, P, U, P, P, P, P, P, P],
    "n2m_decim_init": [P, U, P, P, P],
    "n2m_decim_vcount": [P, U, P, P, P],
    "n2m_decim_vfill": [P, U, P, P, P, P],
    "n2m_decim_quadrics": [P, U, P, P, P, P, P],
    "n2m_decim_edges": [P, U, U, P, P, U, P, P, P],
    "n2m_decim_eval": [P, P, P, U, P, P, P, P, P, P, P, ctypes.c_int, P, P, P],
    "n2m_decim_threshold": [P, U, P, P, P, U, P, P, P],
    "n2m_decim_select": [P, U, U, P, P, P, P, P, P, P, P, P, P, P, P, P, P],
})

_tables = {}


def _device_tables(device):
    key = torch.device(device).index
    if key not in _tables:
        _tables[key] = (torch.from_numpy(mc_table.TRI_TABLE.copy()).to(device), torch.from_numpy(mc_table.NUM_TRIS.copy()).to(device))
    return _tables[key]


def marching_cubes(volume, isovalue):
    """volume [X,Y,Z] float32 CUDA tensor, isovalue float -> (vertices [V,3] float32 in index coordinates, triangles [F,3] int32).
    Inside = value > isovalue; normals point from inside to outside; vertices are shared between cells; deterministic order."""
    if not volume.is_cuda:
        raise RuntimeError("marching_cubes: the volume must be a CUDA tensor (nerf2mesh_b200 has no CPU path)")
    if volume.dim() != 3 or min(volume.shape) < 2:
        raise RuntimeError("marching_cubes: volume must be [X,Y,Z] with at least two samples per axis")
    vol = volume.float().contiguous()
    X, Y, Z = (int(s) for s in vol.shape)
    n = X * Y * Z
    dev = vol.device
    tri_table, num_tris = _device_tables(dev)
    vcount = torch.empty(n, dtype=torch.uint8, device=dev); tcount = torch.empty(n, dtype=torch.uint8, device=dev)
    call("n2m_mc_count", ptr(vol), X, Y, Z, float(isovalue), ptr(num_tris), ptr(vcount), ptr(tcount), stream())
    vinc = torch.cumsum(vcount, 0, dtype=torch.int32); tinc = torch.cumsum(tcount, 0, dtype=torch.int32)
    V, T = int(vinc[-1].item()), int(tinc[-1].item())                     # the one host read-back (output sizes)
    voff = vinc - vcount.to(torch.int32); toff = tinc - tcount.to(torch.int32)
    del vinc, tinc
    vertices = torch.empty(V, 3, device=dev); triangles = torch.empty(T, 3, dtype=torch.int32, device=dev)
    if V > 0 or T > 0:
        call("n2m_mc_emit", ptr(vol), X, Y, Z, float(isovalue), ptr(tri_table), ptr(tcount), ptr(voff), ptr(toff),
             ptr(vertices) if V > 0 else ptr(torch.empty(3, device=dev)), ptr(triangles) if T > 0 else ptr(torch.empty(3, dtype=torch.int32, device=dev)), stream())
    return vertices, triangles


def write_ply(path, vertices, triangles):
    """binary little-endian PLY (float32 x y z, uchar-counted int32 face lists): the format trimesh writes for `mesh_0.ply`
    (renderer.py:543-544) and reads back in stage 1"""
    v = np.ascontiguousarray(vertices.detach().cpu().numpy() if torch.is_tensor(vertices) else vertices, dtype="<f4")
    f = np.ascontiguousarray(triangles.detach().cpu().numpy() if torch.is_tensor(triangles) else triangles, dtype="<i4")
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {v.shape[0]}\nproperty float x\nproperty float y\nproperty float z\n"
              f"element face {f.shape[0]}\nproperty list uchar int vertex_indices\nend_header\n").encode("ascii")
    faces = np.empty(f.shape[0], dtype=[("n", "u1"), ("i", "<i4", (3,))])
    faces["n"] = 3; faces["i"] = f
    with open(path, "wb") as fh:
        fh.write(header); fh.write(v.tobytes()); fh.write(faces.tobytes())


def read_ply(path):
    """the inverse of write_ply (tests, and stage 1 picking the mesh up again)"""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").split("\n")
    nv = int(next(l for l in head if l.startswith("element vertex")).split()[-1])
    nf = int(next(l for l in head if l.startswith("element face")).split()[-1])
    v = np.frombuffer(data, dtype="<f4", count=3 * nv, offset=end).reshape(nv, 3)
    faces = np.frombuffer(data, dtype=[("n", "u1"), ("i", "<i4", (3,))], count=nf, offset=end + 12 * nv)
    assert (faces["n"] == 3).all()
    return v.copy(), faces["i"].copy()


def export_stage0_mesh(trainer, save_path, resolution=512, density_thresh=10.0, *, clean=None, decimate_target=0):
    """NeRFRenderer.export_stage0 for the inner region (renderer.py:471-544): density volume -> marching cubes at
    min(mean_density, density_thresh) -> world coordinates -> with `clean` (a CleanOptions): the visibility test and remove_masked_faces
    when it carries views, then clean_mesh(repair=True) (:531-537) -> with decimate_target > 0 and more faces than int(decimate_target):
    decimate_mesh to that many faces with optimal placement (:540-541) -> `<save_path>/mesh_0.ply`.  Returns (vertices, triangles) on the
    device.  The outer-region meshes of an unbounded scene come from `export_outer_meshes`."""
    vol = trainer.density_volume(resolution=resolution, density_thresh=density_thresh)
    mean = getattr(trainer, "mean_density", None)
    thresh = min(float(mean.item()), density_thresh) if mean is not None else density_thresh
    v, f = marching_cubes(vol, thresh)
    v = v / (resolution - 1.0) * 2 - 1                      # renderer.py:531
    if clean is not None:
        del vol
        v, f = clean.visibility(v, f)
        v, f = clean_mesh(v, f, min_f=clean.min_f, min_d=clean.min_d, repair=True)
    if decimate_target > 0 and f.shape[0] > int(decimate_target):
        v, f = decimate_mesh(v, f, int(decimate_target), optimal_placement=True)
    os.makedirs(save_path, exist_ok=True)
    write_ply(os.path.join(save_path, "mesh_0.ply"), v, f)
    return v, f


# ---- outer cascades of an unbounded scene ---------------------------------------------------------------------------------------------
def _mesh_threshold(trainer, density_thresh):
    mean = getattr(trainer, "mean_density", None)
    return min(float(mean.item()), density_thresh) if mean is not None else density_thresh


def outer_occupancy(grid, grid_size, resolution, thresh):
    """grid [H^3] float32 CUDA (one cascade of the density grid, Morton order) -> float32 [R,R,R] 0/1 volume (x-major) =
    nan_to_num(F.interpolate(occ[None,None], [R]*3, mode='trilinear')[0,0], 0) > thresh, occ the grid re-mapped to [H,H,H]
    (renderer.py:618-628)"""
    H, R = int(grid_size), int(resolution)
    if not grid.is_cuda or grid.dtype != torch.float32 or grid.numel() != H ** 3:
        raise ValueError(f"outer_occupancy: grid must be a float32 CUDA tensor of {H}^3 cells")
    grid = grid.contiguous()
    vol = torch.empty(R, R, R, device=grid.device)
    call("n2m_outer_occupancy", ptr(grid), H, R, float(thresh), ptr(vol), stream())
    return vol


def outer_select(vertices, resolution, scale, box):
    """vertices [V,3] float32 CUDA in index coordinates -> (world [V,3] float32, removed [V] bool): p = idx / (R-1) * 2 - 1, world = p * scale
    in float64 rounded once; removed where every |p_c| <= 0.45 (renderer.py:633-635) or where world is outside the open box
    box = (xmn, ymn, zmn, xmx, ymx, zmx) (:640-649)"""
    V = int(vertices.shape[0])
    vertices = vertices.float().contiguous()
    out = torch.empty(V, 3, device=vertices.device)
    removed = torch.empty(V, dtype=torch.uint8, device=vertices.device)
    call("n2m_outer_select", ptr(vertices), V, int(resolution), float(scale), *(float(b) for b in box), ptr(out), ptr(removed), stream())
    return out, removed.bool()


def remove_selected_vertices(vertices, triangles, removed):
    """pymeshlab's remove_selected_verts (meshutils.py:122-144) on the device: vertices [V,3] float32, triangles [F,3] int32, removed [V] bool
    (CUDA) -> the unflagged vertices in their order (also those no face references any more) and the faces none of whose corners is flagged,
    re-indexed."""
    dev = vertices.device
    vertices = vertices.float().contiguous(); triangles = triangles.int().contiguous()
    V, Fn = int(vertices.shape[0]), int(triangles.shape[0])
    removed = removed.to(dev, torch.uint8).contiguous()
    if removed.numel() != V:
        raise ValueError("remove_selected_vertices: one flag per vertex")
    vkeep = torch.empty(V, dtype=torch.uint8, device=dev); fkeep = torch.empty(Fn, dtype=torch.uint8, device=dev)
    call("n2m_rsv_count", ptr(removed), V, ptr(triangles), Fn, ptr(vkeep), ptr(fkeep), stream())
    return _emit(vertices, triangles, vkeep, fkeep)


def _emit(vertices, triangles, vkeep, fkeep):
    """the flagged vertices in order and the flagged faces re-indexed (every corner of a flagged face must be flagged): exclusive prefix
    sums of the flags, one read-back of the output sizes, n2m_rsv_emit"""
    dev = vertices.device
    V, Fn = int(vertices.shape[0]), int(triangles.shape[0])
    vinc = torch.cumsum(vkeep, 0, dtype=torch.int32); finc = torch.cumsum(fkeep, 0, dtype=torch.int32)
    nv = int(vinc[-1].item()) if V else 0
    nf = int(finc[-1].item()) if Fn else 0                                   # the host read-backs (output sizes)
    voff = vinc - vkeep.to(torch.int32); foff = finc - fkeep.to(torch.int32)
    out_v = torch.empty(nv, 3, device=dev); out_f = torch.empty(nf, 3, dtype=torch.int32, device=dev)
    call("n2m_rsv_emit", ptr(vertices), V, ptr(triangles), Fn, ptr(vkeep), ptr(fkeep), ptr(voff), ptr(foff), ptr(out_v) if nv else None,
         ptr(out_f) if nf else None, stream())
    return out_v, out_f


# ---- mesh clean-up (csrc/meshclean.cu) -----------------------------------------------------------------------------------------------
def _pow2(n):
    return 1 << max(int(n) - 1, 1).bit_length()


def _mesh_args(name, vertices, triangles):
    if not (torch.is_tensor(vertices) and torch.is_tensor(triangles) and vertices.is_cuda and triangles.is_cuda):
        raise RuntimeError(f"{name}: vertices and triangles must be CUDA tensors (nerf2mesh_b200 has no CPU path)")
    if vertices.dim() != 2 or vertices.shape[1] != 3 or triangles.dim() != 2 or triangles.shape[1] != 3:
        raise ValueError(f"{name}: vertices [V,3] and triangles [F,3]")
    if 3 * triangles.shape[0] >= 2 ** 31 or vertices.shape[0] >= 2 ** 31:
        raise ValueError(f"{name}: at most 2^31 / 3 faces and 2^31 vertices")
    if triangles.shape[0] > 0 and vertices.shape[0] == 0:
        raise ValueError(f"{name}: faces without vertices")
    return vertices.float().contiguous(), triangles.to(vertices.device, torch.int32).contiguous()


def _empty(vertices):
    return vertices.new_empty(0, 3), torch.empty(0, 3, dtype=torch.int32, device=vertices.device)


def _referenced(tri, fkeep, V):
    vflag = torch.zeros(V, dtype=torch.uint8, device=tri.device)
    call("n2m_clean_mark_verts", ptr(tri), int(tri.shape[0]), ptr(fkeep), ptr(vflag), stream())
    return vflag


@torch.no_grad()
def remove_masked_faces(vertices, triangles, mask, dilation):
    """remove_masked_trigs (meshutils.py:63-93) on the device.  vertices [V,3] float32, triangles [F,3] int32, mask [F] (0 keeps the face,
    1 removes it), CUDA.  The faces with mask == 0 are the kept set; each of the `dilation` steps selects every vertex of a kept face and
    keeps every face with a selected vertex (MeshLab's selection dilation); the other faces and the vertices no kept face references go.
    Survivors keep their order."""
    v, tri = _mesh_args("remove_masked_faces", vertices, triangles)
    V, Fn = int(v.shape[0]), int(tri.shape[0])
    mask = torch.as_tensor(mask).to(v.device).reshape(-1)
    if mask.numel() != Fn:
        raise ValueError("remove_masked_faces: one mask entry per face")
    if Fn == 0:
        return _empty(v)
    fkeep = (mask == 0).to(torch.uint8)
    vsel = torch.zeros(V, dtype=torch.uint8, device=v.device)
    for _ in range(int(dilation)):
        call("n2m_clean_dilate", ptr(tri), Fn, ptr(fkeep), ptr(vsel), stream())
    return _emit(v, tri, _referenced(tri, fkeep, V), fkeep)


@torch.no_grad()
def clean_mesh(vertices, triangles, v_pct=1, min_f=8, min_d=5, repair=True, info=None):
    """clean_mesh(..., remesh=False) (meshutils.py:146-188) on the device.  vertices [V,3] float32, triangles [F,3] int32 (CUDA, every index
    in 0..V-1) -> (vertices, triangles) of the same types.  In order:

    1. vertices no face references go;
    2. v_pct > 0: close vertices merge with radius r = v_pct / 100 * diag / 10 (diag: the bounding-box diagonal, float64) -- greedily
       in index order, vertex i leads unless a leader j < i lies within r (float64 dx*dx + dy*dy + dz*dz <= r*r), a non-leader takes the
       lowest such leader's index; faces that then repeat an index go;
    3. duplicate faces (the same unordered vertex triple, any winding) go but the lowest;
    4. faces whose float64 cross(b - a, c - a) is the zero vector go;
    5. min_d > 0: edge-connected components (faces sharing two vertices) whose bounding-box diagonal is < min_d / 100 * diag go (diag of
       the vertices still referenced);
    6. min_f > 0: components of fewer than min_f faces go;
    7. repair: the faces on an edge of more than two faces are visited by ascending float64 area (then index); a face goes when one of
       its edges still has more than two faces;
    8. repair: a vertex whose faces form k > 1 fans (faces joined through an edge at the vertex) is split: the fan with the lowest face
       keeps it, each other fan gets a copy appended after all vertices, in (vertex, lowest face of the fan) order.

    Surviving vertices and faces keep their order; the vertices no face references at the end go.  The percentage readings of steps 2
    and 5 are this library's (pymeshlab is not run to confirm them).  `info`, a dict, receives `merge_rounds`: the decision rounds of
    step 2, each one launch and one read-back of a flag."""
    v, tri = _mesh_args("clean_mesh", vertices, triangles)
    tri = tri.clone()                                                        # re-indexed in place by the merge and the split
    dev = v.device
    V, Fn = int(v.shape[0]), int(tri.shape[0])
    rounds = 0
    if info is not None:
        info["merge_rounds"] = 0
    if Fn == 0:
        return _empty(v)
    i32 = dict(dtype=torch.int32, device=dev)
    fkeep = torch.ones(Fn, dtype=torch.uint8, device=dev)
    bbox = torch.empty(6, **i32)
    if v_pct > 0:                                                            # 1. + 2.
        vflag = _referenced(tri, None, V)
        call("n2m_clean_bbox", ptr(v), V, ptr(vflag), ptr(bbox), stream())
        nb = _pow2(2 * V)
        count = torch.zeros(nb, **i32); vbucket = torch.empty(V, **i32)
        call("n2m_clean_merge_bin", ptr(v), V, ptr(vflag), ptr(bbox), float(v_pct), nb, ptr(count), ptr(vbucket), stream())
        start = torch.zeros(nb + 1, **i32)
        torch.cumsum(count, 0, dtype=torch.int32, out=start[1:])
        cursor = start[:-1].clone(); items = torch.empty(V, **i32)
        call("n2m_clean_merge_fill", V, ptr(vflag), ptr(vbucket), ptr(cursor), ptr(items), stream())
        decided = torch.zeros(V, **i32); target = torch.empty(V, **i32); pending = torch.zeros(1, **i32)
        while True:
            rounds += 1
            pending.zero_()
            call("n2m_clean_merge_round", ptr(v), V, ptr(vflag), ptr(bbox), float(v_pct), nb, ptr(start), ptr(items), rounds, ptr(decided),
                 ptr(target), ptr(pending), stream())
            if not int(pending.item()):                                      # the round-termination read-back
                break
        del count, vbucket, start, cursor, items, decided
        call("n2m_clean_merge_apply", ptr(tri), Fn, ptr(target), ptr(fkeep), stream())
        if info is not None:
            info["merge_rounds"] = rounds
    nt = _pow2(2 * Fn)                                                       # 3. + 4.
    table, slot_of = torch.empty(nt, **i32), torch.empty(Fn, **i32)
    call("n2m_clean_dup_null", ptr(v), ptr(tri), Fn, ptr(fkeep), nt, ptr(table), ptr(slot_of), stream())
    if min_d > 0 or min_f > 0 or repair:
        ne = _pow2(6 * Fn)
        table = torch.empty(ne, **i32); slot_of = torch.empty(3 * Fn, **i32)
        call("n2m_clean_edge_table", ptr(tri), Fn, ptr(fkeep), ne, ptr(table), ptr(slot_of), stream())
    if min_d > 0 or min_f > 0:                                               # 5. + 6.
        vflag = _referenced(tri, fkeep, V)
        call("n2m_clean_bbox", ptr(v), V, ptr(vflag), ptr(bbox), stream())
        parent, label, count = (torch.empty(Fn, **i32) for _ in range(3))
        cmin, cmax = torch.empty(3 * Fn, **i32), torch.empty(3 * Fn, **i32)
        call("n2m_clean_components", ptr(v), ptr(tri), Fn, ptr(fkeep), ptr(table), ptr(slot_of), ptr(bbox), float(max(min_d, 0)),
             int(max(min_f, 0)), ptr(parent), ptr(label), ptr(count), ptr(cmin), ptr(cmax), stream())
        del parent, label, count, cmin, cmax
    if repair:                                                               # 7. + 8.
        # once slot_of is known the table's slots are free: they hold the per-edge live face counts, then the per-edge lowest face-edge
        cap = _pow2(3 * Fn)
        keys, vals, ncand = torch.empty(cap, dtype=torch.int64, device=dev), torch.empty(cap, **i32), torch.empty(1, **i32)
        call("n2m_clean_nm_edges", ptr(v), ptr(tri), Fn, ptr(fkeep), ptr(slot_of), ne, ptr(table), ptr(ncand), ptr(keys), ptr(vals), cap,
             stream())
        cparent, clabel, cnew = (torch.empty(3 * Fn, **i32) for _ in range(3))
        vmin, nextra = torch.empty(V, **i32), torch.empty(1, **i32)
        call("n2m_clean_nm_verts_find", ptr(tri), V, Fn, ptr(fkeep), ptr(slot_of), ne, ptr(table), ptr(cparent), ptr(clabel), ptr(vmin),
             ptr(nextra), ptr(keys), ptr(vals), ptr(cnew), cap, stream())
        n = int(nextra.item())                                               # read-back: the number of vertex copies (output size)
        ext = torch.empty(V + n, 3, device=dev)
        ext[:V] = v
        call("n2m_clean_nm_verts_apply", ptr(v), V, ptr(tri), Fn, ptr(fkeep), ptr(clabel), ptr(vmin), ptr(cnew), ptr(ext), stream())
        v, V = ext, V + n
    return _emit(v, tri, _referenced(tri, fkeep, V), fkeep)


class CleanOptions:
    """the reference's post-processing of the stage-0 meshes (`clean=` of export_stage0_mesh / export_outer_meshes): clean_mesh with
    min_f / min_d (opt.clean_min_f, opt.clean_min_d), and -- when mvps, H, W are given (the `mesh_visibility_culling` of -O) -- the faces
    no view sees removed with remove_masked_faces(dilation=visibility_mask_dilation)"""

    def __init__(self, min_f=8, min_d=5, visibility_mask_dilation=5, mvps=None, H=None, W=None):
        if mvps is not None and (H is None or W is None):
            raise ValueError("CleanOptions: the visibility test needs mvps, H and W")
        self.min_f, self.min_d, self.visibility_mask_dilation = min_f, min_d, visibility_mask_dilation
        self.mvps, self.H, self.W = mvps, H, W

    def visibility(self, v, f):
        """remove_masked_faces over mark_unseen_triangles, or the mesh unchanged without views"""
        if self.mvps is None or f.shape[0] == 0:
            return v, f
        return remove_masked_faces(v, f, mark_unseen_triangles(v, f, self.mvps, self.H, self.W), self.visibility_mask_dilation)


# ---- decimation (csrc/decimate.cu) ---------------------------------------------------------------------------------------------------
@torch.no_grad()
def decimate_mesh(vertices, triangles, target, optimal_placement=True, info=None):
    """Quadric edge-collapse decimation to `target` faces on the device: the library's parallel reading of pymeshlab's
    meshing_decimation_quadric_edge_collapse (meshutils.py decimate_mesh, VCG) with its defaults.  vertices [V,3] float32, triangles [F,3]
    int32 (CUDA) -> (vertices, triangles) of the same types.  ValueError when target < 1.  F <= target: no collapse, only the vertices no
    face references go.

    Otherwise faces that repeat an index go, and rounds of collapses run while more than `target` faces live:
    - quadrics: each face's plane quadric from its float64 unit normal n = cross(b - a, c - a) / |.| and d = -n.a, without area weight
      (zero when |cross| = 0); a vertex sums those of its faces in ascending face index;
    - placement of the merged vertex of edge (a, b), a < b, with Q = Q_a + Q_b: optimal_placement solves A p = -b when
      det(A) > 1e-6 trace(A)^3 (every eigenvalue above 1e-6 of the trace), else takes the cheapest of a, b and the midpoint (ties in that
      order); without it, the float64 midpoint.  The position is rounded once to float32; the cost is Q at that point;
    - validity: the edge has 1 or 2 live faces; every vertex adjacent to both a and b is an opposite vertex of those faces (link
      condition); it is a boundary edge or not both ends are boundary vertices; a boundary edge's face does not have its other two edges
      on the boundary too (a lone triangle would vanish, and with it a component); not both (a, c, d) and (b, c, d) are live faces for
      its opposite vertices c, d; and no other face at a or b flips or degenerates (float64 dot(n_old, n_new) <= 0).  A manifold mesh
      stays manifold and keeps its Euler characteristic;
    - key: fkey(float32(cost)) << 32 | e, e the edge's lowest live face-edge 3f + k (faces keep their input index between rounds);
    - budget: K* is the least key at which the valid edges in key order, each counted with its 1 or 2 faces, remove at least
      (live faces - target); only keys <= K* may be selected, so the last round ends at target or target - 1 faces;
    - selection: vmin[v] = the least such key at v, r1[v] = the least vmin over v and its neighbours; an edge whose key equals r1 at
      both ends is selected.  Selected edges share no vertex and no adjacency, so the round equals their collapses in any order;
    - apply: a survives at the float32 position with Q_a + Q_b, every face re-indexes b -> a, and the faces that then repeat an index go.
    The rounds stop at <= target faces or when a round selects nothing (stalled).  Surviving vertices and faces keep their order, and the
    vertices no face references go (VCG's autoclean).

    VCG collapses one edge at a time from a heap, with a quality-threshold penalty and its own placement; this rule keeps its defaults'
    reading (preserveboundary=False, preservetopology=False, planarquadric=False, autoclean=True, no quality penalty) and is not claimed
    to reproduce its output.  `info`, a dict, receives `rounds` (rounds that collapsed something), `stalled` and `faces` (live faces after
    each round); the host reads back one count per round and the output sizes."""
    v, tri = _mesh_args("decimate_mesh", vertices, triangles)
    target = int(target)
    if target < 1:
        raise ValueError("decimate_mesh: target must be at least 1")
    dev = v.device
    V, Fn = int(v.shape[0]), int(tri.shape[0])
    rounds, faces, stalled = 0, [], False
    if Fn == 0:
        out = _empty(v)
    elif Fn <= target:
        out = _emit(v, tri, _referenced(tri, None, V), torch.ones(Fn, dtype=torch.uint8, device=dev))
    else:
        v, tri = v.clone(), tri.clone()                                      # positions move and faces re-index in place
        i32, i64 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.int64, device=dev)
        fkeep, flive = torch.empty(Fn, dtype=torch.uint8, device=dev), torch.empty(1, **i32)
        call("n2m_decim_init", ptr(tri), Fn, ptr(fkeep), ptr(flive), stream())
        ne = _pow2(6 * Fn)
        table, ecount, slot_of = torch.empty(ne, **i32), torch.empty(ne, **i32), torch.empty(3 * Fn, **i32)
        vcount, vstart, vfaces = torch.empty(V, **i32), torch.zeros(V + 1, **i32), torch.empty(3 * Fn, **i32)
        vbnd = torch.empty(V, dtype=torch.uint8, device=dev)
        keys, pos = torch.empty(3 * Fn, **i64), torch.empty(3 * Fn, 3, device=dev)
        Q = torch.empty(V, 10, dtype=torch.float64, device=dev)
        hist, state, vmin, r1 = torch.empty(256, **i64), torch.empty(4, **i64), torch.empty(V, **i64), torch.empty(V, **i64)
        vtarget = torch.empty(V, **i32)
        live = int(flive.item())                                             # read-back: live faces
        while live > target:
            call("n2m_clean_edge_table", ptr(tri), Fn, ptr(fkeep), ne, ptr(table), ptr(slot_of), stream())
            vcount.zero_()
            call("n2m_decim_vcount", ptr(tri), Fn, ptr(fkeep), ptr(vcount), stream())
            torch.cumsum(vcount, 0, dtype=torch.int32, out=vstart[1:])
            cursor = vstart[:-1].clone()
            call("n2m_decim_vfill", ptr(tri), Fn, ptr(fkeep), ptr(cursor), ptr(vfaces), stream())
            if rounds == 0:
                call("n2m_decim_quadrics", ptr(v), V, ptr(tri), ptr(vstart), ptr(vfaces), ptr(Q), stream())
            call("n2m_decim_edges", ptr(tri), V, Fn, ptr(fkeep), ptr(slot_of), ne, ptr(ecount), ptr(vbnd), stream())
            call("n2m_decim_eval", ptr(v), ptr(Q), ptr(tri), Fn, ptr(fkeep), ptr(table), ptr(slot_of), ptr(ecount), ptr(vbnd), ptr(vstart),
                 ptr(vfaces), int(bool(optimal_placement)), ptr(keys), ptr(pos), stream())
            call("n2m_decim_threshold", ptr(keys), Fn, ptr(slot_of), ptr(ecount), ptr(flive), target, ptr(hist), ptr(state), stream())
            call("n2m_decim_select", ptr(keys), V, Fn, ptr(tri), ptr(slot_of), ptr(ecount), ptr(vstart), ptr(vfaces), ptr(state), ptr(pos),
                 ptr(vmin), ptr(r1), ptr(v), ptr(Q), ptr(vtarget), ptr(flive), stream())
            call("n2m_clean_merge_apply", ptr(tri), Fn, ptr(vtarget), ptr(fkeep), stream())
            now = int(flive.item())                                          # the round's read-back: live faces
            if now == live:
                stalled = True
                break
            rounds += 1
            faces.append(now)
            live = now
        del table, ecount, slot_of, vcount, vstart, vfaces, vbnd, keys, pos, Q, vmin, r1, vtarget
        out = _emit(v, tri, _referenced(tri, fkeep, V), fkeep)
    if info is not None:
        info.update(rounds=rounds, stalled=stalled, faces=faces)
    return out


@torch.no_grad()
def export_outer_meshes(trainer, save_path, env_reso=256, density_thresh=10.0, *, clean=None, decimate_target=0):
    """export_stage0's outer meshes (non-SDF, renderer.py:606-672), for every cascade cas = 1 .. C-1: occupancy volume of
    density_grid[cas] at env_reso^3 -> marching cubes at 0.5 -> (idx / (R-1) * 2 - 1) * (bound - half) with bound = min(2^cas, cfg.bound),
    half = bound / R -> removal of the centre box and of the region outside the trainer's AABB shrunk by half -> with `clean` (a
    CleanOptions): clean_mesh(repair=False) -> with decimate_target > 0 and more faces than int(decimate_target) // 2: decimate_mesh to
    that many faces without optimal placement (:609, :657-659) -> with `clean` carrying views: the visibility test and
    remove_masked_faces (:661-668) -> `<save_path>/mesh_{cas}.ply`.  Returns {cas: (vertices [V,3] float32, triangles [F,3] int32)} on
    the device; a cascade left without vertices writes no file and is not in the dict."""
    if hasattr(trainer, "drop_prefetch"):
        trainer.drop_prefetch()
    c = trainer.cfg
    R, H = int(env_reso), int(c.grid_size)
    thresh = _mesh_threshold(trainer, density_thresh)
    xmn, ymn, zmn, xmx, ymx, zmx = trainer.aabb.detach().cpu().numpy().astype(np.float64).tolist()
    os.makedirs(save_path, exist_ok=True)
    meshes = {}
    for cas in range(1, c.cascade):
        bound = min(2 ** cas, c.bound)
        half = bound / R
        vol = outer_occupancy(trainer.density_grid[cas], H, R, thresh)
        v, f = marching_cubes(vol, 0.5)
        del vol
        if v.shape[0] == 0:
            continue
        v, removed = outer_select(v, R, bound - half, (xmn + half, ymn + half, zmn + half, xmx - half, ymx - half, zmx - half))
        v, f = remove_selected_vertices(v, f, removed)
        if clean is not None:
            v, f = clean_mesh(v, f, min_f=clean.min_f, min_d=clean.min_d, repair=False)
        half_target = int(decimate_target) // 2
        if v.shape[0] > 0 and half_target > 0 and f.shape[0] > half_target:
            v, f = decimate_mesh(v, f, half_target, optimal_placement=False)
        if clean is not None and v.shape[0] > 0:
            v, f = clean.visibility(v, f)
        if v.shape[0] == 0:
            continue
        write_ply(os.path.join(save_path, f"mesh_{cas}.ply"), v, f)
        meshes[cas] = (v, f)
    return meshes


@torch.no_grad()
def mark_unseen_triangles(vertices, triangles, mvps, H, W, glctx=None):
    """The reference's visibility test (mark_unseen_triangles, renderer.py:947-981): rasterise the mesh in every view (mvps [B,4,4]) at
    (H, W) and return the [F] bool mask of the faces no view covers.  As in the reference, an uncovered pixel's face index -1 marks the
    last face, so face F-1 counts as seen whenever a view has an empty pixel."""
    dev = torch.device("cuda", torch.cuda.current_device()) if not torch.is_tensor(vertices) or not vertices.is_cuda else vertices.device
    v = torch.as_tensor(vertices).to(dev, torch.float32).contiguous()
    tri = torch.as_tensor(triangles).to(dev, torch.int32).contiguous()
    Fn = int(tri.shape[0])
    seen = torch.zeros(Fn, dtype=torch.uint8, device=dev)
    glctx = glctx or dr.RasterizeCudaContext(dev)
    vh = torch.nn.functional.pad(v, pad=(0, 1), mode="constant", value=1.0)
    for mvp in mvps:
        vclip = torch.matmul(vh, torch.transpose(torch.as_tensor(mvp).to(dev, torch.float32), 0, 1)).float()
        rast, _ = dr.rasterize(glctx, vclip[None], tri, (int(H), int(W)))
        call("n2m_mark_seen_faces", ptr(rast), int(H) * int(W), Fn, ptr(seen), stream())
    return seen == 0


def load_stage0_meshes(mesh_dir, cascade):
    """Per-cascade (vertices, triangles) lists for Stage1Trainer, as the reference's stage 1 loads them (renderer.py:130-157):
    `mesh_{cas}_updated.ply` (written after a refinement) when it exists, else `mesh_{cas}.ply`.  float32 / int32 CPU tensors.
    FileNotFoundError naming the file when a cascade has neither."""
    vertices, triangles = [], []
    for cas in range(int(cascade)):
        path = os.path.join(mesh_dir, f"mesh_{cas}_updated.ply")
        if not os.path.exists(path):
            path = os.path.join(mesh_dir, f"mesh_{cas}.ply")
            if not os.path.exists(path):
                raise FileNotFoundError(f"load_stage0_meshes: no mesh for cascade {cas}: {path} does not exist")
        v, f = read_ply(path)
        vertices.append(torch.from_numpy(v).float()); triangles.append(torch.from_numpy(f.astype(np.int32)))
    return vertices, triangles
