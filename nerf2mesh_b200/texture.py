"""Stage-1 export: the textured mesh of NeRFRenderer.export_stage1 (nerf/renderer.py:298-468) on the device.
Host side of csrc/texture.cu (C ABI include/n2m_b200_texture.h).

    vt, ft = <xatlas UV unwrap of (vertices, triangles)>                  # CPU, the caller's (see INTEGRATION.md 3d)
    export_stage1(s1, save_path, vt, ft, resolution=4096)                 # -> mesh_0.obj, mesh_0.mtl, feat0_0.jpg, feat1_0.jpg, mlp.json
    export_stage1(s1, save_path, [vt0, vt1, ...], [ft0, ft1, ...])       # several cascades: mesh_{cas}.obj ... per cascade, one mlp.json

The UV atlas is the library's own, built on the device (csrc/atlas.cu, C ABI include/n2m_b200_atlas.h) unless the caller passes one:
    vt, ft, vmapping = uv_unwrap(vertices, triangles, resolution, ssaa=2)   # vmapping[ft] == triangles, as xatlas's vmapping
    vts, fts = unwrap_stage1(s1, resolution)                                # one unwrap per cascade mesh (of contract(v) when cfg.contract)
    export_stage1(s1, save_path, resolution=4096)                           # unwrap_stage1, then the bake and the files

The stages, each callable on its own:
    uv_features(t0, vertices, triangles, vt, ft, h, w)  UV raster (n2m_rasterize of (vt * 2 - 1, 0, 1) / ft), positions interpolated with
                                                        the position triangles, hash-grid gather, geo_feat on tensor cores, quantised:
                                                        -> feats [h,w,6] uint8, mask [h,w] bool       (renderer.py:329-376)
    inpaint(feats, mask)                                the 32-texel gutter from the nearest boundary texels, in place  (:378-394)
    downscale(feats, ssaa)                              -> feat0, feat1 [h/ssaa, w/ssaa, 3] uint8 RGB                    (:396-402)
    bake_features(...)                                  the three in a row
    write_obj / write_mtl / write_mlp_json              the files (:409-439, :454-468)

Everything up to the JPEG encode stays on the device; the only host copies are the two finished textures.  A mesh that covers no texel
gives zero textures (the reference fails in its nearest-neighbour fit there).

Looking at the result -- what the viewer (renderer.html) shows, and how much the bake loses against Stage1Trainer.render:
    asset = load_exported(save_path)                                      # the files: OBJ, JPEGs (BGR -> RGB), mlp.json
    asset = ExportedMesh.from_export(s1, vt, ft, feats)                   # the same from export_stage1's return value, before the JPEG
    image, weights_sum, depth = render_exported(asset, mvp, campos, h0, w0, ssaa=1, shading="full", antialias=False)
render_exported rasterizes every cascade into one depth buffer and runs the viewer's fragment shader on the device (n2m_s1_asset_shade:
nearest texel, specular_net in fp32), then the evaluation compose of Stage1Trainer.render.
"""
import ctypes
import itertools
import json
import math
import os

import numpy as np
import torch

from . import _lib
from . import raster as dr
from . import stage0  # noqa: F401  (binds the stage-0 gather n2m_s0_encode_points)
from . import mesh as _mesh  # noqa: F401  (binds n2m_clean_edge_table)
from ._lib import F, I, P, U, call, ptr, stream

_lib.register({
    "n2m_s1_bake_points": [P, P, P, U, U, U, U, U, P, P, P, P],
    "n2m_s1_geo_feat": [P, P, U, P, P, P, P, P],
    "n2m_s1_inpaint": [P, P, U, U, P, P, P],
    "n2m_s1_ssaa_down2": [P, U, U, U, P, P, P],
    "n2m_s1_asset_shade": [P, U, P, P, P, P, P, U, P, P, P, P, F, F, F, U, P, P],
    "n2m_atlas_contract": [P, U, P, P],
    "n2m_atlas_faces": [P, P, U, P, P, P, P, P],
    "n2m_atlas_base": [U, P, P, P, P, U, P, P, P, P, P, P, P],
    "n2m_atlas_chart_count": [U, P, P, P],
    "n2m_atlas_merge_round": [U, U, P, P, P, P, P, P, P, P, P, P, P, P],
    "n2m_atlas_roots": [U, P, P, P],
    "n2m_atlas_orient": [P, P, U, P, P, P, P, P, U, U, P, P, P, P, P, P, P, P],
    "n2m_atlas_sort": [P, P, U, U, P],
    "n2m_atlas_pack": [P, P, U, I, I, I, P, P, P, P, P, P, P, P, P],
    "n2m_atlas_conflicts": [P, P, U, P, P, P, P, P, P, P, P, P, P, U, I, U, P, P, P, P],
    "n2m_atlas_split": [U, U, P, P, P, P, P, P, P, P],
    "n2m_atlas_corner_keys": [P, U, P, P, P, P, P],
    "n2m_atlas_row_flags": [P, U, P, P],
    "n2m_atlas_emit": [P, P, P, U, P, P, P, P, P, P, P, P, I, P, P, P, P],
})

MAX_BAND_POINTS = 1 << 22          # points per band: 512 MiB of gather tiles (128 B per point) + 64 MiB of positions and texel indices


def _as_tensor(x, dtype, device):
    if not torch.is_tensor(x):
        x = torch.from_numpy(np.ascontiguousarray(x))
    return x.to(device=device, dtype=dtype).contiguous()


def validate_mesh(vertices, triangles, vt, ft, h, w):
    """ValueError unless ft matches triangles row for row, every index is in range, vt lies in [0, 1] and h * w fits the rasterizer."""
    V, T = int(vertices.shape[0]), int(vt.shape[0])
    if triangles.dim() != 2 or triangles.shape[1] != 3 or ft.dim() != 2 or ft.shape[1] != 3:
        raise ValueError("triangles and ft must be [F,3]")
    if ft.shape[0] != triangles.shape[0]:
        raise ValueError(f"ft has {ft.shape[0]} rows, triangles {triangles.shape[0]}: one UV triangle per mesh triangle")
    if vt.dim() != 2 or vt.shape[1] != 2:
        raise ValueError("vt must be [Nt,2]")
    if h <= 0 or w <= 0 or h * w >= 1 << 31:
        raise ValueError(f"texture {h}x{w}: the UV raster holds fewer than 2^31 texels")
    if ft.numel():
        if int(ft.min()) < 0 or int(ft.max()) >= T:
            raise ValueError(f"ft indexes outside vt (0..{T - 1})")
        if int(triangles.min()) < 0 or int(triangles.max()) >= V:
            raise ValueError(f"triangles index outside the vertices (0..{V - 1})")
    if vt.numel() and not (bool(torch.isfinite(vt).all()) and float(vt.min()) >= 0.0 and float(vt.max()) <= 1.0):
        raise ValueError("vt must lie in [0, 1]")


class Baker:
    """Band buffers of the feature bake: the points of `band_points` texels at a time (positions, texel indices, gather tiles)."""

    def __init__(self, t0, band_points):
        self.t0 = t0
        dev = t0.device
        self.cap = (int(band_points) + 127) // 128 * 128
        self.pix = torch.zeros(self.cap, dtype=torch.int32, device=dev)
        self.pts = torch.zeros(self.cap, 3, device=dev)
        self.enc_tiles = torch.zeros(self.cap * 64, dtype=torch.float16, device=dev)
        self.counters = torch.zeros(16, dtype=torch.int32, device=dev)

    def band(self, rast, vertices, triangles, w, y0, y1, feats, feats_f32=None, contract=False):
        """rows [y0, y1) of the UV raster: points -> gather -> geo_feat into feats [h*w*6] uint8 (feats_f32 [cap,6]: the float features of
        the band's points, in the order of self.pix / self.pts)."""
        self.points(rast, vertices, triangles, w, y0, y1, contract)
        self.features(feats, feats_f32)

    def points(self, rast, vertices, triangles, w, y0, y1, contract=False):
        """the band's covered texels -> self.pix, self.pts, then the hash-grid gather of those points -> self.enc_tiles"""
        t0 = self.t0
        call("n2m_s1_bake_points", ptr(rast), ptr(vertices), ptr(triangles), w, y0, y1, self.cap, int(bool(contract)), ptr(self.counters),
             ptr(self.pix), ptr(self.pts), stream())
        # with appearance codes the bake uses code 0, as the reference's export does (renderer.py:354-356)
        t0.encode_points(t0._pp(), self.pts, None, self.counters, self.cap, self.enc_tiles, 0)

    def features(self, feats, feats_f32=None):
        """geo_feat of the gathered points, quantised into their texels of feats"""
        call("n2m_s1_geo_feat", ptr(self.enc_tiles), ptr(self.counters), self.cap, ptr(self.t0.wpack), ptr(self.pix), ptr(feats),
             ptr(feats_f32), stream())


def uv_raster(vertices_uv, ft, h, w, glctx=None):
    """dr.rasterize of the atlas: clip positions (vt * 2 - 1, 0, 1), triangles ft, resolution (h, w) (renderer.py:329-338)"""
    uv = vertices_uv * 2.0 - 1.0
    clip = torch.cat((uv, torch.zeros_like(uv[:, :1]), torch.ones_like(uv[:, :1])), dim=-1).contiguous()
    rast, _ = dr.rasterize(glctx or dr.RasterizeCudaContext(vertices_uv.device), clip, ft, (h, w))
    return rast


def uv_features(t0, vertices, triangles, vt, ft, h, w, band_rows=None, contract=None):
    """-> feats [h,w,6] uint8 (geo_feat * 255 truncated at the covered texels, 0 elsewhere), mask [h,w] bool (covered texels).
    `band_rows`: rows per bake band (default: as many as keep a band within MAX_BAND_POINTS texels)."""
    dev = t0.device
    vertices = _as_tensor(vertices, torch.float32, dev); triangles = _as_tensor(triangles, torch.int32, dev)
    vt = _as_tensor(vt, torch.float32, dev); ft = _as_tensor(ft, torch.int32, dev)
    h, w = int(h), int(w)
    validate_mesh(vertices, triangles, vt, ft, h, w)
    contract = t0.cfg.contract if contract is None else bool(contract)
    rast = uv_raster(vt, ft, h, w)
    mask = rast[0, ..., 3] > 0
    feats = torch.zeros(h, w, 6, dtype=torch.uint8, device=dev)
    rows = int(band_rows) if band_rows else max(1, MAX_BAND_POINTS // w)
    rows = max(1, min(rows, h))
    baker = Baker(t0, rows * w)
    overflow = torch.zeros(1, dtype=torch.int32, device=dev)
    for y0 in range(0, h, rows):
        baker.band(rast, vertices, triangles, w, y0, min(h, y0 + rows), feats, contract=contract)
        overflow += baker.counters[2:3]
    if int(overflow.item()) != 0:         # a band holds at most cap texels: cannot happen unless the buffers were resized
        raise RuntimeError("uv_features: point buffer overflow")
    return feats, mask


def inpaint(feats, mask, return_source=False):
    """In place on feats [h,w,6] uint8: the gutter texels (within L1 distance 32 of the mask) copy their Euclidean-nearest boundary texel
    (mask texels within L1 distance 3 of a non-mask texel or of the border); all other non-mask texels become 0.  Ties: smallest row, then
    smallest column of the source.  return_source: also the source texel index per texel (int32 [h,w], -1 where nothing is copied)."""
    h, w = int(feats.shape[0]), int(feats.shape[1])
    if feats.dtype != torch.uint8 or tuple(feats.shape) != (h, w, 6) or not feats.is_contiguous() or not feats.is_cuda:
        raise ValueError("inpaint: feats must be a contiguous CUDA uint8 tensor [h,w,6]")
    m = mask.to(feats.device).reshape(h, w).to(torch.uint8).contiguous()
    scratch = torch.empty(3 * h * w, dtype=torch.uint8, device=feats.device)
    src = torch.empty(h, w, dtype=torch.int32, device=feats.device) if return_source else None
    call("n2m_s1_inpaint", ptr(feats), ptr(m), h, w, ptr(scratch), ptr(src), stream())
    return (feats, src) if return_source else feats


def downscale(feats, ssaa):
    """feats [h,w,6] uint8 -> (feat0, feat1) [h/ssaa, w/ssaa, 3] uint8 RGB: channels 0-2 and 3-5; ssaa 2 averages 2x2 blocks as
    (a + b + c + d + 2) >> 2, which is cv2.resize(INTER_LINEAR) at exactly half size; ssaa 1 splits only."""
    ssaa = int(ssaa)
    if ssaa not in (1, 2):
        raise ValueError("ssaa must be 1 or 2")
    h, w = int(feats.shape[0]), int(feats.shape[1])
    if h % ssaa or w % ssaa:
        raise ValueError("the feature image is not a multiple of ssaa")
    h0, w0 = h // ssaa, w // ssaa
    feats = feats.contiguous()
    feat0 = torch.empty(h0, w0, 3, dtype=torch.uint8, device=feats.device); feat1 = torch.empty_like(feat0)
    call("n2m_s1_ssaa_down2", ptr(feats), h0, w0, ssaa, ptr(feat0), ptr(feat1), stream())
    return feat0, feat1


def bake_features(t0, vertices, triangles, vt, ft, h0, w0, ssaa=2, band_rows=None, contract=None):
    """-> (feat0, feat1): the albedo and specular-feature textures, CUDA uint8 [h0,w0,3] RGB (renderer.py:329-402)."""
    h, w = int(h0) * int(ssaa), int(w0) * int(ssaa)
    feats, mask = uv_features(t0, vertices, triangles, vt, ft, h, w, band_rows=band_rows, contract=contract)
    inpaint(feats, mask)
    del mask
    return downscale(feats, ssaa)


# ---- the UV atlas (csrc/atlas.cu) ----------------------------------------------------------------------------------------------------
# The atlas rule's constants (see uv_unwrap).  At resolution 512 they give 26 charts on icosphere(4) and on the 64^3 marching-cubes
# sphere, 50 on the 64^3 torus, and 897 on the 2,179 faces of the seeded noisy sphere decimated to 10 %, whose rough charts split into
# single faces (tests/test_atlas_cpu.py).
SMALL_CHART = 8          # a chart of fewer faces is small and may merge into a neighbour
MERGE_ROUNDS = 3         # merge rounds
ANGLES = 16              # in-plane rotations k * 90 deg / ANGLES tried per chart
PAD = 2                  # final texels between charts and to the border
BISECT_STEPS = 24        # geometric bisection steps of the common scale over [hi 2^-20, hi]
MERGE_COS = 0.5          # a small chart's faces must all be within 60 deg of the target's axis (the kernel's constant, stated here)


def atlas_tables():
    """(axes [26,3], basis [26,6], rot [ANGLES,2]) float64: the 26 directions normalize(i, j, k), (i, j, k) in {-1, 0, 1}^3 \\ 0 in
    lexicographic order; per axis a right-handed in-plane basis e1 = normalize(cross(h, a)), e2 = cross(a, e1) with h = (0, 0, 1), or
    (1, 0, 0) for the two z axes; (cos, sin) of k * (pi / 2) / ANGLES"""
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


_atlas_tables = {}


def _device_atlas_tables(device):
    key = torch.device(device).index
    if key not in _atlas_tables:
        _atlas_tables[key] = tuple(torch.from_numpy(np.ascontiguousarray(x)).to(device) for x in atlas_tables())
    return _atlas_tables[key]


def _pow2(n):
    return 1 << max(int(n) - 1, 1).bit_length()


@torch.no_grad()
def uv_unwrap(vertices, triangles, resolution, ssaa=2, info=None):
    """The library's UV atlas of a mesh on the device: vertices [V,3] float32, triangles [F,3] int32 -> (vt [Nt,2] float32, ft [F,3] int32,
    vmapping [Nt] int32), all CUDA, with vmapping[ft] == triangles.  The atlas is laid out for a `resolution`^2 texture baked at
    R = resolution * ssaa.  This is a deterministic rule of its own, not xatlas's:

    1. each face's float64 unit normal picks the nearest of 26 axes (the cube's faces, edges and corners; the lowest on a tie), so it
       lies within about 27.6 deg of it: projection stretches area by at most 1.13x and flips no face.  A face that repeats an index or
       whose cross product is zero is a chart of its own (it covers no texel);
    2. faces across an edge of exactly two faces with the same axis share a base chart;
    3. MERGE_ROUNDS rounds: a chart of fewer than SMALL_CHART faces merges into the neighbour it shares the most such edges with (ties:
       the lowest chart id) when all its faces are within 60 deg of that chart's axis and that chart is not merging itself; the merged
       chart keeps the target's axis;
    4. each chart is projected onto its axis's plane and turned by the one of ANGLES angles that gives the least bounding box, then by
       90 deg when the box is taller than wide;
    5. one scale s (final texels per unit length) for every chart: the largest, by bisection, at which next-fit-decreasing-height shelves
       of the charts' ceil(s w) x ceil(s h) rectangles fit, PAD final texels apart and from the border -- on the final texel grid, so no
       texel of the down-sampled texture mixes two charts;
    6. a chart in which two faces cover the same bake-raster texel centre (strictly inside both) splits into its base charts when it is
       a merged chart, else into single faces, and the packing runs again.  A new scale samples the charts anew, so a chart clear at
       one scale may conflict at the next; every split lowers a chart's level (merged, base, single face) and single faces in their own
       rectangles cannot conflict, so the rounds end;
    7. vt has one row per distinct (chart, vertex) in that order, vt = (offset + s * xy) / resolution rounded once to float32.

    `info`, a dict, receives `charts`, `texels_per_unit` (s), `utilization` (the UV area of the faces, of 1) and `split_rounds`.  ValueError
    for malformed input, a bake raster of 2^31 texels or more, or charts that do not fit the texture even at the smallest scale."""
    if not (torch.is_tensor(vertices) and torch.is_tensor(triangles) and vertices.is_cuda):
        raise ValueError("uv_unwrap: vertices and triangles must be tensors, the vertices on a CUDA device")
    if vertices.dim() != 2 or vertices.shape[1] != 3 or triangles.dim() != 2 or triangles.shape[1] != 3:
        raise ValueError("uv_unwrap: vertices [V,3] and triangles [F,3]")
    if vertices.dtype != torch.float32 or triangles.dtype not in (torch.int32, torch.int64):
        raise ValueError("uv_unwrap: vertices must be float32 and triangles int32 or int64")
    resolution, ssaa = int(resolution), int(ssaa)
    R = resolution * ssaa
    if ssaa < 1 or resolution <= 2 * PAD or R * R >= 1 << 31:
        raise ValueError(f"uv_unwrap: texture {resolution} x ssaa {ssaa}: the texture exceeds {2 * PAD} texels and the bake raster holds "
                         "fewer than 2^31 texels")
    dev = vertices.device
    V, Fn = int(vertices.shape[0]), int(triangles.shape[0])
    if 3 * Fn >= 1 << 31:
        raise ValueError("uv_unwrap: at most 2^31 / 3 faces")
    v = vertices.contiguous()
    tri = triangles.to(dev, torch.int32).contiguous()
    if Fn and (int(triangles.min()) < 0 or int(triangles.max()) >= V):
        raise ValueError(f"uv_unwrap: triangles index outside the vertices (0..{V - 1})")
    if V and not bool(torch.isfinite(v).all()):
        raise ValueError("uv_unwrap: vertices must be finite")
    i32 = dict(dtype=torch.int32, device=dev)
    if Fn == 0:
        if info is not None:
            info.update(charts=0, texels_per_unit=0.0, utilization=0.0, split_rounds=0)
        return torch.empty(0, 2, device=dev), torch.empty(0, 3, **i32), torch.empty(0, **i32)
    axes, basis, rot = _device_atlas_tables(dev)
    nrm = torch.empty(Fn, 3, dtype=torch.float64, device=dev)
    bucket, fkeep = torch.empty(Fn, **i32), torch.empty(Fn, dtype=torch.uint8, device=dev)
    call("n2m_atlas_faces", ptr(v), ptr(tri), Fn, ptr(axes), ptr(nrm), ptr(bucket), ptr(fkeep), stream())
    ne = _pow2(6 * Fn)                                                       # 2. base charts
    table, slot_of, ecount, mate = torch.empty(ne, **i32), torch.empty(3 * Fn, **i32), torch.empty(ne, **i32), torch.empty(3 * Fn, **i32)
    call("n2m_clean_edge_table", ptr(tri), Fn, ptr(fkeep), ne, ptr(table), ptr(slot_of), stream())
    parent, base, label, fax = (torch.empty(Fn, **i32) for _ in range(4))
    call("n2m_atlas_base", Fn, ptr(fkeep), ptr(bucket), ptr(table), ptr(slot_of), ne, ptr(ecount), ptr(mate), ptr(parent), ptr(base),
         ptr(label), ptr(fax), stream())
    del table, slot_of, ecount, parent
    count, start, cursor, items, propose = (torch.empty(Fn, **i32) for _ in range(5))
    for _ in range(MERGE_ROUNDS):                                            # 3. small charts
        call("n2m_atlas_chart_count", Fn, ptr(label), ptr(count), stream())
        torch.cumsum(count, 0, dtype=torch.int32, out=start)
        start -= count
        call("n2m_atlas_merge_round", Fn, SMALL_CHART, ptr(nrm), ptr(axes), ptr(bucket), ptr(mate), ptr(count), ptr(start), ptr(cursor),
             ptr(items), ptr(propose), ptr(label), ptr(fax), stream())
    del count, start, cursor, items, propose, mate, nrm
    owner = torch.empty(R * R, **i32)
    nconf, state = torch.empty(1, **i32), torch.empty(2, dtype=torch.float64, device=dev)
    splits = 0
    while True:
        flag = torch.empty(Fn, **i32)                                        # chart indices
        call("n2m_atlas_roots", Fn, ptr(label), ptr(flag), stream())
        incl = torch.cumsum(flag, 0, dtype=torch.int32)
        C = int(incl[-1].item())                                             # read-back: the chart count
        cap = _pow2(C)
        bmin, bmax = torch.empty(C * ANGLES * 2, dtype=torch.int64, device=dev), torch.empty(C * ANGLES * 2, dtype=torch.int64, device=dev)
        orient, org, ext = torch.empty(C, **i32), torch.empty(C, 2, dtype=torch.float64, device=dev), torch.empty(C, 2, dtype=torch.float64, device=dev)
        skey, sval = torch.empty(cap, dtype=torch.int64, device=dev), torch.empty(cap, **i32)
        call("n2m_atlas_orient", ptr(v), ptr(tri), Fn, ptr(label), ptr(incl), ptr(fax), ptr(basis), ptr(rot), ANGLES, C, ptr(bmin), ptr(bmax),
             ptr(orient), ptr(org), ptr(ext), ptr(skey), ptr(sval), stream())
        del bmin, bmax
        call("n2m_atlas_sort", ptr(skey), ptr(sval), C, cap, stream())     # 5. packing
        wid, hgt, nxt, shelf_a, shelf_y = (torch.empty(C, **i32) for _ in range(5))
        prefix, off = torch.empty(C + 1, dtype=torch.int64, device=dev), torch.empty(C, 2, **i32)
        call("n2m_atlas_pack", ptr(ext), ptr(sval), C, resolution, PAD, BISECT_STEPS, ptr(wid), ptr(hgt), ptr(nxt), ptr(shelf_a), ptr(shelf_y),
             ptr(prefix), ptr(off), ptr(state), stream())
        del wid, hgt, nxt, shelf_a, shelf_y, prefix, skey, sval
        scale, fits = state.tolist()                                         # read-back: the scale and whether the charts fit
        if not fits:
            raise ValueError(f"uv_unwrap: {C} charts do not fit a {resolution}^2 texture even at the smallest scale; use a larger resolution")
        conf = torch.empty(C, dtype=torch.uint8, device=dev)                 # 6. texel conflicts
        call("n2m_atlas_conflicts", ptr(v), ptr(tri), Fn, ptr(fkeep), ptr(label), ptr(incl), ptr(fax), ptr(basis), ptr(rot), ptr(orient),
             ptr(org), ptr(off), ptr(state), C, resolution, R, ptr(owner), ptr(conf), ptr(nconf), stream())
        if int(nconf.item()) == 0:                                           # read-back: the conflict count
            break
        merged = torch.empty(C, dtype=torch.uint8, device=dev)
        call("n2m_atlas_split", Fn, C, ptr(incl), ptr(base), ptr(bucket), ptr(conf), ptr(merged), ptr(label), ptr(fax), stream())
        splits += 1
    del owner
    cap = _pow2(3 * Fn)                                                      # 7. emit
    keys, vals = torch.empty(cap, dtype=torch.int64, device=dev), torch.empty(cap, **i32)
    call("n2m_atlas_corner_keys", ptr(tri), Fn, ptr(label), ptr(incl), ptr(keys), ptr(vals), stream())
    call("n2m_atlas_sort", ptr(keys), ptr(vals), 3 * Fn, cap, stream())
    rows = torch.empty(3 * Fn, **i32)
    call("n2m_atlas_row_flags", ptr(keys), 3 * Fn, ptr(rows), stream())
    torch.cumsum(rows, 0, dtype=torch.int32, out=rows)
    Nt = int(rows[-1].item())                                                # read-back: the row count
    vt, ft, vmapping = torch.empty(Nt, 2, device=dev), torch.empty(Fn, 3, **i32), torch.empty(Nt, **i32)
    call("n2m_atlas_emit", ptr(v), ptr(keys), ptr(vals), 3 * Fn, ptr(rows), ptr(fax), ptr(basis), ptr(rot), ptr(orient), ptr(org), ptr(off),
         ptr(state), resolution, ptr(vt), ptr(ft), ptr(vmapping), stream())
    if info is not None:
        info.update(charts=C, texels_per_unit=scale, utilization=uv_area(vt, ft), split_rounds=splits)
    return vt, ft, vmapping


def uv_area(vt, ft):
    """the summed float64 area of the UV triangles (of the unit square)"""
    t = vt.double()[ft.long()]
    d1, d2 = t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]
    return float((0.5 * (d1[:, 0] * d2[:, 1] - d1[:, 1] * d2[:, 0]).abs()).sum())


def unwrap_stage1(s1, resolution):
    """uv_unwrap of every cascade mesh of a Stage1Trainer (s1.cascade_mesh(cas)) for its texture size texture_sizes(resolution, C)[cas] and
    the trainer's ssaa, of the contracted positions when the trainer's cfg.contract (renderer.py:314); the bake itself reads the
    uncontracted ones.  -> (vts, fts): one vt [Nt,2] and ft [F,3] per cascade."""
    vts, fts = [], []
    for cas, size in enumerate(texture_sizes(resolution, s1.cascades)):
        v, f = s1.cascade_mesh(cas)
        v = v.float().contiguous()
        if s1.t0.cfg.contract:
            out = torch.empty_like(v)
            call("n2m_atlas_contract", ptr(v), int(v.shape[0]), ptr(out), stream())
            v = out
        vt, ft, _ = uv_unwrap(v, f, size, ssaa=s1.ssaa)
        vts.append(vt); fts.append(ft)
    return vts, fts


# ---- files ----------------------------------------------------------------------------------------------------------------------
def _np(x, dtype):
    if torch.is_tensor(x):
        x = x.detach().cpu().numpy()
    return np.ascontiguousarray(x, dtype=dtype)


def _rows(fmt, arr):
    return "".join(fmt % tuple(r) for r in arr.tolist())


def write_obj(path, v, f, vt, ft, mtl_name="mesh_0.mtl"):
    """`v x y z`, `vt u (1 - v)`, `f a/at b/bt c/ct` (1-based), the layout of renderer.py:414-429.  Floats are float32 values written with
    9 significant digits, which read back to the same float32."""
    v = _np(v, np.float32); vt = _np(vt, np.float32); f = _np(f, np.int64); ft = _np(ft, np.int64)
    vt_out = np.stack([vt[:, 0], np.float32(1) - vt[:, 1]], axis=1).astype(np.float32)       # float32 arithmetic, as the reference's
    faces = np.stack([f[:, 0] + 1, ft[:, 0] + 1, f[:, 1] + 1, ft[:, 1] + 1, f[:, 2] + 1, ft[:, 2] + 1], axis=1)
    with open(path, "w") as fp:
        fp.write(f"mtllib {mtl_name} \n")
        fp.write(_rows("v %.9g %.9g %.9g \n", v.astype(np.float64)))
        fp.write(_rows("vt %.9g %.9g \n", vt_out.astype(np.float64)))
        fp.write("usemtl defaultMat \n")
        fp.write(_rows("f %d/%d %d/%d %d/%d \n", faces))


def write_mtl(path, texture="feat0_0.jpg"):
    """the material of renderer.py:431-439: map_Kd is the albedo texture"""
    with open(path, "w") as fp:
        fp.write("newmtl defaultMat \nKa 1 1 1 \nKd 1 1 1 \nKs 0 0 0 \nTr 1 \nillum 1 \nNs 0 \n")
        fp.write(f"map_Kd {texture} \n")


def specular_weights(t0):
    """specular_net's weights {net.0.weight [32,6], net.1.weight [3,32]} (fp32) from the trainer's flat parameter vector"""
    st = t0.export_reference_state()
    return {k[len("specular_net."):]: st[k].detach().cpu().numpy() for k in ("specular_net.net.0.weight", "specular_net.net.1.weight")}


def write_mlp_json(path, weights, bound, cascade=1):
    """mlp.json of renderer.py:454-468: each specular_net weight transposed ([in, out]), `bound`, `cascade`"""
    mlp = {k: np.asarray(p, dtype=np.float32).T.tolist() for k, p in weights.items()}
    mlp["bound"] = float(bound)
    mlp["cascade"] = int(cascade)
    with open(path, "w") as fp:
        json.dump(mlp, fp, indent=2)


def write_textures(save_path, feat0, feat1, cas=0):
    """feat0_<cas>.jpg / feat1_<cas>.jpg with cv2's default JPEG settings, BGR channel order (renderer.py:397-407)"""
    import cv2
    for name, img in ((f"feat0_{cas}.jpg", feat0), (f"feat1_{cas}.jpg", feat1)):
        a = _np(img, np.uint8)
        if not cv2.imwrite(os.path.join(save_path, name), np.ascontiguousarray(a[..., ::-1])):
            raise RuntimeError(f"cv2.imwrite failed for {name}")


def texture_sizes(resolution, cascades):
    """the texture size of each cascade (renderer.py:441-452): halved after a cascade while it is > 2048 -- 4096 gives 4096, 2048, 2048, ..."""
    sizes, r = [], int(resolution)
    for _ in range(int(cascades)):
        sizes.append(r)
        if r > 2048:
            r //= 2
    return sizes


def export_stage1(s1, save_path, vt=None, ft=None, resolution=4096, band_rows=None):
    """NeRFRenderer.export_stage1 from a Stage1Trainer (renderer.py:298-468): for every cascade `cas` of the trainer, its mesh
    (s1.cascade_mesh(cas): vertices = base + offsets), the model of its Stage0Trainer (call t0.ema_apply() first to export the EMA
    parameters) and the trainer's ssaa give mesh_{cas}.obj, mesh_{cas}.mtl, feat0_{cas}.jpg, feat1_{cas}.jpg under save_path; then mlp.json
    with `cascade` = the number of cascades.  Without vt / ft the atlas is the library's (unwrap_stage1, one uv_unwrap per cascade).
    Otherwise vt [Nt,2] / ft [F,3] come from the caller's UV unwrap of the mesh (of contract(vertices) when cfg.contract, renderer.py:314);
    a trainer of several cascades takes lists vt[cas] / ft[cas], one unwrap per cascade.  The texture is
    `resolution` for cascade 0 and halves after each cascade while it is > 2048 (texture_sizes).  Returns (feat0, feat1) on the device for
    one mesh, the list of them per cascade for lists."""
    t0 = s1.t0
    C = s1.cascades
    if (vt is None) != (ft is None):
        raise ValueError("export_stage1: pass both vt and ft, or neither (the library's atlas)")
    if vt is None:
        vt, ft = unwrap_stage1(s1, resolution)
        if C == 1:
            vt, ft = vt[0], ft[0]
    per_cascade = isinstance(vt, (list, tuple))
    vts, fts = (list(vt), list(ft)) if per_cascade else ([vt], [ft])
    if len(vts) != C or len(fts) != C:
        raise ValueError(f"export_stage1: the trainer has {C} cascade meshes: pass one (vt, ft) per cascade, as lists")
    os.makedirs(save_path, exist_ok=True)
    feats = []
    for cas, size in enumerate(texture_sizes(resolution, C)):
        v, f = s1.cascade_mesh(cas)
        feat0, feat1 = bake_features(t0, v, f, vts[cas], fts[cas], size, size, ssaa=s1.ssaa, band_rows=band_rows)
        write_textures(save_path, feat0, feat1, cas)
        write_obj(os.path.join(save_path, f"mesh_{cas}.obj"), v, f, vts[cas], fts[cas], mtl_name=f"mesh_{cas}.mtl")
        write_mtl(os.path.join(save_path, f"mesh_{cas}.mtl"), texture=f"feat0_{cas}.jpg")
        feats.append((feat0, feat1))
    write_mlp_json(os.path.join(save_path, "mlp.json"), specular_weights(t0), bound=t0.cfg.bound, cascade=C)
    return feats if per_cascade else feats[0]


# ---- the exported asset, rendered as the viewer draws it -----------------------------------------------------------------------------
SHADE_MODES = {"diffuse": 1, "specular": 2, "full": 3}          # the viewer's `mode` uniform (renderer.html:148-158)


class ExportedMesh:
    """The textured mesh of an export on the device, every cascade concatenated as the viewer draws them into one depth buffer:
    vertices [V,3] float32, triangles [F,3] int32 (indices into the concatenated vertices), st [Nt,2] float32 = the OBJ's texture
    coordinates (s, t) with t = 1 - v as written, ft [F,3] int32 (into the concatenated st), face_offsets [C+1] (host ints; cascade c owns
    faces face_offsets[c] .. face_offsets[c+1]-1), feat0 / feat1 [C] lists of RGB uint8 [H_c,W_c,3] textures, weights
    {net.0.weight [32,6], net.1.weight [3,32]} float32 ([out, in]), bound."""

    def __init__(self, vertices, triangles, st, ft, feat0, feat1, weights, bound=1.0, device="cuda"):
        C = len(vertices)
        if not (len(triangles) == len(st) == len(ft) == len(feat0) == len(feat1) == C and C > 0):
            raise ValueError("ExportedMesh: one (vertices, triangles, st, ft, feat0, feat1) per cascade")
        dev = torch.device(device)
        vs, fs, sts, fts, self.face_offsets = [], [], [], [], [0]
        v_off = t_off = 0
        for v, f, s, t in zip(vertices, triangles, st, ft):
            v = _np(v, np.float32); s = _np(s, np.float32)
            f = _np(f, np.int64); t = _np(t, np.int64)
            if f.shape != t.shape:
                raise ValueError("ExportedMesh: ft must match triangles row for row")
            vs.append(v); sts.append(s); fs.append(f + v_off); fts.append(t + t_off)
            v_off += v.shape[0]; t_off += s.shape[0]
            self.face_offsets.append(self.face_offsets[-1] + f.shape[0])
        self.vertices = torch.from_numpy(np.concatenate(vs)).to(dev).contiguous()
        self.triangles = torch.from_numpy(np.concatenate(fs).astype(np.int32)).to(dev).contiguous()
        self.st = torch.from_numpy(np.concatenate(sts)).to(dev).contiguous()
        self.ft = torch.from_numpy(np.concatenate(fts).astype(np.int32)).to(dev).contiguous()
        self.feat0 = [_as_tensor(x, torch.uint8, dev) for x in feat0]
        self.feat1 = [_as_tensor(x, torch.uint8, dev) for x in feat1]
        for a, b in zip(self.feat0, self.feat1):
            if a.dim() != 3 or a.shape[2] != 3 or a.shape != b.shape:
                raise ValueError("ExportedMesh: feat0 / feat1 of a cascade must both be [H,W,3]")
        self.weights = {k: _np(weights[k], np.float32) for k in ("net.0.weight", "net.1.weight")}
        if self.weights["net.0.weight"].shape != (32, 6) or self.weights["net.1.weight"].shape != (3, 32):
            raise ValueError("ExportedMesh: specular_net weights must be [32,6] and [3,32]")
        self.bound = float(bound)
        # the kernel's view of it: face offsets, texture pointers and sizes, the MLP weights, on the device
        self._offsets = torch.tensor(self.face_offsets, dtype=torch.int32, device=dev)
        self._feat0_ptrs = torch.tensor([t.data_ptr() for t in self.feat0], dtype=torch.int64, device=dev)
        self._feat1_ptrs = torch.tensor([t.data_ptr() for t in self.feat1], dtype=torch.int64, device=dev)
        self._tex_size = torch.tensor([[t.shape[0], t.shape[1]] for t in self.feat0], dtype=torch.int32, device=dev)
        self._mlp = torch.from_numpy(np.concatenate([self.weights["net.0.weight"].ravel(), self.weights["net.1.weight"].ravel()])).to(dev)
        self._topology = None

    @property
    def cascades(self):
        return len(self.feat0)

    def topology(self):
        """the edge hash of the concatenated mesh (antialias), built on first use"""
        if self._topology is None:
            self._topology = dr.TopologyHash(self.triangles)
        return self._topology

    @classmethod
    def from_export(cls, s1, vt, ft, feats):
        """The asset export_stage1(s1, ..., vt, ft) writes, from its in-memory results: `feats` is its return value ((feat0, feat1), or a
        list of them per cascade, with vt / ft lists), the mesh is s1.cascade_mesh(cas), the weights are the trainer's.  The texture
        coordinates are the file's, t = float32(1 - v); the textures are the ones before the JPEG encode."""
        per_cascade = isinstance(vt, (list, tuple))
        vts, fts = (list(vt), list(ft)) if per_cascade else ([vt], [ft])
        feats = list(feats) if per_cascade else [feats]
        meshes = [s1.cascade_mesh(cas) for cas in range(s1.cascades)]
        st = []
        for x in vts:
            x = _np(x, np.float32)
            st.append(np.stack([x[:, 0], np.float32(1) - x[:, 1]], axis=1).astype(np.float32))          # write_obj's float32 expression
        return cls([v for v, _ in meshes], [f for _, f in meshes], st, fts, [a for a, _ in feats], [b for _, b in feats],
                   specular_weights(s1.t0), bound=s1.t0.cfg.bound, device=s1.t0.device)


def read_obj(path):
    """(v [V,3] float32, st [Nt,2] float32, f [F,3] int64, ft [F,3] int64; 0-based) of an OBJ in write_obj's layout: the `v` lines, the `vt`
    lines, `usemtl`, the `f a/at b/bt c/ct` lines -- parsed block by block with numpy, the %.9g floats back to the float32 values written."""
    with open(path) as fp:
        text = fp.read()
    a, b, c = text.find("\nv "), text.find("\nvt "), text.find("\nf ")
    if min(a, b, c) < 0 or not a < b < c:
        raise ValueError(f"{path}: not an OBJ in the layout write_obj writes (v, vt, then f lines)")
    v = np.array(text[a:b].split()).reshape(-1, 4)[:, 1:].astype(np.float32)
    vt_block = text[b:text.find("\nusemtl", b)] if text.find("\nusemtl", b) >= 0 else text[b:c]
    st = np.array(vt_block.split()).reshape(-1, 3)[:, 1:].astype(np.float32)
    faces = np.array(text[c:].replace("/", " ").split()).reshape(-1, 7)[:, 1:].astype(np.int64) - 1
    return v, st, faces[:, 0::2], faces[:, 1::2]


def load_exported(path, device="cuda"):
    """The asset export_stage1 wrote under `path`: mlp.json (the specular_net weights, stored [in, out], transposed back; bound; the
    cascade count), mesh_{cas}.obj and feat0_{cas}.jpg / feat1_{cas}.jpg (cv2.imread, BGR -> RGB) for every cascade -> ExportedMesh."""
    import cv2
    with open(os.path.join(path, "mlp.json")) as fp:
        mlp = json.load(fp)
    weights = {k: np.asarray(mlp[k], dtype=np.float32).T for k in ("net.0.weight", "net.1.weight")}
    vs, fs, sts, fts, f0s, f1s = [], [], [], [], [], []
    for cas in range(int(mlp["cascade"])):
        v, st, f, ft = read_obj(os.path.join(path, f"mesh_{cas}.obj"))
        vs.append(v); sts.append(st); fs.append(f); fts.append(ft)
        for name, out in ((f"feat0_{cas}.jpg", f0s), (f"feat1_{cas}.jpg", f1s)):
            img = cv2.imread(os.path.join(path, name))
            if img is None:
                raise FileNotFoundError(os.path.join(path, name))
            out.append(np.ascontiguousarray(img[..., ::-1]))
    return ExportedMesh(vs, fs, sts, fts, f0s, f1s, weights, bound=mlp["bound"], device=device)


@torch.no_grad()
def render_exported(asset, mvp, campos, h0, w0, ssaa=1, bg_color=1.0, shading="full", antialias=False, glctx=None):
    """The asset as the viewer draws it (renderer.html:54-160): all cascades rasterized together at ssaa * (h0, w0) with the clip-space
    transform mvp [4,4] (nvdiffrast conventions, as Stage1Trainer), the fragment shader on every covered sample (n2m_s1_asset_shade:
    nearest texel, specular_net in fp32 with the view direction normalize(x - campos)), optionally dr.antialias, then the evaluation
    compose of Stage1Trainer.render (n2m_s1_render_compose).  Returns (image [h0*w0,3], weights_sum [h0*w0], depth [h0*w0]).
    ssaa=1 without antialias is pixel for pixel what the viewer draws; ssaa=2 with antialias compares with Stage1Trainer.render."""
    from .stage1 import bg_image
    if shading not in SHADE_MODES:
        raise ValueError(f"shading must be one of {sorted(SHADE_MODES)}")
    ssaa = int(ssaa)
    if ssaa not in (1, 2):
        raise ValueError("ssaa must be 1 or 2")
    dev = asset.vertices.device
    h0, w0 = int(h0), int(w0)
    h, w = h0 * ssaa, w0 * ssaa
    Q = h0 * w0
    bg = bg_image(bg_color, Q, dev)
    cam = [float(x) for x in (campos.tolist() if torch.is_tensor(campos) else np.asarray(campos, dtype=np.float64).ravel())]
    mvp = mvp.to(dev, torch.float32).contiguous()
    vclip = (torch.nn.functional.pad(asset.vertices, (0, 1), value=1.0) @ mvp.T).contiguous()
    rast, _ = dr.rasterize(glctx or dr.RasterizeCudaContext(dev), vclip[None], asset.triangles, (h, w))
    img = torch.empty(h * w, 4, device=dev)
    call("n2m_s1_asset_shade", ptr(rast), h * w, ptr(asset.vertices), ptr(asset.triangles), ptr(asset.st), ptr(asset.ft), ptr(asset._offsets),
         asset.cascades, ptr(asset._feat0_ptrs), ptr(asset._feat1_ptrs), ptr(asset._tex_size), ptr(asset._mlp), cam[0], cam[1], cam[2],
         SHADE_MODES[shading], ptr(img), stream())
    if antialias:
        th = asset.topology()
        aa = torch.empty_like(img)
        call("n2m_antialias_forward", ptr(img), ptr(rast), ptr(vclip), ptr(asset.triangles), ptr(th.keys), ptr(th.opp), th.slots, h, w, 4,
             ptr(aa), stream())
        img = aa
    image = torch.empty(Q, 3, device=dev); weights_sum = torch.empty(Q, device=dev); depth = torch.empty(Q, device=dev)
    call("n2m_s1_render_compose", ptr(img), ptr(rast), ptr(bg), h0, w0, ssaa, ptr(image), ptr(weights_sum), ptr(depth), stream())
    return image, weights_sum, depth
