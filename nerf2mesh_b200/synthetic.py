"""Synthetic, seeded stand-ins for the datasets the reference trains on (no datasets or network
are available): Lego-like orbit cameras, ray sampling exactly as the reference's collate does it,
an analytic "bricks" scene (axis-aligned coloured boxes) with its occupancy grid in the
reference's Morton/bitfield layout, and analytic ground-truth colours for those rays.

Shapes / conventions: 100 poses on the upper hemisphere at radius
4.031 * 0.8, 800x800, fl = 400 / tan(0.5 * 0.6911), rays exactly as nerf/utils.py:282-290
(unnormalised directions, -z forward, y flipped), pixel ids via randint as provider.py:303 and
utils.py:271.  Pure torch/numpy host code; no kernels.
"""
import math

import numpy as np
import torch

LEGO_RADIUS = 4.031 * 0.8
LEGO_FOVX = 0.6911
LEGO_HW = 800


def look_at_pose(cam_pos):
    """camera-to-world, OpenGL convention (camera looks down -z, y up), looking at the origin."""
    c = np.asarray(cam_pos, np.float64)
    fwd = -c / np.linalg.norm(c)                 # viewing direction
    up = np.array([0.0, 0.0, 1.0])
    if abs(np.dot(fwd, up)) > 0.999:
        up = np.array([0.0, 1.0, 0.0])
    right = np.cross(fwd, up); right /= np.linalg.norm(right)
    true_up = np.cross(right, fwd)
    pose = np.eye(4)
    pose[:3, 0] = right
    pose[:3, 1] = true_up
    pose[:3, 2] = -fwd
    pose[:3, 3] = c
    return pose


def orbit_cameras(n=100, radius=LEGO_RADIUS, seed=0, min_elev=0.05, max_elev=1.3):
    """n camera-to-world poses on the upper hemisphere (seeded)."""
    rng = np.random.default_rng(seed)
    az = rng.uniform(0, 2 * math.pi, n)
    el = rng.uniform(min_elev, max_elev, n)
    pos = np.stack([radius * np.cos(el) * np.cos(az), radius * np.cos(el) * np.sin(az), radius * np.sin(el)], -1)
    return torch.from_numpy(np.stack([look_at_pose(p) for p in pos]).astype(np.float32))


def lego_intrinsics(H=LEGO_HW, W=LEGO_HW, fovx=LEGO_FOVX):
    fl = 0.5 * W / math.tan(0.5 * fovx)
    return np.array([fl, fl, W / 2, H / 2], np.float32)


def sample_rays(poses, intrinsics, H, W, N, generator=None):
    """Random (image, pixel) pairs -> rays_o, rays_d [N,3] float32 (host tensors).
    Mirrors provider.py:303 (image index per ray) + utils.py:242-290 (pixel centre +0.5,
    directions ((i-cx)/fx, -(j-cy)/fy, -1) rotated by the pose, unnormalised)."""
    fx, fy, cx, cy = [float(v) for v in intrinsics]
    img = torch.randint(0, poses.shape[0], (N,), generator=generator)
    pix = torch.randint(0, H * W, (N,), generator=generator)
    i = (pix % W).float() + 0.5
    j = (pix // W).float() + 0.5
    dirs = torch.stack([(i - cx) / fx, -(j - cy) / fy, -torch.ones_like(i)], -1)        # [N,3]
    R = poses[img, :3, :3]
    rays_d = torch.einsum("nij,nj->ni", R, dirs).contiguous()
    rays_o = poses[img, :3, 3].contiguous()
    return rays_o, rays_d, img, pix


# ---- analytic bricks scene ------------------------------------------------------------------
def make_bricks(n_boxes=40, extent=0.7, seed=1, min_size=0.08, max_size=0.25):
    """Seeded axis-aligned boxes inside [-extent, extent]^3: (lo [K,3], hi [K,3], rgb [K,3])."""
    rng = np.random.default_rng(seed)
    size = rng.uniform(min_size, max_size, (n_boxes, 3))
    ctr = rng.uniform(-extent, extent, (n_boxes, 3))
    lo = np.clip(ctr - size, -extent, extent)
    hi = np.clip(ctr + size, -extent, extent)
    rgb = rng.uniform(0.1, 0.95, (n_boxes, 3))
    return (torch.from_numpy(lo.astype(np.float32)), torch.from_numpy(hi.astype(np.float32)),
            torch.from_numpy(rgb.astype(np.float32)))


def make_garden_bricks(seed=1):
    """Garden-like content for the bound-16 / 5-cascade configuration: the central object of
    make_bricks(), a ground slab through the scene and a sparse shell of far boxes, so that samples fall inside AND outside the unit
    cube and in every cascade."""
    lo, hi, rgb = make_bricks(seed=seed)
    rng = np.random.default_rng(seed + 100)
    extra_lo, extra_hi, extra_rgb = [[-6.0, -6.0, -0.95]], [[6.0, 6.0, -0.8]], [[0.35, 0.5, 0.3]]          # ground
    for _ in range(36):                                                                                    # far shell
        r = rng.uniform(5.0, 13.0); az = rng.uniform(0, 2 * math.pi); el = rng.uniform(-0.05, 0.5)
        c = np.array([r * math.cos(el) * math.cos(az), r * math.cos(el) * math.sin(az), r * math.sin(el)])
        sz = rng.uniform(0.4, 1.6, 3)
        extra_lo.append(list(np.clip(c - sz, -15.5, 15.5))); extra_hi.append(list(np.clip(c + sz, -15.5, 15.5)))
        extra_rgb.append(list(rng.uniform(0.1, 0.95, 3)))
    f = lambda a: torch.tensor(a, dtype=torch.float32)
    return torch.cat([lo, f(extra_lo)]), torch.cat([hi, f(extra_hi)]), torch.cat([rgb, f(extra_rgb)])


def garden_scene(H=128, bound=16.0, seed=1):
    """(density_grid [5, H^3], bitfield, bricks) of the garden-like scene"""
    bricks = make_garden_bricks(seed)
    cascades = 1 + math.ceil(math.log2(bound))
    grid = occupancy_from_bricks(bricks, H, bound, cascades)
    return grid, packbits_host(grid), bricks


def render_bricks(rays_o, rays_d, bricks):
    """Analytic first-hit render: returns rgba [N,4] (alpha 1 on hit, 0 on miss)."""
    lo, hi, rgb = bricks
    o = rays_o[:, None, :]; d = rays_d[:, None, :]
    inv = 1.0 / torch.where(d.abs() < 1e-9, torch.full_like(d, 1e-9), d)
    t0 = (lo[None] - o) * inv
    t1 = (hi[None] - o) * inv
    tmin = torch.minimum(t0, t1).amax(-1)
    tmax = torch.maximum(t0, t1).amin(-1)
    hit = (tmax >= tmin) & (tmax > 0)
    tmin = torch.where(hit, tmin.clamp(min=0), torch.full_like(tmin, float("inf")))
    t_first, k = tmin.min(-1)
    any_hit = torch.isfinite(t_first)
    col = rgb[k] * any_hit[:, None]
    return torch.cat([col, any_hit[:, None].float()], -1)


def _morton_np(c):
    def spread(v):
        v = v.astype(np.uint64)
        v = (v | (v << 16)) & 0x030000FF
        v = (v | (v << 8)) & 0x0300F00F
        v = (v | (v << 4)) & 0x030C30C3
        v = (v | (v << 2)) & 0x09249249
        return v
    return (spread(c[..., 0]) | (spread(c[..., 1]) << 1) | (spread(c[..., 2]) << 2)).astype(np.int64)


def occupancy_from_bricks(bricks, H=128, bound=1.0, cascades=1, dilate=1):
    """density_grid float32 [cascades, H^3] in the reference's layout (cascade-major, Morton-ordered
    cells, renderer.py:1100-1118) with 1.0 inside (dilated) bricks, 0 elsewhere."""
    lo, hi, _ = bricks
    lo = lo.numpy().astype(np.float64); hi = hi.numpy().astype(np.float64)
    ax = np.arange(H)
    coords = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    mort = _morton_np(coords)
    grid = np.zeros((cascades, H ** 3), np.float32)
    for cas in range(cascades):
        b = min(2 ** cas, bound)
        cell = 2 * b / H
        pad = dilate * cell
        occ = np.zeros((H, H, H), bool)
        # cell centre c_i = (i + 0.5) * cell - b lies in [lo - pad, hi + pad]  <=>  i in [ceil(.), floor(.)]
        i0 = np.ceil((lo - pad + b) / cell - 0.5 - 1e-9).astype(np.int64).clip(0, H)
        i1 = np.floor((hi + pad + b) / cell - 0.5 + 1e-9).astype(np.int64).clip(-1, H - 1)
        for k in range(len(lo)):
            if (i0[k] <= i1[k]).all():
                occ[i0[k, 0]:i1[k, 0] + 1, i0[k, 1]:i1[k, 1] + 1, i0[k, 2]:i1[k, 2] + 1] = True
        grid[cas, mort] = occ.reshape(-1).astype(np.float32)
    return torch.from_numpy(grid)


def packbits_host(grid, thresh=0.5):
    """host-side packbits (bit i of byte n <-> cell 8n+i), for building synthetic inputs only."""
    g = grid.reshape(-1, 8).numpy() > thresh
    return torch.from_numpy((g.astype(np.uint8) << np.arange(8, dtype=np.uint8)).sum(-1).astype(np.uint8))


def occupancy_regime(regime, H=128, cascades=1, bound=1.0, seed=1):
    """'cold' (everything occupied), 'mid' (~30 % cells), 'converged' (bricks; ~16 % of cells, ~70 samples/ray => M ~ 2^18 at 4096 rays).
    Returns (density_grid [cas, H^3] float32, bitfield uint8 [cas*H^3/8], bricks)."""
    bricks = make_bricks(seed=seed)
    if regime == "cold":
        grid = torch.ones(cascades, H ** 3)
    elif regime == "mid":
        g = torch.Generator().manual_seed(seed)
        # blocky 30 %: occupancy decided per 8^3 super-cell so rays see coherent runs
        sc = (torch.rand((H // 8) ** 3, generator=g) < 0.30)
        ax = np.arange(H)
        coords = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
        sidx = (coords[:, 0] // 8) * (H // 8) ** 2 + (coords[:, 1] // 8) * (H // 8) + coords[:, 2] // 8
        grid = torch.zeros(cascades, H ** 3)
        grid[:, torch.from_numpy(_morton_np(coords))] = sc[torch.from_numpy(sidx)].float()
    elif regime == "converged":
        grid = occupancy_from_bricks(bricks, H, bound, cascades)
    else:
        raise ValueError(regime)
    return grid, packbits_host(grid), bricks


# ---- synthetic closed meshes and projections for stage 1 ----
def icosphere(subdiv=3, radius=0.6):
    t = (1.0 + 5 ** 0.5) / 2
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], np.float64)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6], [7, 1, 8],
                  [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]], np.int64)
    for _ in range(subdiv):
        cache, verts = {}, list(v)

        def mid(a, b):
            k = (min(a, b), max(a, b))
            if k not in cache:
                m = (verts[a] + verts[b]) / 2
                verts.append(m / np.linalg.norm(m)); cache[k] = len(verts) - 1
            return cache[k]

        nf = []
        for a, b, c in f:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        v, f = np.array(verts), np.array(nf, np.int64)
    return (v * radius).astype(np.float32), f.astype(np.int32)


def perspective_mvp(cam_pos, fovy=0.6911, aspect=1.0, near=0.05, far=10.0):
    """OpenGL-style projection * view for a camera at cam_pos looking at the origin (y up); returns [4,4] float32"""
    c = np.asarray(cam_pos, np.float64)
    fwd = -c / np.linalg.norm(c)
    up = np.array([0.0, 0.0, 1.0])
    if abs(np.dot(fwd, up)) > 0.999:
        up = np.array([0.0, 1.0, 0.0])
    right = np.cross(fwd, up); right /= np.linalg.norm(right)
    tup = np.cross(right, fwd)
    view = np.eye(4)
    view[0, :3], view[1, :3], view[2, :3] = right, tup, -fwd
    view[:3, 3] = -view[:3, :3] @ c
    f = 1.0 / np.tan(fovy / 2)
    proj = np.array([[f / aspect, 0, 0, 0], [0, f, 0, 0], [0, 0, (far + near) / (near - far), 2 * far * near / (near - far)], [0, 0, -1, 0]])
    return (proj @ view).astype(np.float32)
