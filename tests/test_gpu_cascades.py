"""GPU: unbounded scenes through stage 1 -- the outer-cascade meshes of csrc/cascade.cu (occupancy volume against torch's trilinear
F.interpolate, export_outer_meshes against the CPU oracle chain, mark_unseen_triangles against the reference's torch expression), the
stage-1 step over several cascade meshes against the same step on their concatenation, contraction on the stage-1 hot path, and the
per-cascade export."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cascade_oracle as CO
import texture_oracle as TO
from nerf2mesh_b200 import mesh as M
from nerf2mesh_b200 import raster as dr
from nerf2mesh_b200 import synthetic as S
from nerf2mesh_b200 import texture as X
from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
from nerf2mesh_b200.stage1 import Stage1Trainer
from nerf2mesh_b200.train_synthetic import full_image_rays
from oracle import mcubes_oracle as MO
from test_gpu_refine import _snapshot

pytestmark = pytest.mark.gpu

H = 128


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """the trainers, captured graphs and 256^3 volumes of this module are freed before the next module runs"""
    yield
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _dense(grid_row):
    """[H^3] Morton-ordered -> [H,H,H] (occ[x,y,z] = grid[morton(x,y,z)], renderer.py:618-619)"""
    ax = np.arange(H)
    coords = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    return grid_row[torch.from_numpy(S._morton_np(coords)).to(grid_row.device)].reshape(H, H, H)


@pytest.mark.parametrize("R", [128, 200, 256])
def test_occupancy_volume_matches_torch_trilinear(R):
    grid, _, _ = S.garden_scene(bound=16.0)
    g = torch.Generator().manual_seed(R)
    row = (grid[2] * torch.rand(H ** 3, generator=g) * 20.0).cuda()          # continuous densities around the threshold
    nan_cells = torch.randint(0, H ** 3, (300,), generator=g).cuda()
    row[nan_cells] = float("nan")
    thresh = 5.0
    vol = M.outer_occupancy(row, H, R, thresh)
    ref_v = F.interpolate(_dense(row)[None, None], [R] * 3, mode="trilinear")[0, 0]
    ref = (torch.nan_to_num(ref_v, 0) > thresh).float()
    torch.cuda.synchronize()
    assert vol.shape == (R, R, R) and set(vol.unique().tolist()) <= {0.0, 1.0}
    diff = vol != ref
    near = (ref_v - thresh).abs() <= 1e-6 * max(1.0, abs(thresh))
    assert not (diff & ~near).any()
    assert diff.sum().item() <= 1e-5 * R ** 3
    nan_taps = torch.isnan(ref_v)
    assert nan_taps.sum().item() >= 300 * (1 if R == H else 2) * 0.5 and not vol[nan_taps].any()
    assert ref.sum().item() > 1000


def _garden_trainer(bound=16.0):
    grid, bits, _ = S.garden_scene(bound=bound)
    t0 = Stage0Trainer(Stage0Config(bound=bound, num_rays=1024, max_samples=1024 * 64), seed=0)
    t0.set_occupancy(bits, grid)
    t0.mean_density = torch.tensor([0.5], device=t0.device)               # the garden grid is 0/1: threshold min(0.5, 10)
    return t0


def test_export_outer_meshes_matches_the_oracle_chain(tmp_path):
    t0 = _garden_trainer()
    R = 256
    meshes = M.export_outer_meshes(t0, str(tmp_path), env_reso=R)
    torch.cuda.synchronize()
    assert t0.cfg.cascade == 5 and len(meshes) >= 3
    aabb = t0.aabb.cpu().numpy().astype(np.float64).tolist()
    for cas in range(1, 5):
        vol = M.outer_occupancy(t0.density_grid[cas], H, R, 0.5).cpu().numpy()
        vi, fi = MO.marching_cubes(vol, 0.5)
        v_ref, f_ref = CO.outer_chain(vi, fi, R, min(2 ** cas, 16.0), aabb)
        path = tmp_path / f"mesh_{cas}.ply"
        if v_ref.shape[0] == 0:
            assert cas not in meshes and not path.exists()
            continue
        v, f = meshes[cas]
        assert np.array_equal(v.cpu().numpy(), v_ref), cas                      # bit-equal
        assert np.array_equal(f.cpu().numpy(), f_ref), cas
        pv, pf = M.read_ply(path)
        assert np.array_equal(pv, v_ref) and np.array_equal(pf, f_ref)
    assert not (tmp_path / "mesh_0.ply").exists()


def test_all_centre_cascade_writes_no_file(tmp_path):
    t0 = Stage0Trainer(Stage0Config(bound=4.0, num_rays=1024, max_samples=1024 * 64), seed=0)
    grid = torch.zeros(3, H ** 3)
    dense = torch.zeros(H, H, H); dense[48:80, 48:80, 48:80] = 1.0          # cascade 1: a box well inside the centre (|p| < 0.45)
    ax = np.arange(H)
    coords = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    grid[1, torch.from_numpy(S._morton_np(coords))] = dense.reshape(-1)
    t0.set_occupancy(S.packbits_host(grid), grid)                            # cascade 2: empty
    t0.mean_density = torch.tensor([0.5], device=t0.device)
    vol = M.outer_occupancy(t0.density_grid[1], H, 256, 0.5)
    assert M.marching_cubes(vol, 0.5)[0].shape[0] > 0                        # cascade 1 has a surface, all of it in the centre box
    assert M.export_outer_meshes(t0, str(tmp_path)) == {}
    assert os.listdir(tmp_path) == []


def _views(h0, w0, n=3, scale=1.6, seed=1):
    g = torch.Generator().manual_seed(seed)
    cams = [np.array([1.5, 1.1, 0.9]), np.array([-1.2, 1.4, 1.0]), np.array([0.4, -1.6, 1.2]), np.array([-1.0, -1.0, 1.6])][:n]
    out = []
    for cam in cams:
        cam = cam * scale
        pose = torch.from_numpy(S.look_at_pose(cam).astype(np.float32))
        intr = S.lego_intrinsics(h0, w0)
        _, rays_d = full_image_rays(pose, intr, h0, w0)
        mvp = S.perspective_mvp(cam, fovy=2 * np.arctan(0.5 * h0 / intr[1]), aspect=w0 / h0, far=20.0)
        mvp[1] *= -1
        gt = torch.rand(h0 * w0, 4, generator=g); gt[:, 3] = (gt[:, 3] > 0.5).float()
        bg = torch.rand(h0 * w0, 3, generator=g)
        out.append((torch.from_numpy(np.ascontiguousarray(mvp, np.float32)).cuda(), rays_d.cuda().contiguous(), gt.cuda(), bg.cuda()))
    return out


def test_mark_unseen_triangles_equals_the_reference_expression():
    v, f = S.icosphere(3, 0.6)
    vin, fin = S.icosphere(0, 0.2)                                          # a small sphere inside the big one: hidden from every view
    vt = torch.from_numpy(np.concatenate([v, vin]).astype(np.float32)).cuda()
    ft = torch.from_numpy(np.concatenate([f, fin + v.shape[0]]).astype(np.int32)).cuda()
    Fn = ft.shape[0]
    views = _views(96, 96, n=4)
    mvps = torch.stack([m for m, *_ in views])
    unseen = M.mark_unseen_triangles(vt, ft, mvps, 96, 96)
    # renderer.py:962-977 on this library's rasteriser output
    mask = torch.zeros_like(ft[:, 0])
    glctx = dr.RasterizeCudaContext("cuda")
    ids = []
    for mvp in mvps:
        clip = torch.matmul(F.pad(vt, pad=(0, 1), mode="constant", value=1.0), torch.transpose(mvp, 0, 1)).float().unsqueeze(0)
        rast, _ = dr.rasterize(glctx, clip, ft, (96, 96))
        trig_id = rast[..., -1].long().view(-1) - 1
        mask[trig_id] += 1
        ids.append(trig_id)
    ref = mask == 0
    torch.cuda.synchronize()
    assert unseen.dtype == torch.bool and torch.equal(unseen, ref)
    ids = torch.cat(ids)
    assert (ids < 0).any() and not (ids == Fn - 1).any()                   # the last face is never rendered ...
    assert not unseen[Fn - 1]                                              # ... yet counts as seen (index -1 wraps)
    assert unseen[f.shape[0]:Fn - 1].all() and unseen[:f.shape[0]].any() and not unseen[:f.shape[0]].all()


def _cascade_meshes():
    """three cascade meshes of a bound-4 scene: the inner sphere, a surrounding sphere (the background the cameras sit inside) and a
    small blob below the inner one"""
    v0, f0 = S.icosphere(3, 0.6)
    v1, f1 = S.icosphere(2, 3.8)
    v2, f2 = S.icosphere(1, 0.3)
    v2 = v2 + np.float32([0.0, 0.0, -1.0])
    return [torch.from_numpy(np.asarray(x, np.float32)) for x in (v0, v1, v2)], [torch.from_numpy(np.asarray(x, np.int32)) for x in (f0, f1, f2)]


def _bound4_trainer(contract=False):
    cfg = Stage0Config(bound=4.0, contract=contract, num_rays=1024, max_samples=1024 * 64)
    t0 = Stage0Trainer(cfg, seed=5)
    grid, bits, bricks = S.occupancy_regime("converged", cascades=cfg.cascade, bound=cfg.bound)
    t0.set_occupancy(bits, grid)
    g = torch.Generator().manual_seed(0)
    poses = S.orbit_cameras(100, seed=0)
    for _ in range(5):                   # non-trivial colour parameters
        ro, rd, _, _ = S.sample_rays(poses, S.lego_intrinsics(), 800, 800, 1024, g)
        t0.step(ro, rd, S.render_bricks(ro, rd, bricks), torch.rand(1024, 3, generator=g), torch.rand(1024, generator=g), use_graph=False)
    torch.cuda.synchronize()
    return t0


ORDER = [0, 1, 2, 0, 1, 2]


def test_cascaded_step_equals_the_concatenated_step():
    t0 = _bound4_trainer()
    assert t0.cfg.cascade == 3
    vs, fs = _cascade_meshes()
    cat_v = torch.cat(vs)
    cat_f = torch.cat([fs[0], fs[1] + vs[0].shape[0], fs[2] + vs[0].shape[0] + vs[1].shape[0]])
    kw = dict(ssaa=2, antialias=True, refine=True)
    views = _views(64, 64)
    restore = _snapshot(t0)
    results = {}
    for name in ("cascaded", "concatenated"):
        for use_graph in (False, True):
            restore()
            s1 = Stage1Trainer(t0, vs, fs, 64, 64, **kw) if name == "cascaded" else Stage1Trainer(t0, cat_v, cat_f, 64, 64, **kw)
            for k in ORDER:
                s1.step(*views[k], use_graph=use_graph)
            torch.cuda.synchronize()
            results[name, use_graph] = (s1, s1.rast.clone(), s1.face_counts.clone(), s1.face_errors.clone(), s1.image.clone(), s1.read_loss())
    for use_graph in (False, True):
        a, b = results["cascaded", use_graph], results["concatenated", use_graph]
        assert a[0].f_cumsum == [0, fs[0].shape[0], fs[0].shape[0] + fs[1].shape[0], cat_f.shape[0]] and b[0].f_cumsum == [0, cat_f.shape[0]]
        assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
        assert torch.allclose(a[3], b[3], rtol=1e-4, atol=1e-6), (a[3] - b[3]).abs().max().item()
        assert (a[4] - b[4]).abs().max().item() <= 2e-3 and abs(a[5] - b[5]) <= 1e-3 * abs(b[5])
        ids = a[1][0, ..., 3]
        for c in range(3):                                                  # every cascade is on screen
            assert ((ids > a[0].f_cumsum[c]) & (ids <= a[0].f_cumsum[c + 1])).any(), c
        s1 = a[0]
        mask, _ = s1.refine_mask()
        f1 = s1.f_cumsum[1]
        err, cnt = s1.face_errors[:f1].cpu().numpy().copy(), s1.face_counts[:f1].cpu().numpy()
        seen = cnt > 0
        err[seen] /= cnt[seen]
        t_ref, t_dec = np.percentile(err[seen], 90), np.percentile(err[seen], 50)
        ref = np.zeros_like(err); ref[(err > t_ref) & seen] = 2; ref[(err < t_dec) & seen] = 1
        assert mask.shape == (f1,) and np.array_equal(mask.cpu().numpy(), ref)


def test_cascaded_replace_mesh_rebases_the_outer_cascades():
    t0 = _bound4_trainer()
    vs, fs = _cascade_meshes()
    s1 = Stage1Trainer(t0, vs, fs, 64, 64, ssaa=2, antialias=True, refine=True, lr_vert=1e-4)
    views = _views(64, 64)
    for k in ORDER:
        s1.step(*views[k], use_graph=True)
    torch.cuda.synchronize()
    assert s1.offsets.abs().max().item() > 0
    before = [s1.cascade_mesh(c)[0].clone() for c in range(3)]
    assert torch.equal(s1.vertices, s1.base_vertices + s1.offsets)
    v_new, f_new = S.icosphere(2, 0.6)
    s1.replace_mesh(torch.from_numpy(v_new), torch.from_numpy(f_new))
    V0, F0 = v_new.shape[0], f_new.shape[0]
    assert s1.v_cumsum == [0, V0, V0 + vs[1].shape[0], V0 + vs[1].shape[0] + vs[2].shape[0]]
    assert s1.f_cumsum == [0, F0, F0 + fs[1].shape[0], F0 + fs[1].shape[0] + fs[2].shape[0]]
    for c in (1, 2):
        v, f = s1.cascade_mesh(c)
        assert torch.equal(v, before[c]) and torch.equal(f.cpu(), fs[c])
    assert torch.equal(s1.base_vertices, s1.vertices)
    for b in (s1.offsets, s1.m_vert, s1.v_vert, s1.face_errors, s1.face_counts):
        assert not b.any()
    for k in [0, 1, 0, 1, 0]:
        s1.step(*views[k], use_graph=True)
    torch.cuda.synchronize()
    ids = s1.rast[0, ..., 3]
    assert ((ids > 0) & (ids <= F0)).any() and ids.max().item() <= s1.f_cumsum[-1]
    assert s1.face_counts[:F0].sum().item() > 0 and torch.isfinite(s1.vertices).all()


def _ulp_close(a, b):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    return bool((np.abs(a - b) <= np.spacing(np.abs(b).astype(np.float32))).all())


def test_contract_on_the_stage1_points():
    t0 = _bound4_trainer(contract=True)
    assert t0.cfg.contract and t0.cfg.bound == 2.0
    v, f = S.icosphere(3, 1.6)                                               # most surface points have |x|_inf > 1
    s1 = Stage1Trainer(t0, torch.from_numpy(v), torch.from_numpy(f), 64, 64, ssaa=2)
    mvp, rays_d, gt, bg = _views(64, 64, scale=2.2)[0]
    s1.forward(mvp, rays_d)
    torch.cuda.synchronize()
    inv = s1.inv.long()
    cov = inv >= 0
    k = inv[cov]
    xyz, _ = dr.interpolate(s1.vertices[None], s1.rast, s1.triangles)
    x = xyz.reshape(-1, 3)[cov]
    mag = torch.amax(torch.abs(x), dim=1, keepdim=True)                      # renderer.py:30-31
    ref = torch.where(mag <= 1, x, x * (2 - 1 / mag) / mag)
    assert (mag > 1).float().mean().item() > 0.3
    assert _ulp_close(s1.pts[k], ref)
    # pdirs: the nearest-neighbour up-sampled view directions, as without contraction
    pix = torch.nonzero(cov)[:, 0]
    y, xx = pix // s1.w, pix % s1.w
    q = (y // 2) * (s1.w // 2) + xx // 2
    assert torch.equal(s1.pdirs[k], rays_d[q])
    # the bake contracts the same surface point to the same bits
    baker = X.Baker(t0, s1.h * s1.w)
    baker.points(s1.rast, s1.vertices, s1.triangles, s1.w, 0, s1.h, contract=True)
    torch.cuda.synchronize()
    M_ = int(baker.counters[1].item())
    assert M_ == int(cov.sum().item())
    bp, bpix = baker.pts[:M_], baker.pix[:M_].long()
    assert torch.equal(bp, s1.pts[inv[bpix]])


def test_cascaded_export_bakes_each_cascade_alone(tmp_path):
    t0 = _bound4_trainer()
    vs, fs = _cascade_meshes()
    s1 = Stage1Trainer(t0, vs, fs, 32, 32, ssaa=2)
    vts, fts = [], []
    for f in fs:
        vt, ft = TO.grid_atlas(f.shape[0])
        vts.append(torch.from_numpy(vt).cuda()); fts.append(torch.from_numpy(ft).cuda())
    out = X.export_stage1(s1, str(tmp_path), vts, fts, resolution=64)
    assert len(out) == 3
    for c in range(3):
        v, f = s1.cascade_mesh(c)
        r0, r1 = X.bake_features(t0, v, f, vts[c], fts[c], 64, 64, ssaa=2)
        assert torch.equal(out[c][0], r0) and torch.equal(out[c][1], r1), c
        assert out[c][0].any()
        obj = open(tmp_path / f"mesh_{c}.obj").read().splitlines()
        assert obj[0].split() == ["mtllib", f"mesh_{c}.mtl"]
        assert sum(l.startswith("v ") for l in obj) == vs[c].shape[0] and sum(l.startswith("f ") for l in obj) == fs[c].shape[0]
        mtl = open(tmp_path / f"mesh_{c}.mtl").read().split()
        assert mtl[mtl.index("map_Kd") + 1] == f"feat0_{c}.jpg"
        assert (tmp_path / f"feat0_{c}.jpg").exists() and (tmp_path / f"feat1_{c}.jpg").exists()
    d = json.load(open(tmp_path / "mlp.json"))
    assert d["cascade"] == 3 and d["bound"] == 4.0
