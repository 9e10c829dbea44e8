"""GPU: the stage-1 mesh regularisers of the vertex offsets (lambda_normal * mesh_normal_consistency + lambda_edgelen * mesh_edge_loss,
the reference's utils.py:759-769) -- n2m_s1_mesh_reg alone through the C ABI against the float64 oracle of tests/mesh_reg_oracle.py on
several meshes, the mesh policy (non-manifold edges, repeated-index faces), and Stage1Trainer's vertex step with the new terms: the
gradient and loss it reports, Adam, a skipped step, graph replay and replace_mesh."""
import numpy as np
import pytest
import torch

from nerf2mesh_b200 import mesh as M
from nerf2mesh_b200 import raster as dr
from nerf2mesh_b200 import synthetic as S
from nerf2mesh_b200._lib import call, ptr, stream
from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
from nerf2mesh_b200.stage1 import Stage1Trainer, mesh_reg_counts

import mesh_reg_oracle as O
from test_gpu_stage1 import _setup

pytestmark = pytest.mark.gpu


def _kernel(v, f, lambda_normal, lambda_edgelen):
    """n2m_s1_mesh_reg on its own: (setup counts, loss, grad [V,3])"""
    v = torch.as_tensor(np.asarray(v), dtype=torch.float32).cuda().contiguous()
    tri = torch.as_tensor(np.asarray(f)).to("cuda", torch.int32).contiguous()
    th = dr.TopologyHash(tri)
    counts = mesh_reg_counts(th)
    grad = torch.zeros_like(v)
    loss = torch.zeros(1, device="cuda")
    call("n2m_s1_mesh_reg", ptr(th.keys), ptr(th.opp), th.slots, counts[0], counts[1], ptr(v), lambda_normal, lambda_edgelen, ptr(grad),
         ptr(loss), stream())
    torch.cuda.synchronize()
    return counts, float(loss.item()), grad


def _icosphere(subdiv, seed, scale=0.01, shift=(0, 0, 0)):
    v, f = S.icosphere(subdiv)
    rng = np.random.default_rng(seed)
    v = (v + rng.normal(scale=scale, size=v.shape) + np.asarray(shift)).astype(np.float32)
    return v, f.astype(np.int64)


def _mc_mesh(tmp_path):
    """this repo's marching cubes on the synthetic scene's density (mesh.export_stage0_mesh, as test_gpu_mcubes.py exports it)"""
    tr = Stage0Trainer(Stage0Config(bound=1.0, num_rays=256, max_samples=256 * 128), seed=0)
    grid, bits, _ = S.occupancy_regime("converged")
    tr.set_occupancy(bits, grid)
    thr = 0.5 * float(grid[grid > 0].min().item()) if (grid > 0).any() else 0.5
    v, f = M.export_stage0_mesh(tr, str(tmp_path), resolution=128, density_thresh=thr)
    return v.cpu().numpy(), f.cpu().numpy().astype(np.int64)


def _mesh(name, tmp_path):
    if name == "icosphere3":
        return _icosphere(3, 0)
    if name == "grid":
        v, f = O.grid(12, z=np.random.default_rng(1).normal(scale=0.05, size=169))
        return v.astype(np.float32) * 0.1, f
    if name == "cube":
        return O.cube()
    if name == "zero_area":
        v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [0.5, 1, 0.3], [1.5, -1, 0.2]], np.float32)
        return v, np.array([[0, 1, 2], [1, 0, 3], [2, 1, 4]], np.int64)
    if name == "cascades":
        (v0, f0), (v1, f1) = _icosphere(2, 2), _icosphere(1, 3, shift=(2.0, 0, 0))
        return np.concatenate([v0, v1]), np.concatenate([f0, f1 + len(v0)])
    return _mc_mesh(tmp_path)


@pytest.mark.parametrize("name", ["icosphere3", "grid", "cube", "zero_area", "cascades", "marching_cubes"])
def test_kernel_matches_oracle(name, tmp_path):
    v, f = _mesh(name, tmp_path)
    lam_n, lam_e = 0.3, 0.7
    (E, P, nonmanifold, repeated), loss, grad = _kernel(v, f, lam_n, lam_e)
    ef = O.edge_faces(f)
    assert (E, P, nonmanifold, repeated) == (len(ef), sum(len(o) == 2 for o in ef.values()), 0, 0)
    v64 = np.asarray(v, np.float32).astype(np.float64)            # the oracle sees the kernel's fp32 inputs
    loss_ref, g_ref = O.loss_and_grad(v64, f, lam_n, lam_e)
    g, r = grad.double().cpu(), g_ref
    assert abs(loss - loss_ref) <= 1e-5 * abs(loss_ref), (loss, loss_ref)
    rel = ((g - r).norm() / r.norm()).item()
    err = (g - r).abs().max().item()
    assert rel <= 1e-5 and err <= 1e-4 * r.abs().max().item(), (rel, err, r.abs().max().item())
    if name == "zero_area":
        # the collinear face (0, 1, 2): loss 1 for its pair on (0, 1), and torch's n_other / eps through the clamped norm
        assert r.abs().max().item() > 1e6
    if name == "grid":
        assert O.regularisers(torch.from_numpy(v64), f)[0].item() > 0


def _fin():
    """three triangles on the edge (0, 1): a non-manifold edge"""
    v = np.array([[0, 0, 0], [0.4, 0, 0], [0.2, 0.3, 0], [0.2, -0.2, 0.2], [0.2, -0.2, -0.25]], np.float32)
    return v, np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4]], np.int64)


def test_fin_and_repeated_index():
    v, f = _fin()
    (E, P, nonmanifold, repeated), loss, grad = _kernel(v, f, 0.0, 1.0)
    assert (E, P, nonmanifold, repeated) == (7, 0, 1, 0)
    loss_ref, g_ref = O.loss_and_grad(v.astype(np.float64), f, 0.0, 1.0)
    assert abs(loss - loss_ref) <= 1e-5 * loss_ref and ((grad.double().cpu() - g_ref).norm() / g_ref.norm()).item() <= 1e-5
    rep = np.array([[0, 1, 2], [2, 2, 3]], np.int64)
    assert _kernel(v, rep, 0.0, 1.0)[0][3] == 1
    t0, s1, mvp, rays_d, gt, bg = _setup(ssaa=2, antialias=True, subdiv=2, steps=2, lr_vert=1e-3, lambda_lap=0.0, lambda_normal=1e-3)
    vt, ft = torch.from_numpy(v), torch.from_numpy(f)
    with pytest.raises(ValueError, match="1 non-manifold edges"):
        Stage1Trainer(t0, vt, ft, s1.h0, s1.w0, antialias=True, lr_vert=1e-3, lambda_normal=1e-3)
    with pytest.raises(ValueError, match="replace_mesh: 1 non-manifold edges"):
        s1.replace_mesh(vt, ft)
    for kw in ({"lambda_normal": 1e-3}, {"lambda_edgelen": 1.0}):
        with pytest.raises(ValueError, match="1 faces with a repeated vertex index"):
            Stage1Trainer(t0, vt, torch.from_numpy(rep), s1.h0, s1.w0, antialias=True, lr_vert=1e-3, **kw)
    # the fin trains with the edge loss alone: the vertex step's regulariser part is the oracle's
    fin = Stage1Trainer(t0, vt * 2 - 0.3, ft, s1.h0, s1.w0, antialias=True, lr_vert=1e-3, lambda_lap=0.0, lambda_offsets=0.0, lambda_edgelen=1.0)
    assert (fin.mesh_edges, fin.mesh_pairs) == (7, 0)
    fin.step(mvp.cuda(), rays_d, gt, bg)
    torch.cuda.synchronize()
    _, g_fin = O.loss_and_grad((vt * 2 - 0.3).double(), f, 0.0, 1.0)
    reg = (fin.grad_offsets - fin.vertex_gradient()).double().cpu()
    assert ((reg - g_fin).norm() / g_fin.norm()).item() <= 1e-4


def _oracle_reg(s1, off, lam_lap, ns):
    """autograd of every regulariser of the vertex group at offsets `off` (float64; the reference's laplacian_smooth_loss, which builds
    a float32 sparse matrix, in float32)"""
    x = off.double().detach().clone().requires_grad_(True)
    v = s1.base_vertices.double() + x
    f = s1.triangles.cpu().numpy()
    reg = s1.lambda_offsets * (x ** 2).sum(-1).mean() + O.total(v, f, s1.lambda_normal, s1.lambda_edgelen)
    reg.backward()
    value, grad = float(reg.detach()), x.grad.float()
    if lam_lap:
        x32 = off.detach().clone().requires_grad_(True)
        lap = lam_lap * ns.utils.laplacian_smooth_loss(s1.base_vertices + x32, s1.triangles)
        lap.backward()
        value, grad = value + float(lap.detach()), grad + x32.grad
    return value, grad


@pytest.mark.parametrize("lap", [False, True])
def test_vertex_step_matches_autograd_and_torch_adam(lap):
    """Stage1Trainer(lambda_normal, lambda_edgelen): grad_offsets - vertex_gradient() is the autograd gradient of all the regularisers,
    read_loss() includes the new terms, two steps equal torch.optim.Adam fed the same gradients, a found_inf step leaves the group alone.
    lap: with lambda_lap > 0 as well, checked against the reference's own laplacian_smooth_loss (needs the staged reference)."""
    ns = None
    if lap:
        from oracle import ref_stage
        if not ref_stage.staged():
            pytest.skip("reference Python files not staged")
        ns = ref_stage.load("ref")
    lam_lap, lr_v = (0.01 if lap else 0.0), 1e-3
    t0, s1, mvp, rays_d, gt, bg = _setup(ssaa=2, antialias=True, subdiv=2, steps=8, lr_vert=lr_v, lambda_lap=lam_lap, lambda_offsets=0.1,
                                         lambda_normal=2.0, lambda_edgelen=0.5)
    mvp = mvp.cuda()
    t0.opt_state[0] = 4096.0
    ef = O.edge_faces(s1.triangles.cpu().numpy())
    assert (s1.mesh_edges, s1.mesh_pairs) == (len(ef), len(ef))             # a closed manifold: every edge has two faces
    g = torch.Generator(device="cuda").manual_seed(3)
    s1.offsets.copy_(torch.randn(s1.offsets.shape, device="cuda", generator=g) * 2e-2)
    s1.vertices.copy_(s1.base_vertices + s1.offsets)
    off_old = s1.offsets.clone()
    reg, reg_grad = _oracle_reg(s1, off_old, lam_lap, ns)
    # the image loss alone on the same state (forward + loss_backward do not touch the vertex group)
    s1.forward(mvp, rays_d); s1.loss_backward(gt, bg)
    torch.cuda.synchronize()
    img_loss = s1.read_loss()
    t0.gtable.zero_(); t0.g_mlp.zero_()
    s1.step(mvp, rays_d, gt, bg)
    torch.cuda.synchronize()
    assert t0.opt_state[3].item() == 0 and s1.vert_state[0].item() == 1
    assert reg > 0.05 * img_loss
    assert abs(s1.read_loss() - (img_loss + reg)) <= 1e-5 * (img_loss + reg), (s1.read_loss(), img_loss, reg)
    reg_part = s1.grad_offsets - s1.vertex_gradient()
    rel = ((reg_part - reg_grad).norm() / reg_grad.norm()).item()
    assert rel <= 1e-4, rel
    p = torch.nn.Parameter(off_old.clone())
    opt = torch.optim.Adam([p], lr=lr_v, eps=1e-15)
    p.grad = s1.grad_offsets.clone(); opt.step()
    assert (s1.offsets - p.data).abs().max().item() <= 1e-3 * lr_v
    assert torch.equal(s1.vertices, s1.base_vertices + s1.offsets)
    s1.step(mvp, rays_d, gt, bg)
    torch.cuda.synchronize()
    p.grad = s1.grad_offsets.clone(); opt.step()
    assert (s1.offsets - p.data).abs().max().item() <= 2e-3 * lr_v and s1.vert_state[0].item() == 2
    # a skipped step (found_inf) leaves the group untouched
    before = s1.offsets.clone()
    s1.forward(mvp, rays_d); s1.loss_backward(gt, bg)
    s1.grad_vclip[0, 0] = float("inf")
    call("n2m_s1_vert_check", ptr(s1.grad_vclip), s1.vertices.shape[0], ptr(t0.opt_state), stream())
    scale = t0.opt_state[0].item()
    t0.adam(between=s1._vertex_step)
    torch.cuda.synchronize()
    assert torch.equal(s1.offsets, before) and s1.vert_state[0].item() == 2 and t0.opt_state[0].item() == 0.5 * scale


def _snapshot(t0, s1):
    names = ["table", "color_master", "mlp", "m_table", "v_table", "m_mlp", "v_mlp", "wpack", "opt_state", "g_mlp"]
    bufs = [getattr(t0, n) for n in names] + list(t0.gtables)
    bufs += [getattr(s1, n) for n in ("offsets", "m_vert", "v_vert", "vertices", "vert_state")]
    snap = [b.clone() for b in bufs]

    def restore():
        for b, s in zip(bufs, snap):
            b.copy_(s)
    return restore


def test_graph_replay_and_replace_mesh():
    """a graph-replayed step equals the eager one (colour-field path on: the nullable grad_vworld of the new entry); after replace_mesh
    to a mesh with other E and P the step equals that of a fresh trainer on the mesh"""
    kw = dict(lr_vert=1e-3, lambda_lap=0.0, lambda_offsets=0.1, lambda_normal=0.05, lambda_edgelen=2.0, offset_nerf_grad=True)
    t0, s1, mvp, rays_d, gt, bg = _setup(ssaa=2, antialias=True, subdiv=2, steps=8, **kw)
    mvp = mvp.cuda()
    t0.opt_state[0] = 4096.0
    s1.offsets.copy_(torch.randn(s1.offsets.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4)) * 2e-2)
    s1.vertices.copy_(s1.base_vertices + s1.offsets)
    s1.step(mvp, rays_d, gt, bg)                                     # warm-up (eager)
    restore = _snapshot(t0, s1)
    s1.step(mvp, rays_d, gt, bg)
    torch.cuda.synchronize()
    eager_grad, eager_loss, eager_off = s1.grad_offsets.clone(), s1.read_loss(), s1.offsets.clone()
    for _ in range(2):                                               # capture + replay, then pure replay
        restore()
        s1.step(mvp, rays_d, gt, bg, use_graph=True)
        torch.cuda.synchronize()
        assert len(s1._graphs) == 1 and abs(s1.read_loss() - eager_loss) <= 1e-6 * abs(eager_loss)
        rel = ((s1.grad_offsets - eager_grad).norm() / eager_grad.norm()).item()
        assert rel <= 1e-5, rel
        assert (s1.offsets - eager_off).abs().max().item() <= 1e-6
    # replace_mesh: an open mesh (the icosphere's upper half: boundary edges, so P < E) of other size
    v, f = S.icosphere(3)
    keep = (v[f].mean(1)[:, 1] > -0.1)
    used = np.unique(f[keep])
    remap = -np.ones(len(v), np.int64); remap[used] = np.arange(len(used))
    v2, f2 = torch.from_numpy(v[used].astype(np.float32)), torch.from_numpy(remap[f[keep]])
    s1.replace_mesh(v2, f2)
    fresh = Stage1Trainer(t0, v2, f2, s1.h0, s1.w0, ssaa=2, antialias=True, **kw)
    ef = O.edge_faces(f2.numpy())
    assert (s1.mesh_edges, s1.mesh_pairs) == (fresh.mesh_edges, fresh.mesh_pairs) == (len(ef), sum(len(o) == 2 for o in ef.values()))
    assert s1.mesh_pairs < s1.mesh_edges
    restore2 = _snapshot(t0, fresh)
    out = {}
    for name, tr in (("replaced", s1), ("fresh", fresh)):
        restore2()
        tr.step(mvp, rays_d, gt, bg)
        torch.cuda.synchronize()
        out[name] = (tr.grad_offsets.clone(), tr.read_loss(), tr.offsets.clone())
    (ga, la, oa), (gb, lb, ob) = out["replaced"], out["fresh"]
    assert abs(la - lb) <= 1e-6 * abs(lb) and ((ga - gb).norm() / gb.norm()).item() <= 1e-5
    reg, reg_grad = _oracle_reg(fresh, torch.zeros_like(fresh.offsets), 0.0, None)
    assert ((ga - s1.vertex_gradient() - reg_grad).norm() / reg_grad.norm()).item() <= 1e-4
