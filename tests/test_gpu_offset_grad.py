"""GPU: the colour-field path of the stage-1 vertex gradient (the reference's --enable_offset_nerf_grad, renderer.py:877-879) --
dr.rasterize / dr.interpolate differentiable as nvdiffrast's are (csrc/raster.cu over csrc/raster_grad.cuh) against torch autograd of the
float64 closed form, the reference's default composition left unchanged, Stage1Trainer(offset_nerf_grad=True) against the reference
composition with xyzs not detached (the UNMODIFIED reference NeRFNetwork.rgb over the reference grid-encoder kernels, whose input
gradient is their own calc_grad_inputs), the full step with Adam and graph replay, and the fp16 overflow of the colour-net input
gradient."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from nerf2mesh_b200 import raster as dr
from nerf2mesh_b200 import synthetic as S
from nerf2mesh_b200._lib import call, ptr, stream
from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
from nerf2mesh_b200.stage1 import Stage1Trainer
from nerf2mesh_b200.train_synthetic import full_image_rays
from oracle import raster_oracle as R

pytestmark = pytest.mark.gpu


def _closed_form_loss(pos, attr, tri, rast, wgt):
    """float64 torch: (u, v) of every covered pixel from the closed form at its NDC centre on the triangle ids of `rast`, then the
    interpolation of attr and the linear loss sum(wgt * out)"""
    H, W = rast.shape[1], rast.shape[2]
    r = rast[0].reshape(-1, 4)
    cov = torch.nonzero(r[:, 3] > 0)[:, 0]
    f = r[cov, 3].long() - 1
    X = ((cov % W).double() + 0.5) / W * 2 - 1
    Y = ((cov // W).double() + 0.5) / H * 2 - 1
    idx = tri.long()[f]                                                  # [n,3]
    P = pos[idx]                                                         # [n,3,4]
    q = P[..., :2] - torch.stack([X, Y], -1)[:, None, :] * P[..., 3:4]
    cr = lambda a, b: a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]
    a0, a1, a2 = cr(q[:, 1], q[:, 2]), cr(q[:, 2], q[:, 0]), cr(q[:, 0], q[:, 1])
    s = a0 + a1 + a2
    u, v = a0 / s, a1 / s
    A = attr[idx]
    out = u[:, None] * A[:, 0] + v[:, None] * A[:, 1] + (1 - u - v)[:, None] * A[:, 2]
    return (wgt.reshape(-1, attr.shape[1])[cov] * out).sum()


def _ground_scene(H, W):
    """a ground grid running from behind the camera to far in front (triangles crossing the camera plane) and a small sphere"""
    near, far, f = 0.1, 100.0, 1.0 / np.tan(0.3)
    P = np.array([[f * H / W, 0, 0, 0], [0, f, 0, 0], [0, 0, (far + near) / (near - far), 2 * far * near / (near - far)], [0, 0, -1, 0]])
    gx, gz = np.meshgrid(np.linspace(-20, 20, 13), np.linspace(6, -40, 13), indexing="ij")
    gv = np.stack([gx.reshape(-1), np.full(gx.size, -0.2), gz.reshape(-1)], 1)
    gf = [[i * 13 + j, i * 13 + j + 13, i * 13 + j + 14] for i in range(12) for j in range(12)] + \
         [[i * 13 + j, i * 13 + j + 14, i * 13 + j + 1] for i in range(12) for j in range(12)]
    tv, tf = R.icosphere(2, radius=0.7)
    tv = tv + np.array([0.5, 0.2, -4.0], np.float32)
    v = np.concatenate([gv, tv]).astype(np.float32)
    fcs = np.concatenate([np.array(gf), tf + len(gv)]).astype(np.int32)
    return v, fcs, P.astype(np.float32)


@pytest.mark.parametrize("scene", ["icosphere", "ground"])
def test_rasterize_interpolate_gradients_match_closed_form(scene):
    H, W = 96, 128
    if scene == "icosphere":
        v, fcs = R.icosphere(3)
        mvp = R.perspective_mvp([1.6, 0.9, 1.1], aspect=W / H)
    else:
        v, fcs, mvp = _ground_scene(H, W)
    v = torch.from_numpy(v).cuda().float()
    tri = torch.from_numpy(fcs).cuda()
    mvp = torch.from_numpy(np.asarray(mvp, np.float32)).cuda()
    pos = (F.pad(v, (0, 1), value=1.0) @ mvp.T).contiguous().requires_grad_(True)
    attr = v.clone().requires_grad_(True)
    if scene == "ground":
        w = pos[:, 3].detach()
        assert ((w[tri.long()] <= 0).any(1) & (w[tri.long()] > 0).any(1)).sum().item() > 10
    g = torch.Generator(device="cuda").manual_seed(1)
    wgt = torch.randn(1, H, W, 3, device="cuda", generator=g)
    rast, _ = dr.rasterize(dr.RasterizeCudaContext(), pos[None], tri, (H, W))
    out, _ = dr.interpolate(attr[None], rast, tri)
    (wgt * out).sum().backward()
    rast_d = rast.detach()
    if scene == "ground":          # crossing triangles are visible
        ids = rast_d[0, ..., 3].long() - 1
        w = pos[:, 3].detach()
        crossing = (w[tri.long()] <= 0).any(1)
        assert crossing[ids[ids >= 0]].float().mean().item() > 0.05
    p64 = pos.detach().double().requires_grad_(True)
    a64 = attr.detach().double().requires_grad_(True)
    _closed_form_loss(p64, a64, tri, rast_d, wgt.double()).backward()
    for ours, ref in ((pos.grad, p64.grad), (attr.grad, a64.grad)):
        o, r = ours.double().flatten(), ref.flatten()
        assert r.abs().max().item() > 0
        rel = ((o - r).norm() / r.norm()).item()
        assert rel <= 1e-3, rel
    assert pos.grad[:, 2].abs().max().item() == 0           # clip z gets nothing


def _setup(ssaa=2, contract=False, subdiv=2, steps=8, h0=64, w0=64, **s1_kw):
    N = 1024
    if contract:
        cfg = Stage0Config(bound=2.0, contract=True, num_rays=N, max_samples=N * 64)
        radius, cam = 1.3, np.array([1.5, 1.1, 0.9]) * 2.3                      # |x|_inf of the surface from 0.75 to 1.3
    else:
        cfg = Stage0Config(bound=1.0, num_rays=N, max_samples=N * 256)
        radius, cam = 0.6, np.array([1.5, 1.1, 0.9]) * 1.6
    t0 = Stage0Trainer(cfg, seed=5)
    grid, bits, bricks = S.occupancy_regime("converged", cascades=cfg.cascade, bound=cfg.bound)
    t0.set_occupancy(bits, grid)
    g = torch.Generator().manual_seed(0)
    poses = S.orbit_cameras(100, seed=0)
    for _ in range(steps):            # non-trivial colour parameters
        ro, rd, _, _ = S.sample_rays(poses, S.lego_intrinsics(), 800, 800, N, g)
        t0.step(ro, rd, S.render_bricks(ro, rd, bricks), torch.rand(N, 3, generator=g), torch.rand(N, generator=g), use_graph=False)
    v, f = R.icosphere(subdiv, radius=radius) if subdiv else R.icosphere(2)
    pose = torch.from_numpy(S.look_at_pose(cam).astype(np.float32))
    intr = S.lego_intrinsics(h0, w0)
    _, rays_d = full_image_rays(pose, intr, h0, w0)
    mvp = R.perspective_mvp(cam, fovy=2 * np.arctan(0.5 * h0 / intr[1]), aspect=w0 / h0)
    mvp[1] *= -1
    s1 = Stage1Trainer(t0, torch.from_numpy(v), torch.from_numpy(f), h0, w0, ssaa=ssaa, antialias=True, **s1_kw)
    gt = torch.rand(h0 * w0, 4, generator=g); gt[:, 3] = (gt[:, 3] > 0.5).float()
    bg = torch.rand(h0 * w0, 3, generator=g)
    return t0, s1, torch.from_numpy(mvp), rays_d.cuda(), gt.cuda(), bg.cuda()


def _contract(x):          # renderer.py:25-32
    mag = torch.amax(torch.abs(x), dim=1, keepdim=True)
    return torch.where(mag <= 1, x, x * (2 - 1 / mag) / mag)


def _reference_stage1(ns, ref_stage, t0, s1, mvp, rays_d, gt, bg, offset_nerf_grad, rast_pos_probe=False, lambda_mask=0.1):
    """render_stage1 (renderer.py:824-907, antialias on) + the stage-1 loss (utils.py:703-712) with the unmodified reference model;
    offset_nerf_grad: xyzs[mask_flatten] not detached (renderer.py:877-879).  rast_pos_probe: dr.rasterize gets its own leaf copy of
    the clip-space vertices, so that the gradient it sends to pos can be read on its own."""
    contract = bool(t0.cfg.contract)
    opt = ref_stage.default_opt(bound=t0.cfg.real_bound, contract=contract, dt_gamma=0.0, adaptive_num_rays=False)
    model = ns.make_model(opt)
    model.load_state_dict(t0.export_reference_state(), strict=True)
    model.cuda().train()
    h0, w0, ssaa = s1.h0, s1.w0, s1.ssaa
    h, w = h0 * ssaa, w0 * ssaa
    dirs = rays_d.view(h0, w0, 3)
    dirs = F.interpolate(dirs.permute(2, 0, 1)[None], (h, w), mode="nearest")[0].permute(1, 2, 0).reshape(-1, 3).contiguous()
    dirs = dirs / torch.sqrt(torch.clamp((dirs * dirs).sum(-1, keepdim=True), min=1e-20))
    vertices = s1.vertices.clone().requires_grad_(True)
    vclip = torch.matmul(F.pad(vertices, pad=(0, 1), mode="constant", value=1.0), torch.transpose(mvp.cuda(), 0, 1)).float().unsqueeze(0)
    probe = vclip.detach().clone().requires_grad_(True) if rast_pos_probe else None
    rast, _ = dr.rasterize(dr.RasterizeCudaContext(), probe if rast_pos_probe else vclip, s1.triangles, (h, w))
    xyzs, _ = dr.interpolate(vertices.unsqueeze(0), rast, s1.triangles)
    mask, _ = dr.interpolate(torch.ones_like(vertices[:, :1]).unsqueeze(0), rast, s1.triangles)
    mask_flatten = (mask > 0).view(-1).detach()
    xyzs = xyzs.view(-1, 3)
    if contract:
        xyzs = _contract(xyzs)
    rgbs = torch.zeros(h * w, 3, device="cuda", dtype=torch.float32)
    with torch.autocast("cuda", dtype=torch.float16):
        mask_rgbs, _ = model.rgb(xyzs[mask_flatten] if offset_nerf_grad else xyzs[mask_flatten].detach(), dirs[mask_flatten], None, "full")
    rgbs[mask_flatten] = mask_rgbs.float()
    rgbs = rgbs.view(1, h, w, 3)
    alphas = mask.float()
    alphas = dr.antialias(alphas, rast, vclip, s1.triangles, pos_gradient_boost=1.0).squeeze(0).clamp(0, 1)
    rgbs = dr.antialias(rgbs, rast, vclip, s1.triangles, pos_gradient_boost=1.0).squeeze(0).clamp(0, 1)
    image = alphas * rgbs
    T = 1 - alphas

    def down(x):
        return F.interpolate(x.permute(2, 0, 1)[None], (h0, w0), mode="bilinear")[0].permute(1, 2, 0).contiguous()

    if ssaa > 1:
        image, T = down(image), down(T)
    image = image + T * bg.view(h0, w0, 3)
    ws = (1 - T).view(-1)
    gt_mask = gt[:, 3:]
    gt_rgb = gt[:, :3] * gt_mask + bg * (1 - gt_mask)
    loss = (((image.view(-1, 3) - gt_rgb) ** 2).mean(-1) + lambda_mask * (ws - gt_mask.squeeze(1)) ** 2).mean()
    scale = float(t0.opt_state[0].item())
    (loss * scale).backward()
    return dict(loss=float(loss), grad_vertices=vertices.grad / scale, probe=probe)


def _ref():
    from oracle import ref_stage
    if not ref_stage.staged():
        pytest.skip("reference Python files not staged")
    return ref_stage, ref_stage.load("ref")


def test_default_composition_gets_no_rasterize_gradient():
    """xyzs detached (the reference's default): the only differentiable use of rast is interpolate(ones) for the mask, whose (u, v)
    gradient is exactly zero -- dr.rasterize sends all zeros to pos, so the vertex gradient is the antialias gradient alone"""
    ref_stage, ns = _ref()
    t0, s1, mvp, rays_d, gt, bg = _setup(ssaa=2)
    t0.opt_state[0] = 4096.0
    ref = _reference_stage1(ns, ref_stage, t0, s1, mvp, rays_d, gt, bg, offset_nerf_grad=False, rast_pos_probe=True)
    gp = ref["probe"].grad
    assert gp is not None and gp.shape == ref["probe"].shape and gp.abs().max().item() == 0
    assert ref["grad_vertices"].abs().max().item() > 0


@pytest.mark.parametrize("ssaa,contract", [(2, False), (1, False), (2, True), (1, True)])
def test_offset_nerf_grad_matches_reference_composition(ssaa, contract):
    ref_stage, ns = _ref()
    t0, s1, mvp, rays_d, gt, bg = _setup(ssaa=ssaa, contract=contract, lr_vert=1e-4, offset_nerf_grad=True)
    t0.opt_state[0] = 4096.0
    on = _reference_stage1(ns, ref_stage, t0, s1, mvp, rays_d, gt, bg, offset_nerf_grad=True)
    off = _reference_stage1(ns, ref_stage, t0, s1, mvp, rays_d, gt, bg, offset_nerf_grad=False)
    t0.gtable.zero_(); t0.g_mlp.zero_()
    s1.forward(mvp, rays_d)
    s1.loss_backward(gt, bg)
    torch.cuda.synchronize()
    assert t0.opt_state[3].item() == 0 and s1.counters[2].item() == 0
    if contract:
        mag = s1.vertices.abs().amax(1)
        assert (mag > 1).any() and (mag < 1).any()
    gv, rv, ra = s1.vertex_gradient().double().flatten(), on["grad_vertices"].double().flatten(), off["grad_vertices"].double().flatten()
    cos = (torch.dot(gv, rv) / (gv.norm() * rv.norm() + 1e-300)).item()
    rel = ((gv - rv).norm() / rv.norm()).item()
    assert cos > 0.999 and rel <= 3e-2, (cos, rel)
    # the colour-field part is a real share of the total: the antialias path alone misses the bar by far
    share = ((rv - ra).norm() / rv.norm()).item()
    assert share > 0.1, share
    assert torch.isfinite(s1.grad_vworld).all() and s1.grad_vworld.abs().max().item() > 0


def test_full_step_adam_and_graph_replay():
    """grad_offsets = image part (both paths) + regularisers; the update equals torch.optim.Adam fed that gradient; a graph-replayed step
    equals an eager one"""
    ref_stage, ns = _ref()
    lam_lap, lam_off, lr_v = 0.01, 0.1, 1e-3
    t0, s1, mvp, rays_d, gt, bg = _setup(ssaa=2, lr_vert=lr_v, lambda_lap=lam_lap, lambda_offsets=lam_off, offset_nerf_grad=True)
    mvp = mvp.cuda()
    t0.opt_state[0] = 4096.0
    g = torch.Generator(device="cuda").manual_seed(3)
    s1.offsets.copy_(torch.randn(s1.offsets.shape, device="cuda", generator=g) * 2e-3)
    s1.vertices.copy_(s1.base_vertices + s1.offsets)
    off_old = s1.offsets.clone()
    off = off_old.clone().requires_grad_(True)
    reg = lam_lap * ns.utils.laplacian_smooth_loss(s1.base_vertices + off, s1.triangles) + lam_off * (off ** 2).sum(-1).mean()
    reg.backward()
    names = ["table", "color_master", "mlp", "m_table", "v_table", "m_mlp", "v_mlp", "wpack", "opt_state", "g_mlp"]
    snap = {n: getattr(t0, n).clone() for n in names}
    snap_g = [x.clone() for x in t0.gtables]
    snap_s1 = {n: getattr(s1, n).clone() for n in ("offsets", "m_vert", "v_vert", "vertices", "vert_state")}

    def restore():
        for n in names:
            getattr(t0, n).copy_(snap[n])
        for x, s in zip(t0.gtables, snap_g):
            x.copy_(s)
        for n, s in snap_s1.items():
            getattr(s1, n).copy_(s)

    s1.step(mvp, rays_d, gt, bg)
    torch.cuda.synchronize()
    assert t0.opt_state[3].item() == 0 and s1.vert_state[0].item() == 1
    img_part = s1.vertex_gradient()
    reg_part = s1.grad_offsets - img_part
    assert ((reg_part - off.grad).norm() / off.grad.norm()).item() <= 1e-4
    assert s1.grad_vworld.abs().max().item() > 0
    p = torch.nn.Parameter(off_old.clone())
    opt = torch.optim.Adam([p], lr=lr_v, eps=1e-15)
    p.grad = s1.grad_offsets.clone(); opt.step()
    assert (s1.offsets - p.data).abs().max().item() <= 1e-3 * lr_v
    assert torch.equal(s1.vertices, s1.base_vertices + s1.offsets)
    eager_grad, eager_loss = s1.grad_offsets.clone(), s1.read_loss()
    restore()
    s1.step(mvp, rays_d, gt, bg, use_graph=True)              # the first step after a restore of a warm trainer: captured + replayed
    torch.cuda.synchronize()
    assert len(s1._graphs) == 1 and abs(s1.read_loss() - eager_loss) <= 1e-6 * abs(eager_loss)
    rel = ((s1.grad_offsets - eager_grad).norm() / eager_grad.norm()).item()
    assert rel <= 1e-5, rel
    restore()
    s1.step(mvp, rays_d, gt, bg, use_graph=True)              # pure replay
    torch.cuda.synchronize()
    rel = ((s1.grad_offsets - eager_grad).norm() / eager_grad.norm()).item()
    assert rel <= 1e-5 and s1.vert_state[0].item() == 1, rel


def test_overflow_of_the_colour_net_input_gradient_skips_the_step():
    """a loss scale past fp16's range overflows the x columns of denc: n2m_s1_offset_grad itself sets found_inf and scatters nothing;
    the step then skips the vertex group and halves the scale"""
    t0, s1, mvp, rays_d, gt, bg = _setup(ssaa=2, lr_vert=1e-4, offset_nerf_grad=True)
    mvp = mvp.cuda()
    t0.opt_state[0] = 2.0 ** 40
    s1.forward(mvp, rays_d)
    s1.loss_backward(gt, bg)
    t0.opt_state[3] = 0.0
    s1.grad_vworld.zero_()
    call("n2m_s1_offset_grad", s1._pp(), ptr(s1.rast), ptr(s1.vertices), ptr(s1.vclip), ptr(s1.triangles), ptr(s1.inv), s1.h, s1.w,
         ptr(s1.pts), ptr(s1.denc_tiles), ptr(t0.table), ptr(t0.offsets), ptr(s1.grad_vclip), ptr(s1.grad_vworld), ptr(t0.opt_state), stream())
    torch.cuda.synchronize()
    assert t0.opt_state[3].item() == 1
    assert torch.isfinite(s1.grad_vworld).all()
    before = s1.offsets.clone()
    scale = t0.opt_state[0].item()
    s1.step(mvp, rays_d, gt, bg)
    torch.cuda.synchronize()
    assert torch.equal(s1.offsets, before) and s1.vert_state[0].item() == 0 and t0.opt_state[0].item() == 0.5 * scale
