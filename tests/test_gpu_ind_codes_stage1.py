"""GPU: per-image appearance codes in stage 1 and evaluation -- the stage-1 step's code-row gradient against a float64 restatement and its
optimizer touching the view's row only; Stage1Trainer.render and the texture bake against the reference's render_stage1 /
geo_feat(x, codes[[0]]); the stage-0 evaluation render against the reference's inference render (code 0); the EMA swap's repacked
code columns; save_reference_checkpoint read back by the reference Trainer built with --ind_dim."""
import pytest
import torch
import torch.nn.functional as F

from nerf2mesh_b200 import raster as dr
from nerf2mesh_b200 import synthetic as S
from nerf2mesh_b200 import texture as X
from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
from nerf2mesh_b200.stage1 import Stage1Trainer
from oracle import raster_oracle as R
from test_gpu_stage1_render import _view
from test_gpu_texture import _mesh

pytestmark = pytest.mark.gpu
D, K = 4, 16


def _cols(enc, M):
    T = (M + 127) // 128
    return enc[:T * 8192].view(T, 8, 128, 8).permute(0, 2, 1, 3).reshape(T * 128, 64)[:M]


def _t0(steps=20):
    N = 1024
    t0 = Stage0Trainer(Stage0Config(bound=1.0, num_rays=N, max_samples=N * 256, ind_dim=D, ind_num=K), seed=5)
    grid, bits, bricks = S.occupancy_regime("converged")
    t0.set_occupancy(bits, grid)
    g = torch.Generator().manual_seed(0)
    poses = S.orbit_cameras(100, seed=0)
    for _ in range(steps):
        ro, rd, _, _ = S.sample_rays(poses, S.lego_intrinsics(), 800, 800, N, g)
        t0.step(ro, rd, S.render_bricks(ro, rd, bricks), torch.rand(N, 3, generator=g), torch.rand(N, generator=g), use_graph=False,
                index=torch.randint(0, K, (N,), generator=g, dtype=torch.int32))
    t0.ind[64 * D:].normal_()               # codes of order 1: a wrong row shows
    t0.load_reference_state(t0.export_reference_state())
    torch.cuda.synchronize()
    return t0


def _s1(t0, h0=64, w0=64):
    v, f = R.icosphere(4)
    return Stage1Trainer(t0, torch.from_numpy(v), torch.from_numpy(f), h0, w0, ssaa=2)


def _ref(t0):
    from oracle import ref_stage
    if not ref_stage.staged():
        pytest.skip("reference Python files not staged")
    ns = ref_stage.load("ref")
    opt = ref_stage.default_opt(bound=1.0, dt_gamma=0.0, adaptive_num_rays=False, ind_dim=D, ind_num=K)
    model = ns.make_model(opt)
    model.load_state_dict(t0.export_reference_state(), strict=True)
    return ns, ref_stage, opt, model.cuda().eval()


def test_stage1_step_trains_the_views_code_row():
    t0 = _t0()
    s1 = _s1(t0)
    mvp, rays_d = _view(s1.h0, s1.w0)
    g = torch.Generator().manual_seed(1)
    gt = torch.rand(s1.h0 * s1.w0, 4, generator=g).cuda(); bg = torch.rand(s1.h0 * s1.w0, 3, generator=g).cuda()
    with pytest.raises(ValueError):
        s1.step(mvp, rays_d, gt, bg)                       # index required with codes
    with pytest.raises(ValueError):
        s1.step(mvp, rays_d, gt, bg, index=K)
    k = 5
    s1._index = k
    t0.g_ind.zero_()
    s1.forward(mvp, rays_d)
    s1.loss_backward(gt, bg)
    torch.cuda.synchronize()
    M = int(s1.counters[1].item())
    assert M > 1000 and t0.opt_state[3].item() == 0
    terms = _cols(s1.denc_tiles, M)[:, 54:54 + D].double()
    want = terms.sum(0)
    rows = t0.g_ind[64 * D:].view(K, D).double()
    assert torch.all((rows[k] - want).abs() <= 1e-5 * terms.abs().sum(0) + 1e-30), (rows[k], want)
    assert want.abs().max() > 0 and torch.all(rows[torch.arange(K) != k] == 0)
    assert t0.g_ind[:64 * D].abs().max() > 0                  # the code columns' weight gradient
    # a whole step moves the view's code row only (the other rows have no gradient and no moments)
    t0.g_ind.zero_(); t0.g_mlp.zero_(); t0.gtable.zero_(); t0.m_ind.zero_(); t0.v_ind.zero_()
    before = t0.ind[64 * D:].view(K, D).clone()
    s1.step(mvp, rays_d, gt, bg, index=k)
    torch.cuda.synchronize()
    after = t0.ind[64 * D:].view(K, D)
    assert not torch.equal(after[k], before[k])
    assert torch.equal(after[torch.arange(K) != k], before[torch.arange(K) != k])


def test_stage1_render_and_bake_use_code_0_as_the_reference():
    t0 = _t0()
    ns, ref_stage, opt, model = _ref(t0)
    s1 = _s1(t0)
    mvp, rays_d = _view(s1.h0, s1.w0)
    bg = torch.rand(s1.h0 * s1.w0, 3, device="cuda")
    image, ws, _ = s1.render(mvp, rays_d, bg_color=bg, shading="full")
    # render_stage1 at inference (renderer.py:845-907) with individual_codes[[0]]
    h0, w0, ssaa = s1.h0, s1.w0, s1.ssaa
    h, w = h0 * ssaa, w0 * ssaa
    dirs = rays_d.view(h0, w0, 3)
    dirs = F.interpolate(dirs.permute(2, 0, 1)[None], (h, w), mode="nearest")[0].permute(1, 2, 0).reshape(-1, 3).contiguous()
    dirs = dirs / torch.sqrt(torch.clamp((dirs * dirs).sum(-1, keepdim=True), min=1e-20))
    vclip = torch.matmul(F.pad(s1.vertices, pad=(0, 1), value=1.0), mvp.T).float().unsqueeze(0)
    rast, _ = dr.rasterize(dr.RasterizeCudaContext(), vclip, s1.triangles, (h, w))
    xyzs, _ = dr.interpolate(s1.vertices.unsqueeze(0), rast, s1.triangles)
    mask, _ = dr.interpolate(torch.ones_like(s1.vertices[:, :1]).unsqueeze(0), rast, s1.triangles)
    mf = (mask > 0).view(-1)
    rgbs = torch.zeros(h * w, 3, device="cuda")
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        mrgb, _ = model.rgb(xyzs.view(-1, 3)[mf], dirs[mf], model.individual_codes[[0]], "full")
    rgbs[mf] = mrgb.float()
    rgbs = dr.antialias(rgbs.view(1, h, w, 3), rast, vclip, s1.triangles).squeeze(0).clamp(0, 1)
    alphas = dr.antialias(mask.float(), rast, vclip, s1.triangles).squeeze(0).clamp(0, 1)

    def down(x):
        return F.interpolate(x.permute(2, 0, 1)[None], (h0, w0), mode="bilinear")[0].permute(1, 2, 0).contiguous()

    ref = down(alphas * rgbs) + (1 - down(alphas)) * bg.view(h0, w0, 3)
    torch.cuda.synchronize()
    assert (ws > 0).float().mean().item() > 0.1
    assert (image - ref.view(-1, 3)).abs().max().item() <= 2e-3
    # the bake: geo_feat(x, codes[[0]]) (renderer.py:354-366)
    v, f, vt, ft = _mesh(3)
    rast_uv = X.uv_raster(vt, ft, 256, 256)
    baker = X.Baker(t0, 256 * 256)
    feats = torch.zeros(256, 256, 6, dtype=torch.uint8, device="cuda")
    f32 = torch.zeros(baker.cap, 6, device="cuda")
    baker.band(rast_uv, v, f, 256, 0, 256, feats, feats_f32=f32)
    torch.cuda.synchronize()
    M = int(baker.counters[1].item())
    assert M > 10000
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        gref = model.geo_feat(baker.pts[:M].clone(), model.individual_codes[[0]]).float()
        gother = model.geo_feat(baker.pts[:M].clone(), model.individual_codes[[1]]).float()
    assert (gref - f32[:M]).abs().max().item() <= 2e-3
    assert (gother - f32[:M]).abs().max().item() > 1e-2          # the code matters at this size


def test_stage0_evaluation_render_uses_code_0():
    """Stage0Trainer.render (early-stop rounds and all-samples) against the reference's NeRFRenderer.render in eval mode, which uses
    individual_codes[[0]] (renderer.py:702-703)"""
    from nerf2mesh_b200.train_synthetic import full_image_rays
    t0 = _t0()
    ns, ref_stage, opt, model = _ref(t0)
    pose = S.orbit_cameras(3, seed=99)[1]
    ro, rd = full_image_rays(pose, S.lego_intrinsics() / 8, 100, 100)
    ro, rd = ro.cuda(), rd.cuda()
    with torch.no_grad():
        ev = model.render(ro, rd, bg_color=1, perturb=False, **{k: v for k, v in vars(opt).items() if k not in ("bg_color", "perturb")})
    img, ws, _ = t0.render(ro, rd, bg_color=1.0)
    img2, _, _ = t0.render(ro, rd, bg_color=1.0, early_stop=False)
    torch.cuda.synchronize()
    assert 0.02 < (ws > 0.5).float().mean().item() < 0.98
    assert (img - ev["image"]).abs().max().item() <= 2e-3, (img - ev["image"]).abs().max().item()
    assert (img2 - ev["image"]).abs().max().item() <= 2e-3, (img2 - ev["image"]).abs().max().item()


def test_ema_swap_repacks_the_code_columns_and_checkpoint_reads_back(tmp_path):
    t0 = _t0(steps=4)
    t0.enable_ema(0.95)
    N = t0.N
    g = torch.Generator().manual_seed(7)
    poses = S.orbit_cameras(10, seed=1)
    ro, rd, _, _ = S.sample_rays(poses, S.lego_intrinsics(), 800, 800, N, g)
    t0.step(ro, rd, torch.rand(N, 4, generator=g), torch.rand(N, 3, generator=g), torch.rand(N, generator=g), use_graph=False,
            index=3)
    t0.ema_update()
    pts = (torch.rand(4096, 3, device="cuda") * 2 - 1).contiguous()
    dirs = F.normalize(torch.randn(4096, 3, device="cuda"), dim=-1).contiguous()
    cnt = torch.full((4,), 4096, dtype=torch.int32, device="cuda")
    enc = torch.zeros(4096 * 64, dtype=torch.float16, device="cuda")
    out = torch.zeros(4096, 4, device="cuda")

    def fwd(row):
        t0.encode_points(t0._pp(), pts, dirs, cnt, 4096, enc, row)
        from nerf2mesh_b200._lib import call, ptr, stream
        call("n2m_s0_mlp_fwd", t0._pp(), ptr(enc), ptr(cnt), 4096, ptr(t0.wpack), ptr(out), None, 0, 1, stream())
        torch.cuda.synchronize()
        return out.clone()

    t0.ema_apply()
    swapped = fwd(3)
    ema_state = t0.export_reference_state()
    t0.ema_restore()
    live = fwd(3)
    assert not torch.equal(swapped, live)
    live_state = t0.export_reference_state()
    t0.load_reference_state(ema_state)
    assert torch.equal(fwd(3), swapped)                     # the swap repacked the EMA code columns
    t0.load_reference_state(live_state)
    assert torch.equal(fwd(3), live)
    # checkpoint: the reference Trainer built with --ind_dim reads model and EMA back
    path = str(tmp_path / "ckpt.pth")
    t0.save_reference_checkpoint(path, full=True)
    ns, ref_stage, opt, model = _ref(t0)
    rt = ns.utils.Trainer("ngp", opt, model, device=torch.device("cuda"), workspace=None, mute=True,
                          optimizer=lambda m: torch.optim.Adam(m.get_params(opt.lr), eps=1e-15),
                          criterion=torch.nn.MSELoss(reduction="none"), ema_decay=0.95, fp16=True,
                          use_checkpoint="scratch", use_tensorboardX=False, scheduler_update_every_step=True)
    for p in rt.model.parameters():
        p.data.zero_()
    rt.load_checkpoint(checkpoint=path, model_only=True)
    sd = rt.model.state_dict()
    assert torch.equal(sd["individual_codes"].cpu(), live_state["individual_codes"].cpu())
    assert torch.equal(sd["color_net.net.0.weight"].cpu(), live_state["color_net.net.0.weight"].cpu())
    rt.ema.copy_to()
    assert torch.equal(rt.model.individual_codes.detach().cpu(), ema_state["individual_codes"].cpu())
    assert torch.equal(rt.model.color_net.net[0].weight.detach().cpu(), ema_state["color_net.net.0.weight"].cpu())
