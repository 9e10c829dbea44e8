"""GPU: per-image appearance codes (Stage0Config.ind_dim / ind_num, the reference's --ind_dim / --ind_num) through the stage-0 step.

Checked here: the code columns of the gather (stand-alone, fused forward, explicit points) against fp16(codes[ray_img[ray]]) with every
other column bit-identical to the gather without codes; the code gradient against the float64 per-image sum of the denc values the
kernel read, for every part count, the adaptive ray count and a non-finite term; the optimizer against torch Adam with the reference's
groups through a skipped step; EMA swap / restore; graph replay against eager; one step against the reference's NeRFNetwork /
Trainer.train_step built with ind_dim = 4, with a per-ray and a scalar index."""
import pytest
import torch

import ind_codes_oracle as O
from nerf2mesh_b200 import synthetic as S
from nerf2mesh_b200._lib import call, ptr, stream
from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _cols(enc, M):
    """enc_tiles (fp16, core-matrix layout: [tile][chunk][row][8]) -> [M, 64] rows"""
    T = (M + 127) // 128
    return enc[:T * 8192].view(T, 8, 128, 8).permute(0, 2, 1, 3).reshape(T * 128, 64)[:M]


def _trainer(D, N=1024, ind_num=16, **kw):
    cfg = Stage0Config(bound=1.0, dt_gamma=0.0, num_rays=N, max_samples=N * 160, ind_dim=D, ind_num=ind_num, lambda_tv=0.0, **kw)
    tr = Stage0Trainer(cfg, seed=5)
    grid, bits, _ = S.occupancy_regime("converged", cascades=1, bound=1.0)
    tr.set_occupancy(bits, grid)
    return tr


def _batch(N, seed, ind_num=16):
    g = torch.Generator().manual_seed(seed)
    poses = S.orbit_cameras(20, radius=S.LEGO_RADIUS, seed=seed)
    ro, rd, _, _ = S.sample_rays(poses, S.lego_intrinsics(), 800, 800, N, g)
    gt = torch.rand(N, 4, generator=g)
    bg = torch.rand(N, 3, generator=g)
    noises = torch.rand(N, generator=g)
    idx = torch.randint(0, ind_num, (N,), generator=g, dtype=torch.int32)
    return (ro.to(DEV), rd.to(DEV), gt.to(DEV), bg.to(DEV), noises.to(DEV)), idx.to(DEV)


def _load(tr, batch, idx):
    tr.slots[tr.cur].load(*batch)
    tr.slots[tr.cur].load_index(idx)


def _codes(tr):
    return tr.ind[64 * tr.ind_dim:].view(tr.ind_num, tr.ind_dim)


# ------------------------------------------------------------------------------------------------
# gather
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [1, 4, 10])
def test_gather_writes_the_codes_and_leaves_every_other_column(D):
    tr = _trainer(D)
    _codes(tr).normal_()                                  # codes of order 1: every fp16 rounding matters
    batch, idx = _batch(tr.N, 1)
    _load(tr, batch, idx)
    tr.march()
    torch.cuda.synchronize()
    M = int(tr.counters[1].item())
    assert M > 10000
    tr.encode_fwd()
    with_codes = _cols(tr.enc_tiles, M).clone()
    plain = torch.zeros_like(tr.enc_tiles)
    call("n2m_s0_encode_fwd", tr._pp(), ptr(tr.recs), ptr(tr.counters), tr.Mcap, ptr(tr.rays_o), ptr(tr.rays_d), ptr(tr.table),
         ptr(tr.offsets), ptr(plain), 0, 1, stream())
    plain = _cols(plain, M)
    ray = tr.recs[:M, 3].contiguous().view(torch.int32).long()
    want = _codes(tr)[idx.long()[ray]].half()
    assert torch.equal(with_codes[:, 54:54 + D], want)
    keep = [c for c in range(64) if not 54 <= c < 54 + D]
    assert torch.equal(with_codes[:, keep].view(torch.int16), plain[:, keep].view(torch.int16))
    assert torch.all(with_codes[:, 54 + D:] == 0)
    # the fused forward builds the same images, and its MLP output equals the two-launch forward's
    tr.mlp_fwd()
    out_two = tr.out[:M].clone()
    tr.enc_tiles.zero_()
    tr.fwd_fused()
    torch.cuda.synchronize()
    assert torch.equal(_cols(tr.enc_tiles, M).view(torch.int16), with_codes.view(torch.int16))
    assert torch.equal(tr.out[:M], out_two)
    # explicit points with one code row
    P = 4096
    pts = (torch.rand(P, 3, device=DEV) * 2 - 1).contiguous()
    cnt = torch.full((4,), P, dtype=torch.int32, device=DEV)
    enc = torch.zeros(P * 64, dtype=torch.float16, device=DEV)
    enc0 = torch.zeros_like(enc)
    row = _codes(tr)[3].contiguous()
    call("n2m_s0_encode_points_codes", tr._pp(), ptr(pts), None, ptr(cnt), P, ptr(tr.table), ptr(tr.offsets), ptr(row), ptr(enc), stream())
    call("n2m_s0_encode_points", tr._pp(), ptr(pts), None, ptr(cnt), P, ptr(tr.table), ptr(tr.offsets), ptr(enc0), stream())
    torch.cuda.synchronize()
    a, b = _cols(enc, P), _cols(enc0, P)
    assert torch.equal(a[:, 54:54 + D], row.half().expand(P, D))
    assert torch.equal(a[:, keep].view(torch.int16), b[:, keep].view(torch.int16))


# ------------------------------------------------------------------------------------------------
# code gradient
# ------------------------------------------------------------------------------------------------
def _oracle_grad(tr, idx, M, n_active=None):
    denc = _cols(tr.denc_tiles, M)[:, 54:54 + tr.ind_dim].double().cpu().numpy()
    return torch.from_numpy(O.code_grad(denc, tr.rays.cpu().numpy(), idx.cpu().numpy(), tr.ind_num, tr.ind_dim, M, n_active))


@pytest.mark.parametrize("nparts", [1, 2, 4, 8])
def test_code_grad_equals_the_per_image_sum(nparts):
    D = 4
    tr = _trainer(D)
    tr.nparts = nparts
    batch, idx = _batch(tr.N, 2)
    _load(tr, batch, idx)
    tr.forward_backward()
    torch.cuda.synchronize()
    M = int(tr.counters[1].item())
    got = tr.g_ind[64 * D:].view(tr.ind_num, D).double().cpu()
    want = _oracle_grad(tr, idx, M)
    assert want.abs().max() > 0 and tr.opt_state[3].item() == 0
    scale = _cols(tr.denc_tiles, M)[:, 54:54 + D].double().abs().sum(0).cpu()      # fp32 summation-order bound per dimension
    assert torch.all((got - want).abs() <= 1e-5 * scale + 1e-30), ((got - want).abs().max(), scale)


def test_code_grad_honours_the_active_ray_count_and_flags_non_finite_terms():
    D = 3
    tr = _trainer(D)
    batch, idx = _batch(tr.N, 3)
    _load(tr, batch, idx)
    tr.forward_backward()
    torch.cuda.synchronize()
    M = int(tr.counters[1].item())
    g_codes = tr.g_ind.data_ptr() + 4 * 64 * D
    for n in (1, 300, tr.N):
        for nparts in (1, 2, 8):
            tr.g_ind.zero_()
            active = torch.tensor([n], dtype=torch.int32, device=DEV)
            for k in range(nparts):
                call("n2m_s0_code_grad", tr._pp(), ptr(tr.rays), ptr(tr.counters), tr.N, ptr(tr.denc_tiles), ptr(tr.slots[tr.cur].ray_img),
                     g_codes, ptr(tr.opt_state), ptr(active), k, nparts, stream())
            torch.cuda.synchronize()
            want = _oracle_grad(tr, idx, M, n_active=n)
            got = tr.g_ind[64 * D:].view(tr.ind_num, D).double().cpu()
            assert torch.allclose(got, want, rtol=1e-5, atol=1e-6 * want.abs().max().item()), (n, nparts)
    assert tr.opt_state[3].item() == 0
    # a non-finite term of the first sample of a ray with samples
    r = int(torch.nonzero(tr.rays[:, 1] > 0)[0].item())
    j = int(tr.rays[r, 0].item())
    tr.denc_tiles[(j // 128) * 8192 + 7 * 1024 + (j % 128) * 8 + 0] = float("inf")          # column 56
    call("n2m_s0_code_grad", tr._pp(), ptr(tr.rays), ptr(tr.counters), tr.N, ptr(tr.denc_tiles), ptr(tr.slots[tr.cur].ray_img), g_codes,
         ptr(tr.opt_state), None, 0, 1, stream())
    torch.cuda.synchronize()
    assert tr.opt_state[3].item() == 1


# ------------------------------------------------------------------------------------------------
# optimizer, EMA, graph replay
# ------------------------------------------------------------------------------------------------
def test_optimizer_matches_torch_adam_with_the_reference_groups():
    D, lr = 4, 1e-2
    tr = _trainer(D)
    w = tr.ind[:64 * D].double().cpu().clone().requires_grad_(True)
    c = tr.ind[64 * D:].double().cpu().clone().requires_grad_(True)
    opt = torch.optim.Adam([{"params": [w], "lr": lr}, {"params": [c], "lr": lr * 0.1, "weight_decay": 0}], eps=1e-15)
    scaler_scale = tr.opt_state[0].item()
    for it in range(5):
        batch, idx = _batch(tr.N, 10 + it)
        _load(tr, batch, idx)
        tr.forward_backward()
        if it == 2:
            tr.g_ind[5] = float("nan")           # GradScaler skips the step and halves the scale
        torch.cuda.synchronize()
        g = tr.g_ind.double().cpu() / tr.opt_state[0].item()
        assert tr.opt_state[0].item() == scaler_scale
        tr.adam()
        torch.cuda.synchronize()
        if it == 2:
            scaler_scale *= 0.5
            assert tr.opt_state[0].item() == scaler_scale
            continue
        w.grad, c.grad = g[:64 * D].clone(), g[64 * D:].clone()
        opt.step()
        assert torch.all(tr.g_ind == 0)
    got = tr.ind.double().cpu()
    assert torch.allclose(got[:64 * D], w.detach(), rtol=1e-4, atol=1e-6)
    assert torch.allclose(got[64 * D:], c.detach(), rtol=1e-4, atol=1e-6)
    # the repacked code columns are what the next forward reads: the exported model re-imported gives the same images
    st = tr.export_reference_state()
    batch, idx = _batch(tr.N, 99)
    _load(tr, batch, idx)
    tr.march(); tr.encode_fwd(); tr.mlp_fwd(); torch.cuda.synchronize()
    M = int(tr.counters[1].item())
    out_a = tr.out[:M].clone()
    tr.load_reference_state(st)
    tr.encode_fwd(); tr.mlp_fwd(); torch.cuda.synchronize()
    assert torch.equal(tr.out[:M], out_a)


def test_ema_swap_and_restore_cover_the_code_block():
    D = 2
    tr = _trainer(D)
    tr.enable_ema(0.95)
    before = tr.ind.clone()
    batch, idx = _batch(tr.N, 20)
    tr.step(*batch, index=idx, use_graph=False)
    tr.ema_update()
    torch.cuda.synchronize()
    live = tr.ind.clone()
    shadow = tr._ema["ind"].clone()
    decay = min(0.95, 2 / 11)
    assert torch.allclose(shadow, before - (1 - decay) * (before - live), rtol=1e-6, atol=1e-7)
    sd = tr.ema_state_dict()
    assert sd["shadow_params"][0].shape == (tr.ind_num, D) and sd["shadow_params"][5].shape == (64, 35 + D)
    tr.ema_apply()
    assert torch.equal(tr.ind, shadow)
    tr.ema_restore()
    assert torch.equal(tr.ind, live) and torch.equal(tr._ema["ind"], shadow)


def test_graph_replay_with_a_changing_index_equals_eager():
    D = 4
    trs = [_trainer(D), _trainer(D)]
    for it in range(4):
        batch, idx = _batch(1024, 30 + it)
        nxt = _batch(1024, 31 + it)
        for tr, g in zip(trs, (True, False)):
            tr.step(*batch, index=idx if it == 0 else None, use_graph=g, next_batch=nxt[0], next_index=nxt[1])
    torch.cuda.synchronize()
    a, b = trs
    assert torch.allclose(a.ind, b.ind, rtol=1e-4, atol=1e-6)
    assert torch.allclose(a.mlp, b.mlp, rtol=1e-4, atol=1e-6)
    assert not torch.equal(a.ind[64 * D:], _trainer(D).ind[64 * D:])         # the codes did train


# ------------------------------------------------------------------------------------------------
# one step against the reference model built with ind_dim
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("per_ray", [True, False])
def test_step_matches_reference_with_codes(per_ray):
    import test_gpu_reference_parity as RP
    ref_stage, ns = RP._ref_stack()
    D, K, N = 4, 100, RP.N
    c = RP.CASES["lego"]
    grid, bits, bricks = RP._scene(c)
    cfg = Stage0Config(bound=c["bound"], dt_gamma=c["dt_gamma"], num_rays=N, max_samples=N * c["cap"], ind_dim=D, ind_num=K)
    tr = Stage0Trainer(cfg, seed=3)
    tr.set_occupancy(bits, grid)
    g = torch.Generator().manual_seed(77)
    for it in range(20):
        ro, rd = RP._batch(c, 100 + it)
        gg = torch.Generator().manual_seed(1000 + it)
        tr.step(ro, rd, RP._gt(c, ro, rd, bricks), torch.rand(N, 3, generator=gg), torch.rand(N, generator=gg),
                shading="diffuse" if it < 10 else "full", use_graph=False,
                index=torch.randint(0, K, (N,), generator=g, dtype=torch.int32).cuda())
    torch.cuda.synchronize()
    state = tr.export_reference_state()
    ro, rd = RP._batch(c, 7)
    gt = RP._gt(c, ro, rd, bricks)
    index = torch.randint(0, K, (N,), generator=g, dtype=torch.int32) if per_ray else 17
    data = dict(rays_o=ro.cuda(), rays_d=rd.cuda(), images=gt.cuda(),
                index=index.long().cuda() if per_ray else [index])
    seed = 4242
    torch.manual_seed(seed)
    bg = torch.rand(N, 3, device=DEV); noises = torch.rand(N, device=DEV)

    def ref_trainer(fp16, scale=None):
        opt = ref_stage.default_opt(bound=c["bound"], dt_gamma=c["dt_gamma"], lambda_entropy=c["lambda_entropy"], fp16=fp16,
                                    adaptive_num_rays=False, num_rays=N, ind_dim=D, ind_num=K)
        model = ns.make_model(opt)
        model.load_state_dict({k: v.clone() for k, v in state.items()}, strict=True)
        model.cuda().train()
        rt = ns.utils.Trainer("ngp", opt, model, device=torch.device("cuda"), workspace=None, mute=True,
                              optimizer=lambda m: torch.optim.Adam(m.get_params(opt.lr), eps=1e-15),
                              criterion=torch.nn.MSELoss(reduction="none"), ema_decay=None, fp16=fp16,
                              use_checkpoint="scratch", use_tensorboardX=False, scheduler_update_every_step=True)
        rt.global_step = 2000
        rt.ns = ns
        if scale is not None and fp16:
            rt.scaler = torch.amp.GradScaler("cuda", init_scale=float(scale))
        return rt

    scale = 65536.0
    for _ in range(16):
        r16a = RP._ref_step(ref_trainer(True, scale), data, seed)
        if all(torch.isfinite(v).all().item() for v in r16a["grads"].values()):
            break
        scale *= 0.5
    r16b = RP._ref_step(ref_trainer(True, scale), data, seed)
    r32 = RP._ref_step(ref_trainer(False), data, seed)
    tr.opt_state[0] = scale
    tr.slots[tr.cur].load(data["rays_o"], data["rays_d"], data["images"], bg, noises)
    tr.slots[tr.cur].load_index(index.cuda() if per_ray else index)
    tr._fill_params(True, c["alpha"])
    tr.forward_backward()
    torch.cuda.synchronize()
    assert tr.opt_state[3].item() == 0
    M = int(tr.counters[1].item())
    assert M == r16a["M"]
    ours = tr.export_reference_grads()
    img = RP._cmp(tr.image, r16a["image"])
    assert img["max_err_of_scale"] <= 1e-3, img
    assert abs(tr.read_loss() - r16a["loss"]) <= 1e-3 * abs(r16a["loss"])
    for nm in ("color_net.net.0.weight", "individual_codes"):
        ga, gb, g32 = r16a["grads"][nm], r16b["grads"][nm], r32["grads"][nm]
        o16, o32 = RP._cmp(ours[nm], ga), RP._cmp(ours[nm], g32)
        r_16_32, r_rr = RP._cmp(ga, g32), RP._cmp(gb, ga)
        floor = max(r_16_32["rel_l2"], r_rr["rel_l2"])
        assert o32["rel_l2"] <= 1.5 * r_16_32["rel_l2"] + 1e-3, (nm, o32, r_16_32)
        assert o16["rel_l2"] <= 2.0 * floor + 1e-3, (nm, o16, floor)
    # the code columns alone (35..38) carry the code path's weight gradient
    cc = RP._cmp(ours["color_net.net.0.weight"][:, 35:], r32["grads"]["color_net.net.0.weight"][:, 35:])
    ref_cc = RP._cmp(r16a["grads"]["color_net.net.0.weight"][:, 35:], r32["grads"]["color_net.net.0.weight"][:, 35:])
    assert cc["rel_l2"] <= 1.5 * ref_cc["rel_l2"] + 1e-3, (cc, ref_cc)
