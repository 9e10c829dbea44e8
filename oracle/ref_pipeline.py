"""oracle/ref_pipeline.py -- TEST / BASELINE INFRASTRUCTURE, NOT PRODUCT.

The reference's stage-0 training pipeline re-composed around the reference's OWN, unmodified CUDA kernels
(oracle/_ref: raymarching / gridencoder extensions compiled from the reference tree by oracle/build_ref.py).
It exists so that the same GPU can run "the reference" beside nerf2mesh_b200:

  * same-box throughput baseline (samples/s of the reference CUDA path), and
  * PSNR-vs-reference on the synthetic scene (BASELINE.json: "PSNR vs ref").

The Python layer restates, with citations, what the reference does around its kernels -- it cannot import
nerf/renderer.py / nerf/utils.py on the GPU box (they are not shipped, and need trimesh, nvdiffrast, ...):
  raymarching wrappers   raymarching/raymarching.py:184-302
  GridEncoder            gridencoder/grid.py:24-192
  NeRFNetwork            nerf/network.py:10-189, activation.py:5-17
  render (train branch)  nerf/renderer.py:688-747,804
  train_step / TV / step nerf/utils.py:628-738,801-823,1163-1182 ; optimizer + schedule main.py:221,239
  update_extra_state     nerf/renderer.py:1074-1149

    python -m oracle.ref_pipeline --iters 3000        # train + test PSNR + samples/s
"""
import argparse
import json
import math
import time

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as Fnn
from torch.autograd import Function

from .build_ref import load_ref

_rm = None
_ge = None


def backends():
    global _rm, _ge
    if _rm is None:
        _rm = load_ref("_ref_raymarching")
        _ge = load_ref("_ref_gridencoder")
    return _rm, _ge


# ---- raymarching wrappers (raymarching.py) -------------------------------------------------------
def near_far_from_aabb(rays_o, rays_d, aabb, min_near):
    rm, _ = backends()
    N = rays_o.shape[0]
    nears = torch.empty(N, device=rays_o.device); fars = torch.empty(N, device=rays_o.device)
    rm.near_far_from_aabb(rays_o, rays_d, aabb, N, min_near, nears, fars)
    return nears, fars


def march_rays_train(rays_o, rays_d, bound, contract, bitfield, C, H, nears, fars, perturb, dt_gamma, max_steps):
    rm, _ = backends()
    N = rays_o.shape[0]
    counter = torch.zeros(1, dtype=torch.int32, device=rays_o.device)
    noises = torch.rand(N, device=rays_o.device) if perturb else torch.zeros(N, device=rays_o.device)
    rays = torch.empty(N, 2, dtype=torch.int32, device=rays_o.device)
    rm.march_rays_train(rays_o, rays_d, bitfield, bound, contract, dt_gamma, max_steps, N, C, H, nears, fars, None, None, None, rays, counter, noises)
    M = counter.item()                                                     # the reference's host sync (raymarching.py:232)
    xyzs = torch.zeros(M, 3, device=rays_o.device); dirs = torch.zeros(M, 3, device=rays_o.device); ts = torch.zeros(M, 2, device=rays_o.device)
    rm.march_rays_train(rays_o, rays_d, bitfield, bound, contract, dt_gamma, max_steps, N, C, H, nears, fars, xyzs, dirs, ts, rays, counter, noises)
    return xyzs, dirs, ts, rays


class _CompositeTrain(Function):
    @staticmethod
    def forward(ctx, sigmas, rgbs, ts, rays, T_thresh):
        rm, _ = backends()
        sigmas = sigmas.float().contiguous(); rgbs = rgbs.float().contiguous()
        M, N = sigmas.shape[0], rays.shape[0]
        weights = torch.zeros(M, device=sigmas.device); ws = torch.empty(N, device=sigmas.device)
        depth = torch.empty(N, device=sigmas.device); image = torch.empty(N, 3, device=sigmas.device)
        rm.composite_rays_train_forward(sigmas, rgbs, ts, rays, M, N, T_thresh, False, weights, ws, depth, image)
        ctx.save_for_backward(sigmas, rgbs, ts, rays, ws, depth, image)
        ctx.T = T_thresh
        return weights, ws, depth, image

    @staticmethod
    def backward(ctx, gw, gws, gd, gi):
        rm, _ = backends()
        sigmas, rgbs, ts, rays, ws, depth, image = ctx.saved_tensors
        M, N = sigmas.shape[0], rays.shape[0]
        gs = torch.zeros_like(sigmas); gr = torch.zeros_like(rgbs)
        rm.composite_rays_train_backward(gw.contiguous(), gws.contiguous(), gd.contiguous(), gi.contiguous(), sigmas, rgbs, ts, rays,
                                         ws, depth, image, M, N, ctx.T, False, gs, gr)
        return gs, gr, None, None, None


# ---- grid encoder (grid.py) ----------------------------------------------------------------------
class _GridEncode(Function):
    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, inputs, embeddings, offsets, S, H):
        _, ge = backends()
        inputs = inputs.contiguous()
        B, D = inputs.shape
        L = offsets.shape[0] - 1
        C = embeddings.shape[1]
        if torch.is_autocast_enabled() and C % 2 == 0:
            embeddings = embeddings.to(torch.half)
        outputs = torch.empty(L, B, C, device=inputs.device, dtype=embeddings.dtype)
        ge.grid_encode_forward(inputs, embeddings, offsets, outputs, B, D, C, L, L, S, H, None, 0, False, 0)
        ctx.save_for_backward(inputs, embeddings, offsets)
        ctx.dims = (B, D, C, L, S, H)
        return outputs.permute(1, 0, 2).reshape(B, L * C)

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, grad):
        _, ge = backends()
        inputs, embeddings, offsets = ctx.saved_tensors
        B, D, C, L, S, H = ctx.dims
        grad = grad.reshape(B, L, C).permute(1, 0, 2).contiguous()
        gemb = torch.zeros_like(embeddings)
        ge.grid_encode_backward(grad, inputs, embeddings, offsets, gemb, B, D, C, L, L, S, H, None, None, 0, False, 0)
        return None, gemb, None, None, None


class RefGridEncoder(nn.Module):
    def __init__(self, level_dim, bound):
        super().__init__()
        from .grid_oracle import level_offsets
        self.pls = float(np.exp2(np.log2(2048 * bound / 16) / 15))
        self.S = float(np.log2(self.pls))
        self.register_buffer("offsets", torch.from_numpy(level_offsets(3, 16, self.pls, 16, 19, False)))
        self.embeddings = nn.Parameter(torch.empty(int(self.offsets[-1]), level_dim).uniform_(-1e-4, 1e-4))

    def forward(self, x, bound):
        return _GridEncode.apply((x + bound) / (2 * bound), self.embeddings, self.offsets, self.S, 16)

    @torch.amp.autocast("cuda", enabled=False)
    def grad_total_variation(self, weight, x, bound):
        _, ge = backends()
        inp = ((x + bound) / (2 * bound)).contiguous()
        ge.grad_total_variation(inp, self.embeddings, self.embeddings.grad, self.offsets, weight, inp.shape[0], 3,
                                self.embeddings.shape[1], 16, self.S, 16, 0, False)


class _TruncExp(Function):
    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, g):
        return g * torch.exp(ctx.saved_tensors[0].clamp(-15, 15))


def _mlp(i, o, h, n):
    return nn.ModuleList([nn.Linear(i if l == 0 else h, o if l == n - 1 else h, bias=False) for l in range(n)])


def _run_mlp(net, x):
    for l, lin in enumerate(net):
        x = lin(x)
        if l != len(net) - 1:
            x = Fnn.relu(x, inplace=True)
    return x


class RefField(nn.Module):
    """nerf/network.py NeRFNetwork (density + colour hash grids, three bias-free ReLU MLPs)."""

    def __init__(self, bound=1.0):
        super().__init__()
        self.bound = bound
        self.encoder = RefGridEncoder(1, bound)
        self.encoder_color = RefGridEncoder(2, bound)
        self.sigma_net = _mlp(19, 1, 32, 2)
        self.color_net = _mlp(35, 6, 64, 3)
        self.specular_net = _mlp(6, 3, 32, 2)

    def load_reference_state(self, st):
        with torch.no_grad():
            self.encoder.embeddings.copy_(st["encoder.embeddings"]); self.encoder_color.embeddings.copy_(st["encoder_color.embeddings"])
            for name in ("sigma_net", "color_net", "specular_net"):
                for l, lin in enumerate(getattr(self, name)):
                    lin.weight.copy_(st[f"{name}.net.{l}.weight"])

    def density(self, x):
        h = self.encoder(x, self.bound)
        h = _run_mlp(self.sigma_net, torch.cat([x, h], -1))
        return _TruncExp.apply(h[..., 0])

    def forward(self, x, d, shading):
        sigma = self.density(x)
        h = self.encoder_color(x, self.bound)
        feat = torch.sigmoid(_run_mlp(self.color_net, torch.cat([x, h], -1)))
        diffuse = feat[..., :3]
        if shading == "diffuse":
            return sigma, diffuse, None
        spec = torch.sigmoid(_run_mlp(self.specular_net, torch.cat([d, feat[..., 3:]], -1)))
        return sigma, (spec + diffuse).clamp(0, 1), spec


class RefTrainer:
    """renderer.render (training branch) + Trainer.train_step / post_train_step / optimizer step."""

    def __init__(self, bound=1.0, grid_size=128, lr=1e-2, lambda_tv=1e-8, lambda_mask=0.1, lambda_specular=1e-5, device="cuda"):
        self.bound, self.H = bound, grid_size
        self.cascade = 1 + math.ceil(math.log2(bound))
        self.field = RefField(bound).to(device)
        self.density_grid = torch.zeros(self.cascade, grid_size ** 3, device=device)
        self.density_bitfield = torch.zeros(self.cascade * grid_size ** 3 // 8, dtype=torch.uint8, device=device)
        self.aabb = torch.tensor([-bound] * 3 + [bound] * 3, dtype=torch.float32, device=device)
        self.opt = torch.optim.Adam(self.field.parameters(), lr=lr, eps=1e-15)
        self.scaler = torch.amp.GradScaler("cuda")
        self.lambda_tv, self.lambda_mask, self.lambda_specular = lambda_tv, lambda_mask, lambda_specular
        self.device = device

    def render(self, rays_o, rays_d, bg, perturb, shading, dt_gamma=0.0, max_steps=1024, T_thresh=1e-4):
        nears, fars = near_far_from_aabb(rays_o, rays_d, self.aabb, 0.05)
        xyzs, dirs, ts, rays = march_rays_train(rays_o, rays_d, self.bound, False, self.density_bitfield, self.cascade, self.H,
                                                nears, fars, perturb, dt_gamma, max_steps)
        dirs = dirs / torch.sqrt(torch.clamp((dirs * dirs).sum(-1, keepdim=True), min=1e-20))
        with torch.autocast("cuda", dtype=torch.float16):
            sigmas, rgbs, specs = self.field(xyzs, dirs, shading)
        weights, ws, depth, image = _CompositeTrain.apply(sigmas, rgbs, ts, rays, T_thresh)
        image = image + (1 - ws).unsqueeze(-1) * bg
        return dict(image=image, weights_sum=ws, xyzs=xyzs, speculars=specs, num_points=xyzs.shape[0])

    def step(self, rays_o, rays_d, gt, bg, shading="full", lr=None):
        if lr is not None:
            for g in self.opt.param_groups:
                g["lr"] = lr
        self.opt.zero_grad()
        out = self.render(rays_o, rays_d, bg, True, shading)
        mask = gt[:, 3:]
        gt_rgb = gt[:, :3] * mask + bg * (1 - mask)
        loss = ((out["image"] - gt_rgb) ** 2).mean(-1) + self.lambda_mask * (out["weights_sum"] - mask.squeeze(1)) ** 2
        loss = loss.mean()
        if out["speculars"] is not None:
            loss = loss + self.lambda_specular * (out["speculars"] ** 2).sum(-1).mean()
        self.scaler.scale(loss).backward()
        self.scaler.unscale_(self.opt)                                     # post_train_step (utils.py:812)
        if self.lambda_tv > 0 and out["num_points"] > 0:
            self.field.encoder.grad_total_variation(self.lambda_tv, out["xyzs"], self.bound)
        self.scaler.step(self.opt)
        self.scaler.update()
        return loss, out["num_points"]

    @torch.no_grad()
    def update_extra_state(self, decay=0.95, density_thresh=10.0):
        rm, _ = backends()
        H = self.H
        idx = torch.arange(H ** 3, dtype=torch.int32, device=self.device)
        coords = torch.empty(H ** 3, 3, dtype=torch.int32, device=self.device)
        rm.morton3D_invert(idx, H ** 3, coords)
        xyzs = 2 * coords.float() / (H - 1) - 1
        for cas in range(self.cascade):
            bound = min(2 ** cas, self.bound)
            hgs = bound / H
            cas_xyzs = xyzs * (bound - hgs) + (torch.rand_like(xyzs) * 2 - 1) * hgs
            with torch.autocast("cuda", dtype=torch.float16):
                sig = self.field.density(cas_xyzs).reshape(-1)
            g = self.density_grid[cas]
            valid = (g >= 0) & (sig >= 0)
            g[valid] = torch.maximum(g[valid] * decay, sig[valid])
        mean = self.density_grid.clamp(min=0).mean().item()
        rm.packbits(self.density_grid, self.density_bitfield.numel(), min(mean, density_thresh), self.density_bitfield)

    @torch.no_grad()
    def render_eval(self, rays_o, rays_d, bg_color=1.0, shading="full", chunk=4096):
        img = torch.empty(rays_o.shape[0], 3, device=self.device)
        for a in range(0, rays_o.shape[0], chunk):
            ro, rd = rays_o[a:a + chunk].contiguous(), rays_d[a:a + chunk].contiguous()
            out = self.render(ro, rd, torch.full((ro.shape[0], 3), float(bg_color), device=self.device), False, shading)
            img[a:a + chunk] = out["image"]
        return img


def main(argv=None):
    from nerf2mesh_b200 import synthetic as S
    from nerf2mesh_b200.train_synthetic import full_image_rays, lr_at, psnr
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3000)
    ap.add_argument("--num_rays", type=int, default=4096)
    ap.add_argument("--eval_res", type=int, default=200)
    ap.add_argument("--eval_views", type=int, default=4)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--init_from_b200", action="store_true", help="start from the same parameters as Stage0Trainer(seed)")
    args = ap.parse_args(argv)
    torch.manual_seed(args.seed)
    dev = "cuda"
    bricks = S.make_bricks()
    poses = S.orbit_cameras(100, seed=0)
    test_poses = S.orbit_cameras(args.eval_views, seed=12345)
    intr = S.lego_intrinsics()
    tr = RefTrainer(1.0)
    if args.init_from_b200:
        from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
        t0 = Stage0Trainer(Stage0Config(num_rays=128, max_samples=128 * 128), seed=args.seed)
        tr.field.load_reference_state(t0.export_reference_state())
        del t0
    g = torch.Generator().manual_seed(args.seed + 1)
    t_start = time.time(); samples = 0; step_ms = []
    for it in range(args.iters):
        if it % 16 == 0:
            tr.update_extra_state()
        ro, rd, _, _ = S.sample_rays(poses, intr, 800, 800, args.num_rays, g)
        gt = S.render_bricks(ro, rd, bricks); bg = torch.rand(args.num_rays, 3, generator=g)
        _ = torch.rand(args.num_rays, generator=g)          # keep the host RNG stream aligned with train_synthetic
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        ro, rd, gt, bg = ro.to(dev), rd.to(dev), gt.to(dev), bg.to(dev)
        e0.record()
        loss, m = tr.step(ro, rd, gt, bg, "diffuse" if it < 1000 else "full", lr_at(it, args.iters))
        e1.record()
        samples += m
        if it % 250 == 0 or it == args.iters - 1:
            torch.cuda.synchronize()
            step_ms.append((it, e0.elapsed_time(e1), m))
            print({"it": it, "loss": float(loss), "samples": m, "step_ms": e0.elapsed_time(e1)}, flush=True)
    torch.cuda.synchronize()
    secs = time.time() - t_start
    scale = 800 // args.eval_res
    vals = []
    for k in range(args.eval_views):
        ro, rd = full_image_rays(test_poses[k], intr / scale, args.eval_res, args.eval_res)
        gt = S.render_bricks(ro, rd, bricks)
        gt_rgb = gt[:, :3] * gt[:, 3:] + (1 - gt[:, 3:])
        img = tr.render_eval(ro.to(dev), rd.to(dev), 1.0, "full" if args.iters > 1000 else "diffuse")
        vals.append(psnr(img.clamp(0, 1).cpu(), gt_rgb))
    print(json.dumps({"impl": "reference-cuda", "iters": args.iters, "train_seconds": secs, "psnr_views": vals,
                      "psnr_mean": sum(vals) / len(vals), "step_ms_samples": step_ms,
                      "late_samples_per_s": [m / (ms * 1e-3) for _, ms, m in step_ms[-3:]]}))


if __name__ == "__main__":
    main()
