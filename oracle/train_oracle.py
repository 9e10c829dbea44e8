"""oracle/train_oracle.py -- TEST INFRASTRUCTURE ONLY (also the cpu_baseline / --impl reference leg).

PyTorch (CPU) restatement of one stage-0 train step of the reference:
  NeRFNetwork (nerf/network.py:66-189)  +  NeRFRenderer.render, training branch
  (nerf/renderer.py:676-747,804)  +  Trainer.train_step loss (nerf/utils.py:628-738)
  +  post_train_step TV gradient (utils.py:801-823)  +  Adam(eps=1e-15) (main.py:221).
The reference has no CPU path (every operator calls .cuda()); this module composes the oracle's
numpy marcher, a differentiable torch hash-grid lookup and a padded differentiable compositor,
the repo's own PyTorch restatement of the reference step.

`amp=True` emulates torch.autocast(fp16) + the reference's fp16 colour table: Linear inputs,
weights and outputs are rounded to fp16 (fp32 accumulate), sigmoid/clamp run on fp16 values.
"""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as Fnn

from . import grid_oracle, raymarching_oracle as R


# ------------------------------------------------------------------------------------------------
# differentiable hash-grid lookup (gridencoder.cu:88-196 forward math, autograd does the scatter)
# ------------------------------------------------------------------------------------------------
def grid_encode(inputs01, embeddings, offsets, S, H, half_table=False):
    """inputs01 [B,3] in [0,1]; embeddings [rows,C] (requires_grad ok) -> [B, L*C] (level-major features)."""
    B, D = inputs01.shape
    L = len(offsets) - 1
    emb = embeddings
    if half_table:
        emb = emb + (emb.detach().half().float() - emb.detach())        # straight-through fp16 rounding
    outs = []
    oob = ((inputs01 < 0) | (inputs01 > 1)).any(-1)
    for level in range(L):
        scale, res, rows = grid_oracle._level_geom(level, S, H, offsets)
        pos = (inputs01.detach().double() * float(scale) + 0.5).float()
        pg = torch.floor(pos).clamp(min=0).to(torch.int64)
        frac = pos - pg.float()
        acc = 0
        for corner in range(8):
            w = torch.ones(B)
            p = pg.clone()
            for d in range(3):
                if corner & (1 << d):
                    w = w * frac[:, d]; p[:, d] += 1
                else:
                    w = w * (1 - frac[:, d])
            row = grid_oracle._row_index(p, res, rows, 0, False) + int(offsets[level])
            acc = acc + w[:, None] * emb[row]
        acc = acc * (~oob)[:, None]
        outs.append(acc)
    return torch.cat(outs, -1)


def _h(x):
    """fp16 rounding with straight-through gradient."""
    return x + (x.detach().half().float() - x.detach())


class Linear16(nn.Module):
    """bias-free Linear; with amp=True behaves like nn.Linear under autocast(fp16)."""

    def __init__(self, i, o):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(o, i))
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))      # nn.Linear default init

    def forward(self, x, amp):
        if amp:
            return _h(Fnn.linear(_h(x), _h(self.weight)))
        return Fnn.linear(x, self.weight)


class MLP(nn.Module):
    """nerf/network.py:10-54 (bias=False, ReLU)."""

    def __init__(self, dim_in, dim_out, dim_hidden, num_layers):
        super().__init__()
        self.net = nn.ModuleList([Linear16(dim_in if l == 0 else dim_hidden, dim_out if l == num_layers - 1 else dim_hidden)
                                  for l in range(num_layers)])

    def forward(self, x, amp):
        for l, lin in enumerate(self.net):
            x = lin(x, amp)
            if l != len(self.net) - 1:
                x = torch.relu(x)
        return x


class _Enc(nn.Module):
    def __init__(self, rows, C):
        super().__init__()
        self.embeddings = nn.Parameter(torch.empty(rows, C).uniform_(-1e-4, 1e-4))     # grid.py:144-146


class _TruncExp(torch.autograd.Function):
    """activation.py:5-17"""
    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        return g * torch.exp(ctx.saved_tensors[0].clamp(-15, 15))


class OracleField(nn.Module):
    """Parameter names match the reference checkpoint schema:
    encoder.embeddings, encoder_color.embeddings, sigma_net.net.{0,1}.weight,
    color_net.net.{0,1,2}.weight, specular_net.net.{0,1}.weight."""

    def __init__(self, bound=1.0, num_levels=16, log2_hashmap_size=19, base_resolution=16):
        super().__init__()
        self.bound = float(bound)
        desired = 2048 * bound
        self.per_level_scale = float(np.exp2(np.log2(desired / base_resolution) / (num_levels - 1)))
        self.S = float(np.log2(self.per_level_scale))
        self.H = base_resolution
        self.offsets = grid_oracle.level_offsets(3, num_levels, self.per_level_scale, base_resolution, log2_hashmap_size)
        rows = int(self.offsets[-1])
        self.encoder = _Enc(rows, 1)
        self.encoder_color = _Enc(rows, 2)
        self.sigma_net = MLP(3 + num_levels, 1, 32, 2)
        self.color_net = MLP(3 + 2 * num_levels, 6, 64, 3)
        self.specular_net = MLP(6, 3, 32, 2)

    def density(self, x, amp=True):
        x01 = (x + self.bound) / (2 * self.bound)
        h = grid_encode(x01, self.encoder.embeddings, self.offsets, self.S, self.H, half_table=False)
        h = self.sigma_net(torch.cat([x, h], -1), amp)
        return _TruncExp.apply(h[..., 0])

    def forward(self, x, d, shading="full", amp=True):
        sigma = self.density(x, amp)
        x01 = (x + self.bound) / (2 * self.bound)
        h = grid_encode(x01, self.encoder_color.embeddings, self.offsets, self.S, self.H, half_table=amp)
        h = self.color_net(torch.cat([x, h], -1), amp)
        feat = torch.sigmoid(h)
        if amp:
            feat = _h(feat)
        diffuse = feat[..., :3]
        if shading == "diffuse":
            return sigma, diffuse, None
        spec = torch.sigmoid(self.specular_net(torch.cat([d, feat[..., 3:]], -1), amp))
        if amp:
            spec = _h(spec)
        color = spec + diffuse
        if amp:
            color = _h(color)
        return sigma, color.clamp(0, 1), spec


# ------------------------------------------------------------------------------------------------
# differentiable compositor (raymarching.cu:501-578 as padded tensor algebra)
# ------------------------------------------------------------------------------------------------
def composite_train(sigmas, rgbs, ts, rays, T_thresh=1e-4):
    rays = torch.as_tensor(rays).long()
    N = rays.shape[0]
    cnt = rays[:, 1]
    K = int(cnt.max().item()) if N else 0
    M = sigmas.shape[0]
    if K == 0:
        z = sigmas.sum() * 0
        return torch.zeros(M) + z, torch.zeros(N) + z, torch.zeros(N) + z, torch.zeros(N, 3) + z
    k = torch.arange(K)[None, :]
    valid = k < cnt[:, None]
    idx = (rays[:, :1] + k).clamp(max=max(M - 1, 0))
    sig = sigmas[idx] * valid
    dt = ts[:, 1][idx]
    tt = ts[:, 0][idx]
    alpha = (1 - torch.exp(-sig * dt)) * valid
    Tpost = torch.cumprod(1 - alpha, 1)
    Tpre = torch.cat([torch.ones(N, 1), Tpost[:, :-1]], 1)
    # the kernel stops AFTER the first sample whose post-update T drops below the threshold
    stopped_before = torch.cat([torch.zeros(N, 1, dtype=torch.bool), (Tpost < T_thresh)[:, :-1]], 1)
    live = valid & ~(torch.cumsum(stopped_before.int(), 1) > 0)
    w = alpha * Tpre * live
    weights = torch.zeros(M) + sigmas.sum() * 0
    weights = weights.index_put((idx[live],), w[live])
    ws = w.sum(1)
    depth = (w * tt).sum(1)
    image = (w[..., None] * rgbs[idx]).sum(1)
    return weights, ws, depth, image


class _CompositeRef(torch.autograd.Function):
    """composite_rays_train with the REFERENCE's backward (raymarching.py:248-302 -> raymarching.cu:605-694), which adds
    grad_weights[k] to grad_weights_sum in sample k's own term instead of differentiating the weights exactly.  Needed
    whenever a loss touches `weights` (the entropy regulariser); identical to autograd when grad_weights == 0."""

    @staticmethod
    def forward(ctx, sigmas, rgbs, ts, rays, T_thresh):
        w, ws, depth, image = R.composite_rays_train_forward(sigmas.detach().numpy(), rgbs.detach().numpy(), ts.numpy(),
                                                             np.asarray(rays), T_thresh)
        out = [torch.from_numpy(np.ascontiguousarray(a)) for a in (w, ws, depth, image)]
        ctx.save_for_backward(sigmas.detach(), rgbs.detach(), ts, *out[1:])
        ctx.rays, ctx.T = np.asarray(rays), T_thresh
        return tuple(out)

    @staticmethod
    def backward(ctx, gw, gws, gd, gi):
        sigmas, rgbs, ts, ws, depth, image = ctx.saved_tensors
        g_sig, g_rgb = R.composite_rays_train_backward(gw.numpy(), gws.numpy(), gd.numpy(), gi.numpy(), sigmas.numpy(),
                                                       rgbs.numpy(), ts.numpy(), ctx.rays, ws.numpy(), depth.numpy(),
                                                       image.numpy(), ctx.T)
        return torch.from_numpy(g_sig), torch.from_numpy(g_rgb), None, None, None


# ------------------------------------------------------------------------------------------------
# one train step
# ------------------------------------------------------------------------------------------------
def render_train(field, rays_o, rays_d, bits, cfg, noises, bg_color, shading="full", amp=True):
    """renderer.py:688-747,804."""
    b = cfg["bound"]
    aabb = [-b, -b, -b, b, b, b]
    nears, fars = R.near_far_from_aabb(rays_o.numpy(), rays_d.numpy(), aabb, cfg.get("min_near", 0.05))
    xyzs, dirs, ts, rays = R.march_rays_train(rays_o.numpy(), rays_d.numpy(), b, cfg.get("contract", False), bits.numpy(),
                                              cfg["C"], cfg["H"], nears, fars, noises.numpy(), cfg.get("dt_gamma", 0.0),
                                              cfg.get("max_steps", 1024))
    xyzs = torch.from_numpy(xyzs); dirs = torch.from_numpy(dirs); ts = torch.from_numpy(ts)
    dirs = dirs / torch.sqrt(torch.clamp((dirs * dirs).sum(-1, keepdim=True), min=1e-20))      # safe_normalize
    sigmas, rgbs, specs = field(xyzs, dirs, shading, amp)
    if cfg.get("ref_composite", False):
        weights, ws, depth, image = _CompositeRef.apply(sigmas.float(), rgbs.float(), ts, rays, cfg.get("T_thresh", 1e-4))
    else:
        weights, ws, depth, image = composite_train(sigmas, rgbs.float(), ts, rays, cfg.get("T_thresh", 1e-4))
    image = image + (1 - ws).unsqueeze(-1) * bg_color
    return dict(image=image, weights_sum=ws, depth=depth, weights=weights, xyzs=xyzs, dirs=dirs, ts=ts, rays=rays,
                sigmas=sigmas, rgbs=rgbs, speculars=specs, num_points=xyzs.shape[0])


def train_loss(out, gt_rgba, bg_color, lambda_mask=0.1, lambda_specular=1e-5, lambda_entropy=0.0):
    """utils.py:660-667,679-683,728-738 (MSE criterion, reduction='none')."""
    if gt_rgba.shape[-1] == 4:
        mask = gt_rgba[:, 3:]
        gt_rgb = gt_rgba[:, :3] * mask + bg_color * (1 - mask)
    else:
        mask, gt_rgb = None, gt_rgba
    loss = ((out["image"] - gt_rgb) ** 2).mean(-1)
    if mask is not None and lambda_mask > 0:
        loss = loss + lambda_mask * (out["weights_sum"] - mask.squeeze(1)) ** 2
    loss = loss.mean()
    if lambda_entropy > 0:
        w = out["weights"].clamp(1e-5, 1 - 1e-5)
        e = -w * torch.log2(w) - (1 - w) * torch.log2(1 - w)
        w2 = out["weights_sum"].clamp(1e-5, 1 - 1e-5)
        e2 = -w2 * torch.log2(w2) - (1 - w2) * torch.log2(1 - w2)
        loss = loss + lambda_entropy * (e.mean() + e2.mean())
    if lambda_specular > 0 and out["speculars"] is not None:
        loss = loss + lambda_specular * (out["speculars"].float() ** 2).sum(-1).mean()
    return loss


def train_step(field, optimizer, rays_o, rays_d, gt_rgba, bits, cfg, noises, bg_color, shading="full", amp=True,
               lambda_tv=1e-8, lambda_mask=0.1, lambda_specular=1e-5):
    """One optimizer step (utils.py:1163-1179): zero_grad, render, loss, backward, TV grad, Adam."""
    optimizer.zero_grad(set_to_none=False)
    out = render_train(field, rays_o, rays_d, bits, cfg, noises, bg_color, shading, amp)
    loss = train_loss(out, gt_rgba, bg_color, lambda_mask, lambda_specular)
    loss.backward()
    if lambda_tv > 0 and out["num_points"] > 0:
        x01 = (out["xyzs"] + field.bound) / (2 * field.bound)
        tv = grid_oracle.grad_total_variation(x01, field.encoder.embeddings.detach(), field.offsets, lambda_tv, field.S, field.H)
        field.encoder.embeddings.grad += tv.float()
    optimizer.step()
    return loss.item(), out
