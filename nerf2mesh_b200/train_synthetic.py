"""Train the fused stage-0 pipeline on the analytic bricks scene with the reference's lego recipe and report
test PSNR (no dataset is needed):

    python -m nerf2mesh_b200.train_synthetic --iters 3000

Recipe (reference defaults): 4096 rays/step, lr 1e-2 with LambdaLR warm-up 500 it then
0.1^((it-500)/(iters-500)) (main.py:239), 'diffuse' shading for the first 1000 steps (utils.py:669-672), density
grid update every 16 steps (utils.py:1155-1156), random background (utils.py:660), lambda_tv 1e-8 (readme.md:64).
"""
import argparse
import json
import math
import time

import torch

from . import synthetic as S
from .stage0 import Stage0Config, Stage0Trainer


def lr_at(it, iters, lr0=1e-2):
    f = 0.01 + 0.99 * (it / 500) if it <= 500 else 0.1 ** ((it - 500) / max(iters - 500, 1))
    return lr0 * f


def full_image_rays(pose, intr, H, W):
    fx, fy, cx, cy = [float(v) for v in intr]
    j, i = torch.meshgrid(torch.arange(H, dtype=torch.float32) + 0.5, torch.arange(W, dtype=torch.float32) + 0.5, indexing="ij")
    dirs = torch.stack([(i - cx) / fx, -(j - cy) / fy, -torch.ones_like(i)], -1).reshape(-1, 3)
    rays_d = dirs @ pose[:3, :3].T
    rays_o = pose[:3, 3].expand_as(rays_d)
    return rays_o.contiguous(), rays_d.contiguous()


def psnr(a, b):
    return -10.0 * math.log10(max(torch.mean((a - b) ** 2).item(), 1e-12))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3000)
    ap.add_argument("--num_rays", type=int, default=4096)
    ap.add_argument("--eval_res", type=int, default=200)
    ap.add_argument("--eval_views", type=int, default=4)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--update_interval", type=int, default=16)
    ap.add_argument("--diffuse_step", type=int, default=1000)
    ap.add_argument("--device_dataset", action="store_true",
                    help="render the training views once into a device-resident uint8 image set and sample the batches with the "
                         "on-device sampler (nerf2mesh_b200/sampler.py) instead of synthesising every batch on the host")
    ap.add_argument("--train_res", type=int, default=400, help="resolution of the device-resident training views")
    ap.add_argument("--samples_per_ray", type=int, default=512,
                    help="sample-slab capacity per ray; the cold-start occupancy grid marches far more samples than a converged one")
    ap.add_argument("--adaptive_num_rays", action="store_true",
                    help="resize every batch to march about --num_points samples, as the reference's -O preset does (main.py:68-69); "
                         "batches start at --num_rays and are drawn with 4 x --num_rays rows, of which the trainer uses the first n")
    ap.add_argument("--num_points", type=int, default=2 ** 18, help="target samples per step with --adaptive_num_rays")
    args = ap.parse_args(argv)

    torch.manual_seed(args.seed)
    dev = "cuda"
    bricks = S.make_bricks()
    poses = S.orbit_cameras(100, seed=0)
    test_poses = S.orbit_cameras(args.eval_views, seed=12345)
    intr = S.lego_intrinsics()
    cfg = Stage0Config(bound=1.0, num_rays=args.num_rays, max_samples=args.num_rays * args.samples_per_ray,
                       adaptive_num_rays=args.adaptive_num_rays, num_points=args.num_points)
    tr = Stage0Trainer(cfg, seed=args.seed)
    rows = tr.N                   # rows per batch: num_rays, or max_rays with the adaptive ray count
    # cold start as the reference: empty density grid => first update marks everything with sigma > mean
    tr.density_grid.zero_()
    g = torch.Generator().manual_seed(args.seed + 1)

    if args.device_dataset:
        from .sampler import DeviceRaySampler
        R = args.train_res
        bricks_d = tuple(t.to(dev) for t in bricks)
        intr_t = intr * (R / 800.0)
        imgs = torch.empty(poses.shape[0], R, R, 4, dtype=torch.uint8, device=dev)
        for k in range(poses.shape[0]):
            ro, rd = full_image_rays(poses[k], intr_t, R, R)
            rgba = S.render_bricks(ro.to(dev), rd.to(dev), bricks_d)
            imgs[k] = (rgba * 255).round().clamp(0, 255).to(torch.uint8).view(R, R, 4)
        sampler = DeviceRaySampler(poses, intr_t, R, R, imgs)
        gd = torch.Generator(device=dev).manual_seed(args.seed + 1)

        def batch():
            ro, rd, gt = sampler.sample(rows, generator=gd)
            bg = torch.rand(rows, 3, device=dev, generator=gd)
            noises = torch.rand(rows, device=dev, generator=gd)
            return ro, rd, gt, bg, noises
    else:
        def batch():
            ro, rd, _, _ = S.sample_rays(poses, intr, 800, 800, rows, g)
            gt = S.render_bricks(ro, rd, bricks)
            bg = torch.rand(rows, 3, generator=g)
            noises = torch.rand(rows, generator=g)
            return tuple(t.pin_memory() for t in (ro, rd, gt, bg, noises))

    t0 = time.time()
    samples = 0
    log = []
    for it in range(args.iters):
        if it % args.update_interval == 0:
            tr.update_density_grid()
        shading = "diffuse" if it < args.diffuse_step else "full"
        tr.step(*batch(), shading=shading, lr=lr_at(it, args.iters))
        if it % 250 == 0 or it == args.iters - 1:
            torch.cuda.synchronize()
            m = int(tr.counters[1].item())
            n = int(tr.counters[16].item()) if args.adaptive_num_rays else args.num_rays
            log.append({"it": it, "loss": tr.read_loss(), "n": n, "samples": m, "overflow": int(tr.counters[2].item()),
                        "occ": float((tr.density_bitfield != 0).float().mean().item()), "loss_scale": float(tr.opt_state[0].item())})
            print(log[-1], flush=True)
    torch.cuda.synchronize()
    train_s = time.time() - t0

    # test PSNR vs the analytic render on a white background
    scale = 800 // args.eval_res
    intr_e = intr / scale
    vals = []
    for k in range(args.eval_views):
        ro, rd = full_image_rays(test_poses[k], intr_e, args.eval_res, args.eval_res)
        gt = S.render_bricks(ro, rd, bricks)
        gt_rgb = gt[:, :3] * gt[:, 3:] + (1 - gt[:, 3:])
        img, ws, _ = tr.render(ro.to(dev), rd.to(dev), bg_color=1.0, shading="full" if args.iters > args.diffuse_step else "diffuse")
        vals.append(psnr(img.clamp(0, 1).cpu(), gt_rgb))
    out = {"iters": args.iters, "device_dataset": bool(args.device_dataset), "train_seconds": train_s, "psnr_views": vals, "psnr_mean": sum(vals) / len(vals), "log": log}
    print(json.dumps(out))
    return out


if __name__ == "__main__":
    main()
