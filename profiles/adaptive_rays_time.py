"""Step time and sample rate of stage 0 with a fixed 4096-ray batch against the adaptive ray count (--adaptive_num_rays of the `-O`
preset, Stage0Config.adaptive_num_rays), on bench.py's two synthetic scenes.

    python profiles/adaptive_rays_time.py [--steps 200] [--warmup 30] [--num-points 262144] [--max-rays 16384]

For each workload (lego_stage0_converged, garden_stage0: bench.WORKLOADS / bench.scene, fixed occupancy) and each mode a fresh trainer
runs `warmup` steps, then `steps` timed steps with CUDA events around the whole window (graph replay, one stream, no host sync inside).
Batches are drawn on the host beforehand (bench.make_batches' cameras, `--max-rays` rows each in adaptive mode), moved to the device and
cycled.  Every step copies its slot's counters (M in [0], n in [16]) into a device-side log, the same one small copy in both modes.
Reported per run: ms per step, mean n, mean M, samples per second (sum of M over the window / its time).  In adaptive mode the count
starts at 4096 and settles within a few steps at about num_points / (samples per ray); the occupancy grid is not updated here, so the
count does not drift the way it does while a real grid is carved.
Prints one JSON line with the device name and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=20)
        return r.stdout.strip() or None
    except Exception:      # noqa: BLE001
        return None


def batches(workload, rows, count, seed=0):
    import bench
    from nerf2mesh_b200 import synthetic as S
    w = bench.WORKLOADS[workload]
    grid, bits, bricks = bench.scene(workload)
    poses = S.orbit_cameras(100, radius=w["radius"] or S.LEGO_RADIUS, seed=0)
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(count):
        ro, rd, _, _ = S.sample_rays(poses, S.lego_intrinsics(), 800, 800, rows, g)
        gt = S.render_bricks(ro, rd, bricks)
        if not w["alpha"]:
            gt = (gt[:, :3] * gt[:, 3:] + (1 - gt[:, 3:])).contiguous()
        b = [ro, rd, gt, torch.rand(rows, 3, generator=g), torch.rand(rows, generator=g)]
        if w["cam_nf"]:
            d = ro.norm(dim=-1)
            b.append(torch.stack([(d - 1.1).clamp(min=0.05), d + 14.0], -1).contiguous())
        out.append([t.cuda() for t in b])
    return out, grid, bits


def run(workload, adaptive, args):
    import bench
    from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
    w = bench.WORKLOADS[workload]
    cfg = Stage0Config(bound=w["bound"], dt_gamma=w["dt_gamma"], lambda_entropy=w["lambda_entropy"], num_rays=4096,
                       max_samples=4096 * w["cap"], adaptive_num_rays=adaptive, num_points=args.num_points,
                       max_rays=args.max_rays if adaptive else None)
    tr = Stage0Trainer(cfg, seed=0)
    tr.use_cam_near_far = w["cam_nf"]
    bs, grid, bits = batches(workload, tr.N, 16)
    tr.set_occupancy(bits, grid)

    def step(i):
        b = bs[i % len(bs)]
        tr.step(*b[:5], cam_near_far=b[5] if len(b) > 5 else None)

    for i in range(args.warmup):
        step(i)
    torch.cuda.synchronize()
    log = torch.zeros(args.steps, 17, dtype=torch.int32, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        step(args.warmup + i)
        log[i].copy_(tr.counters)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    log = log.cpu().double()
    over, max_m = tr.check_capacity(grow=False)
    clamped, largest, _ = tr.check_rays()
    return {"ms_per_step": ms / args.steps, "mean_n": log[:, 16].mean().item() if adaptive else 4096.0,
            "mean_M": log[:, 0].mean().item(), "samples_per_s": log[:, 0].sum().item() / (ms * 1e-3),
            "overflowed_steps": over, "clamped_steps": clamped, "largest_requested_n": largest}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--num-points", type=int, default=2 ** 18)
    ap.add_argument("--max-rays", type=int, default=4 * 4096)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("adaptive_rays_time.py needs a CUDA device")
    res = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "steps": args.steps, "warmup": args.warmup,
           "num_points": args.num_points, "max_rays": args.max_rays, "runs": {}}
    for workload in ("lego_stage0_converged", "garden_stage0"):
        for mode, adaptive in (("fixed_4096", False), ("adaptive", True)):
            res["runs"][f"{workload}/{mode}"] = run(workload, adaptive, args)
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
