"""Time the outer-cascade meshes of an unbounded scene and what they cost the stage-1 step.

    python profiles/cascade_time.py [--env-reso 256] [--reps 5] [--steps 100] [--rounds 3]

1. export_outer_meshes on the garden_scene(bound=16) density grid (5 cascades): per outer cascade, the device time of its chain (occupancy
   volume, marching cubes, transform + selection, vertex removal; a host clock around work that ends in a synchronise -- marching cubes and
   the removal each read their output sizes back), median of --reps runs, and the mesh sizes.
2. The stage-1 step (800 x 800, ssaa 2, antialias, lr_vert 1e-4, 8 views around the inner mesh) on the inner mesh alone (icosphere(7),
   327,680 faces) and on the inner mesh + the outer meshes of 1. as they come from the device (not cleaned or decimated), eager and with
   one CUDA graph per view; CUDA events over --steps steps, alternating the two meshes, --rounds rounds, every run from the same state.
Prints one JSON line with the card's name and power limit.

Measured on an NVIDIA H100 80GB HBM3 at a 400 W power limit (defaults): the outer chain takes 1.24 / 1.19 / 1.15 / 1.19 ms for cascades
1-4 (4.8 ms in all) and gives 118k / 128k / 180k / 40k vertices (234k / 252k / 357k / 78k faces).  Step medians: 2.64 ms eager and
2.63 ms with graphs on the inner mesh (327,680 faces), 5.87 / 5.87 ms on inner + outer (1,249,582 faces, every one of the 2.56 M
super-samples covered instead of 1.1 M).  The outer meshes here are not decimated; the reference's decimation to decimate_target // 2
faces per cascade makes them smaller.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from refine_time import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--env-reso", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cascade_time.py: no CUDA device")
    from nerf2mesh_b200 import mesh as M
    from nerf2mesh_b200 import synthetic as S
    from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
    from nerf2mesh_b200.stage1 import Stage1Trainer
    from nerf2mesh_b200.train_synthetic import full_image_rays
    torch.cuda.set_device(0)
    R = args.env_reso

    # ---- 1. the outer meshes -----------------------------------------------------------------------------------------------------
    grid, bits, _ = S.garden_scene(bound=16.0)
    t0 = Stage0Trainer(Stage0Config(bound=16.0, num_rays=1024, max_samples=1024 * 128), seed=0)
    t0.set_occupancy(bits, grid)
    t0.mean_density = torch.tensor([0.5], device=t0.device)
    c = t0.cfg
    xmn, ymn, zmn, xmx, ymx, zmx = t0.aabb.cpu().numpy().astype(np.float64).tolist()

    def chain(cas):
        bound = min(2 ** cas, c.bound)
        half = bound / R
        vol = M.outer_occupancy(t0.density_grid[cas], c.grid_size, R, 0.5)
        v, f = M.marching_cubes(vol, 0.5)
        if v.shape[0] == 0:
            return v, f
        v, removed = M.outer_select(v, R, bound - half, (xmn + half, ymn + half, zmn + half, xmx - half, ymx - half, zmx - half))
        return M.remove_selected_vertices(v, f, removed)

    export_ms, sizes = {}, {}
    for cas in range(1, c.cascade):
        chain(cas)                                                     # warm-up
        ts = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            a = time.perf_counter()
            v, f = chain(cas)
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - a) * 1e3)
        export_ms[cas] = round(float(np.median(ts)), 3)
        sizes[cas] = [int(v.shape[0]), int(f.shape[0])]
    with tempfile.TemporaryDirectory() as tmp:
        outer = M.export_outer_meshes(t0, tmp, env_reso=R)            # the same meshes, through the public entry point
    torch.cuda.synchronize()

    # ---- 2. the stage-1 step with and without them --------------------------------------------------------------------------------
    h0 = w0 = 800
    v, f = S.icosphere(7)
    vs = [torch.from_numpy(v)] + [outer[k][0] for k in sorted(outer)]
    fs = [torch.from_numpy(f)] + [outer[k][1] for k in sorted(outer)]
    kw = dict(ssaa=2, antialias=True, lr_vert=1e-4)
    trainers = {"inner": Stage1Trainer(t0, vs[0], fs[0], h0, w0, **kw), "inner+outer": Stage1Trainer(t0, vs, fs, h0, w0, **kw)}
    g = torch.Generator().manual_seed(0)
    views = []
    for k in range(8):
        cam = S.orbit_cameras(8, radius=2.35, seed=3)[k, :3, 3].numpy().astype(np.float64)
        pose = torch.from_numpy(S.look_at_pose(cam).astype(np.float32))
        intr = S.lego_intrinsics(h0, w0)
        _, rd = full_image_rays(pose, intr, h0, w0)
        mvp = S.perspective_mvp(cam, fovy=2 * np.arctan(0.5 * h0 / intr[1]), aspect=w0 / h0, far=100.0); mvp[1] *= -1
        gt = torch.rand(h0 * w0, 4, generator=g); gt[:, 3] = 1.0
        views.append((torch.from_numpy(np.ascontiguousarray(mvp, np.float32)).cuda(), rd.cuda(), gt.cuda(),
                      torch.rand(h0 * w0, 3, generator=g).cuda()))
    for s1 in trainers.values():                                       # every view's graph captured
        for it in range(17):
            s1.step(*views[it % 8], use_graph=True)
    torch.cuda.synchronize()
    vert = ("vertices", "base_vertices", "offsets", "m_vert", "v_vert", "vert_state")
    state = [getattr(t0, n) for n in ("table", "color_master", "mlp", "m_table", "v_table", "m_mlp", "v_mlp", "wpack", "opt_state")]
    state += list(t0.gtables) + [t0.g_mlp]
    for s1 in trainers.values():
        state += [getattr(s1, n) for n in vert]
    snap = [x.clone() for x in state]
    ms = {(m, gr): [] for m in trainers for gr in ("eager", "graph")}
    covered = {}
    for rnd in range(args.rounds):
        for mode in ("eager", "graph"):
            for name in (list(trainers) if rnd % 2 == 0 else list(trainers)[::-1]):
                s1 = trainers[name]
                for x, y in zip(state, snap):
                    x.copy_(y)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for it in range(args.steps):
                    s1.step(*views[it % 8], use_graph=mode == "graph")
                e1.record()
                torch.cuda.synchronize()
                ms[name, mode].append(e0.elapsed_time(e1) / args.steps)
                covered[name] = int(s1.counters[0].item())
    name, power = card()
    print(json.dumps({
        "device": name, "power_limit": power, "env_reso": R,
        "outer_export_ms_per_cascade": export_ms, "outer_mesh_vertices_faces": sizes,
        "outer_export_total_ms": round(sum(export_ms.values()), 3),
        "step_faces": {n: int(s.triangles.shape[0]) for n, s in trainers.items()},
        "step_covered_pixels_last_view": covered, "image": [h0, w0], "ssaa": 2, "antialias": True, "lr_vert": 1e-4,
        "steps_per_run": args.steps, "rounds": args.rounds,
        "ms_per_step": {f"{n}/{m}": [round(x, 4) for x in v] for (n, m), v in ms.items()},
        "median_ms_per_step": {f"{n}/{m}": round(float(np.median(v)), 4) for (n, m), v in ms.items()}}))


if __name__ == "__main__":
    main()
