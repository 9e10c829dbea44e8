"""Time the stage-0 mesh clean-up on the device: remove_masked_faces + clean_mesh on the 512^3 marching-cubes mesh of the synthetic bricks scene.

    python profiles/mesh_clean_time.py [--resolution 512] [--reps 10] [--views 8]

The mesh is what export_stage0_mesh gives for a Stage0Trainer on the converged bricks occupancy (the density volume of its untrained
field, thresholded as tests/test_gpu_mcubes.py does).  The visibility mask comes from mark_unseen_triangles over --views orbit cameras at
800 x 800, computed once outside the timed window.  Timed: remove_masked_faces(dilation=5) then clean_mesh(min_f=8, min_d=5,
repair=True), the mesh_0 order of the reference's export; CUDA events around both calls (each ends in read-backs of its output sizes, the
merge in one flag per round), one warm-up run, median of --reps.  Prints one JSON line with the face counts, the merge rounds and the
card's name and power limit.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (defaults): 1,137,024 vertices / 2,274,040 faces from marching cubes,
1,116,612 faces unseen by the 8 views, 1,470,753 faces after remove_masked_faces, 742,209 vertices / 1,470,009 faces after clean_mesh
with 1 merge round (no two vertices of the masked mesh lie within r = diag / 1000 of each other); 11.8 ms for both calls (median of 5).
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from refine_time import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--resolution", type=int, default=512)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--views", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_clean_time.py: no CUDA device")
    from nerf2mesh_b200 import mesh as M
    from nerf2mesh_b200 import synthetic as S
    from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
    torch.cuda.set_device(0)

    tr = Stage0Trainer(Stage0Config(bound=1.0, num_rays=1024, max_samples=512 * 512), seed=0)
    grid, bits, _ = S.occupancy_regime("converged")
    tr.set_occupancy(bits, grid)
    thr = 0.5 * float(grid[grid > 0].min().item())
    with tempfile.TemporaryDirectory() as tmp:
        v, f = M.export_stage0_mesh(tr, tmp, resolution=args.resolution, density_thresh=thr)
    h0 = w0 = 800
    mvps = []
    for cam in S.orbit_cameras(args.views, radius=2.35, seed=3)[:, :3, 3].numpy().astype(np.float64):
        intr = S.lego_intrinsics(h0, w0)
        mvp = S.perspective_mvp(cam, fovy=2 * np.arctan(0.5 * h0 / intr[1]), aspect=w0 / h0, far=100.0); mvp[1] *= -1
        mvps.append(torch.from_numpy(np.ascontiguousarray(mvp, np.float32)))
    mvps = torch.stack(mvps).cuda()
    unseen = M.mark_unseen_triangles(v, f, mvps, h0, w0)
    torch.cuda.synchronize()

    def run(info):
        vm, fm = M.remove_masked_faces(v, f, unseen, 5)
        vc, fc = M.clean_mesh(vm, fm, min_f=8, min_d=5, repair=True, info=info)
        return fm, vc, fc

    run({})                                                             # warm-up
    ms, info = [], {}
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fm, vc, fc = run(info)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    name, power = card()
    print(json.dumps({
        "device": name, "power_limit": power, "resolution": args.resolution, "views": args.views,
        "vertices_in": int(v.shape[0]), "faces_in": int(f.shape[0]), "faces_unseen": int(unseen.sum().item()),
        "faces_after_mask": int(fm.shape[0]), "vertices_out": int(vc.shape[0]), "faces_out": int(fc.shape[0]),
        "merge_rounds": info["merge_rounds"], "reps": args.reps,
        "ms": [round(x, 3) for x in ms], "median_ms": round(float(np.median(ms)), 3)}))


if __name__ == "__main__":
    main()
