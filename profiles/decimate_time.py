"""Time the stage-0 mesh decimation on the device: decimate_mesh on the cleaned 512^3 marching-cubes mesh of the synthetic bricks scene.

    python profiles/decimate_time.py [--resolution 512] [--target 300000] [--reps 5] [--views 8]

The mesh is what profiles/mesh_clean_time.py cleans: export_stage0_mesh of a Stage0Trainer on the converged bricks occupancy, then
remove_masked_faces(dilation=5) over the faces --views orbit cameras at 800 x 800 see and clean_mesh(min_f=8, min_d=5, repair=True), all
outside the timed window.  Timed: decimate_mesh to --target faces (the reference's decimate_target default, 3e5) with optimal placement
(mesh_0) and with midpoints (the outer cascades' setting); CUDA events around the call (it ends in read-backs of the output sizes, and
reads one face count per round), one warm-up run per placement, median of --reps.  Prints one JSON line with the face counts, the rounds
and the card's name and power limit.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (defaults): 742,209 vertices / 1,470,009 faces in, 300,000 faces out with
either placement.  Optimal placement: 146 rounds, 288 ms (median of 5), 153,209 vertices out.  Midpoints: 180 rounds, 336 ms, 153,191
vertices out.  That is about 2 ms per round either way; the bricks' flat faces cost exactly 0, so their keys order by edge id alone.
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
    ap.add_argument("--target", type=int, default=300000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--views", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decimate_time.py: no CUDA device")
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
    v, f = M.remove_masked_faces(v, f, M.mark_unseen_triangles(v, f, mvps, h0, w0), 5)
    v, f = M.clean_mesh(v, f, min_f=8, min_d=5, repair=True)
    torch.cuda.synchronize()

    result = {}
    for name, optimal in (("optimal", True), ("midpoint", False)):
        M.decimate_mesh(v, f, args.target, optimal_placement=optimal)          # warm-up
        ms, info = [], {}
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            vo, fo = M.decimate_mesh(v, f, args.target, optimal_placement=optimal, info=info)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        result[name] = {"vertices_out": int(vo.shape[0]), "faces_out": int(fo.shape[0]), "rounds": info["rounds"], "stalled": info["stalled"],
                        "ms": [round(x, 3) for x in ms], "median_ms": round(float(np.median(ms)), 3)}
    name, power = card()
    print(json.dumps({"device": name, "power_limit": power, "resolution": args.resolution, "views": args.views, "target": args.target,
                      "vertices_in": int(v.shape[0]), "faces_in": int(f.shape[0]), "reps": args.reps, **result}))


if __name__ == "__main__":
    main()
