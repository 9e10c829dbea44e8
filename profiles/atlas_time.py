"""Time the device UV atlas, step by step, next to the feature bake of the same mesh.

    python profiles/atlas_time.py [--resolution 512] [--target 300000] [--reps 3] [--sizes 2048 4096]

The mesh is profiles/decimate_time.py's: the converged bricks scene's 512^3 marching-cubes mesh, cleaned and decimated to --target faces
on the device (outside the timed window).  For each texture size (ssaa 2): uv_unwrap, one warm-up, then --reps timed calls with CUDA
events around each; every C entry the unwrap calls gets events of its own (the host's read-backs of the chart count, the scale, the
conflict count and the row count sit between entries), summed per entry.  Then bake_features of the same mesh on that atlas with the
same trainer.  Prints one JSON line with the card's name and power limit.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (defaults, 150,004 vertices / 300,000 faces, median of 3):
- texture 2048: 34,234 charts after 2 split rounds, utilization 0.478.  uv_unwrap 17.2 ms against 7.1 ms for bake_features.
- texture 4096: 35,298 charts after 2 split rounds, utilization 0.567.  uv_unwrap 20.2 ms against 23.5 ms for bake_features.
- by step (2048 / 4096, summed over the 3 packings): n2m_atlas_pack 9.5 / 9.4 ms (one CTA, 26 layouts per packing), conflicts 2.2 /
  4.7 ms, orient 1.8 / 2.1 ms, the bitonic sorts 1.8 / 1.8 ms, everything else below 0.25 ms each.
So the unwrap is cheaper than the bake at 4096 but not at 2048; the single-CTA bisection is where the time goes.
"""
import argparse
import json
import os
import sys
import tempfile
from collections import defaultdict

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
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", type=int, nargs="+", default=[2048, 4096])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("atlas_time.py: no CUDA device")
    from nerf2mesh_b200 import mesh as M
    from nerf2mesh_b200 import synthetic as S
    from nerf2mesh_b200 import texture as X
    from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
    torch.cuda.set_device(0)

    tr = Stage0Trainer(Stage0Config(bound=1.0, num_rays=1024, max_samples=512 * 512), seed=0)
    grid, bits, _ = S.occupancy_regime("converged")
    tr.set_occupancy(bits, grid)
    thr = 0.5 * float(grid[grid > 0].min().item())
    with tempfile.TemporaryDirectory() as tmp:
        v, f = M.export_stage0_mesh(tr, tmp, resolution=args.resolution, density_thresh=thr)
    v, f = M.clean_mesh(v, f, min_f=8, min_d=5, repair=True)
    v, f = M.decimate_mesh(v, f, args.target)
    torch.cuda.synchronize()

    steps = defaultdict(list)
    plain_call = X.call

    def timed_call(name, *a):                    # events around every entry of the unwrap
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        plain_call(name, *a)
        e1.record()
        steps[name].append((e0, e1))

    result = {}
    for size in args.sizes:
        info = {}
        vt, ft, _ = X.uv_unwrap(v, f, size, ssaa=2, info=info)                 # warm-up
        total = []
        per = defaultdict(float)
        for _ in range(args.reps):
            steps.clear()
            X.call = timed_call
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            X.uv_unwrap(v, f, size, ssaa=2)
            e1.record()
            X.call = plain_call
            torch.cuda.synchronize()
            total.append(e0.elapsed_time(e1))
            for name, evs in steps.items():
                per[name] += sum(a.elapsed_time(b) for a, b in evs) / args.reps
        X.bake_features(tr, v, f, vt, ft, size, size, ssaa=2)                  # warm-up
        bake = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            X.bake_features(tr, v, f, vt, ft, size, size, ssaa=2)
            e1.record()
            torch.cuda.synchronize()
            bake.append(e0.elapsed_time(e1))
        result[str(size)] = {"charts": info["charts"], "split_rounds": info["split_rounds"], "utilization": round(info["utilization"], 4),
                             "texels_per_unit": round(info["texels_per_unit"], 3), "unwrap_median_ms": round(float(np.median(total)), 3),
                             "steps_ms": {k[len("n2m_"):]: round(x, 3) for k, x in sorted(per.items(), key=lambda kv: -kv[1])},
                             "bake_median_ms": round(float(np.median(bake)), 3)}
    name, power = card()
    print(json.dumps({"device": name, "power_limit": power, "vertices": int(v.shape[0]), "faces": int(f.shape[0]), "reps": args.reps,
                      **result}))


if __name__ == "__main__":
    main()
