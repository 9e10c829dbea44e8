"""Time the two stage-1 evaluation renderers launch by launch: Stage1Trainer.render (render_stage1 at inference) and
texture.render_exported (the exported asset as the viewer draws it).

    python profiles/stage1_render_time.py [--res 800] [--ssaa 2] [--subdiv 7] [--texture 4096] [--repeats 20]

Scene: an icosphere (subdiv 7: 327,680 faces) filling most of an --res x --res view at --ssaa, an untrained colour field, for the asset a
per-triangle grid atlas and random --texture^2 uint8 textures.  Every C-ABI launch of a render call (rasterize, points, gather, MLPs,
rgba, antialias, compose; rasterize, shade, antialias, compose) is bracketed by CUDA events; after two warm-up calls the median over
--repeats calls of each launch and of the whole call is printed as one JSON line, with the card's name and power limit.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (defaults: 800x800, ssaa 2, 327,680 faces, 4096^2 textures, 32% of the
pixels covered; median of 20), in ms per call:
    Stage1Trainer.render, full          0.725  (rasterize 0.076, points 0.056, gather 0.220, MLPs 0.075, rgba 0.024, antialias 0.107,
                                                compose 0.038)
    render_exported, full, ssaa 2 + aa  0.400  (rasterize 0.076, shade 0.062, antialias 0.104, compose 0.038)
    render_exported, ssaa 1, no aa      0.217  (rasterize 0.038, shade 0.034, compose 0.020)
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


class LaunchTimer:
    """wraps the `call` of the given modules: every launch is bracketed by a pair of CUDA events, recorded under its entry point's name"""

    def __init__(self, modules):
        self.modules, self.marks = modules, []

    def _call(self, orig):
        def timed(name, *args):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); orig(name, *args); b.record()
            self.marks.append((name, a, b))
        return timed

    def __enter__(self):
        self.saved = [(m, m.call) for m in self.modules]
        for m, orig in self.saved:
            m.call = self._call(orig)
        return self

    def __exit__(self, *exc):
        for m, orig in self.saved:
            m.call = orig

    def collect(self):
        torch.cuda.synchronize()
        out = {}
        for name, a, b in self.marks:
            out[name] = out.get(name, 0.0) + a.elapsed_time(b)
        self.marks = []
        return out


def timed_runs(fn, timer, repeats):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    per, total = [], []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with timer:
            a.record(); fn(); b.record()
        per.append(timer.collect())
        total.append(a.elapsed_time(b))
    return {"ms_total": round(float(np.median(total)), 3),
            "ms": {k: round(float(np.median([p.get(k, 0.0) for p in per])), 3) for k in per[0]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=800)
    ap.add_argument("--ssaa", type=int, default=2)
    ap.add_argument("--subdiv", type=int, default=7)
    ap.add_argument("--texture", type=int, default=4096)
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stage1_render_time.py: no CUDA device")
    from nerf2mesh_b200 import raster, stage1, texture as X
    from nerf2mesh_b200 import synthetic as S
    from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
    from nerf2mesh_b200.train_synthetic import full_image_rays
    from oracle import raster_oracle as R
    import texture_oracle as TO
    torch.cuda.set_device(0)
    t0 = Stage0Trainer(Stage0Config(bound=1.0, num_rays=1024, max_samples=1024 * 128), seed=0)
    v, f = S.icosphere(args.subdiv)
    h0 = w0 = args.res
    cam = np.array([1.5, 1.1, 0.9]) * 1.3
    pose = torch.from_numpy(S.look_at_pose(cam).astype(np.float32))
    intr = S.lego_intrinsics(h0, w0)
    _, rays_d = full_image_rays(pose, intr, h0, w0)
    rays_d = rays_d.cuda().contiguous()
    mvp = R.perspective_mvp(cam, fovy=2 * np.arctan(0.5 * h0 / intr[1]), aspect=w0 / h0)
    mvp[1] *= -1
    mvp = torch.from_numpy(np.ascontiguousarray(mvp, np.float32)).cuda()
    s1 = stage1.Stage1Trainer(t0, torch.from_numpy(v), torch.from_numpy(f), h0, w0, ssaa=args.ssaa, antialias=True)
    vt, ft = TO.grid_atlas(f.shape[0])
    g = torch.Generator(device="cuda").manual_seed(0)
    tex = [torch.randint(0, 256, (args.texture, args.texture, 3), dtype=torch.uint8, device="cuda", generator=g) for _ in range(2)]
    asset = X.ExportedMesh.from_export(s1, vt, ft, (tex[0], tex[1]))
    timer = LaunchTimer([stage1, X, raster])
    name, power = card()
    res = {"device": name, "power_limit": power, "faces": int(f.shape[0]), "res": [h0, w0], "ssaa": args.ssaa, "texture": args.texture,
           "repeats": args.repeats}
    _, ws, _ = s1.render(mvp, rays_d)
    res["covered_fraction"] = round(float((ws > 0).float().mean()), 3)
    for shading in ("diffuse", "full"):
        res[f"render_{shading}"] = timed_runs(lambda: s1.render(mvp, rays_d, shading=shading), timer, args.repeats)
        res[f"render_exported_{shading}"] = timed_runs(
            lambda: X.render_exported(asset, mvp, cam, h0, w0, ssaa=args.ssaa, shading=shading, antialias=True), timer, args.repeats)
    res["render_exported_viewer"] = timed_runs(lambda: X.render_exported(asset, mvp, cam, h0, w0), timer, args.repeats)    # ssaa 1, no aa
    print(json.dumps(res))


if __name__ == "__main__":
    main()
