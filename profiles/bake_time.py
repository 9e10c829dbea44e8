"""Time the stage-1 texture bake (nerf2mesh_b200/texture.py) stage by stage.

    python profiles/bake_time.py [--sizes 2048 4096] [--ssaa 2] [--subdiv 7] [--repeats 3] [--oracle-max 2048]

Mesh: an icosphere (subdiv 7: 327,680 faces) with a per-triangle grid atlas (each triangle in its own cell, with gutters).  For each
texture size, after one warm-up bake, CUDA events time (median over --repeats): the UV raster, points + hash-grid gather, geo_feat,
inpaint, down-sample and the device-to-host copy of the two textures.  geo_feat's share of its shape bound: per point 128 B of gather
tile read + 4 B texel index read + 6 B written, at the data-sheet HBM bandwidth (H100 SXM: 3.35 TB/s), against 9,216 multiply-adds as
issued at the data-sheet dense fp16 rate (989 TFLOP/s) -- the bytes bound.  Also: covered and inpaint texel counts, peak device memory of
one bake_features call, and, for context at sizes up to --oracle-max, the wall time of the reference's CPU post-processing (scipy
dilation / erosion, sklearn KD-tree, cv2.resize: tests/texture_oracle.py, so the host needs scipy, scikit-learn and opencv) on the same
host's CPU.  Prints one JSON line.

Measured on an NVIDIA H100 80GB HBM3 at a 400 W power limit (defaults: 327,680 faces, ssaa 2, median of 3), in ms:
    texture  texels   covered  inpaint  uv_raster  points+gather  geo_feat (bound)  inpaint  down-sample  D2H    peak memory
    2048     4096^2   3.43 M   13.3 M   0.74       1.26           0.26 (0.14)       2.23     0.11         12.4   0.92 GiB
    4096     8192^2   13.7 M   53.4 M   2.85       4.67           1.05 (0.57)       8.80     0.28         44.6   2.00 GiB
The reference's CPU post-processing of the 2048 texture took 30.3 s on that host.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

GEO_BYTES = 128 + 4 + 6
GEO_MACS = 64 * 64 + 64 * 64 + 16 * 64
PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def bake_timed(X, t0, v, f, vt, ft, h, w, glctx):
    """one bake, stage by stage, with events; returns (times in ms, (feat0, feat1) on the host, feats, mask)"""
    ev = lambda: torch.cuda.Event(enable_timing=True)                              # noqa: E731
    t = {k: 0.0 for k in ("uv_raster", "points_gather", "geo_feat", "inpaint", "downsample", "d2h")}
    a, b = ev(), ev()
    a.record(); rast = X.uv_raster(vt, ft, h, w, glctx); b.record()
    torch.cuda.synchronize(); t["uv_raster"] = a.elapsed_time(b)
    mask = rast[0, ..., 3] > 0
    feats = torch.zeros(h, w, 6, dtype=torch.uint8, device="cuda")
    rows = max(1, min(h, X.MAX_BAND_POINTS // w))            # the band size uv_features uses
    baker = X.Baker(t0, rows * w)
    marks = []
    for y0 in range(0, h, rows):
        e0, e1, e2 = ev(), ev(), ev()
        e0.record()
        baker.points(rast, v, f, w, y0, min(h, y0 + rows))
        e1.record()
        baker.features(feats)
        e2.record()
        marks.append((e0, e1, e2))
    torch.cuda.synchronize()
    for e0, e1, e2 in marks:
        t["points_gather"] += e0.elapsed_time(e1); t["geo_feat"] += e1.elapsed_time(e2)
    del rast, baker
    a, b = ev(), ev()
    a.record(); X.inpaint(feats, mask); b.record()
    torch.cuda.synchronize(); t["inpaint"] = a.elapsed_time(b)
    a, b = ev(), ev()
    a.record(); f0, f1 = X.downscale(feats, 2); b.record()
    torch.cuda.synchronize(); t["downsample"] = a.elapsed_time(b)
    a, b = ev(), ev()
    a.record(); h0 = (f0.cpu(), f1.cpu()); b.record()
    torch.cuda.synchronize(); t["d2h"] = a.elapsed_time(b)
    return t, h0, feats, mask


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[2048, 4096])
    ap.add_argument("--ssaa", type=int, default=2)
    ap.add_argument("--subdiv", type=int, default=7)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--oracle-max", type=int, default=2048)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bake_time.py: no CUDA device")
    assert args.ssaa == 2, "the stage timings split the ssaa-2 path"
    from nerf2mesh_b200 import synthetic as S
    from nerf2mesh_b200 import raster as dr
    from nerf2mesh_b200 import texture as X
    from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
    import texture_oracle as O
    torch.cuda.set_device(0)
    t0 = Stage0Trainer(Stage0Config(bound=1.0, num_rays=1024, max_samples=1024 * 128), seed=0)
    v, f = S.icosphere(args.subdiv)
    vt, ft = O.grid_atlas(f.shape[0])
    v, f, vt, ft = (torch.from_numpy(x).cuda() for x in (v, f, vt, ft))
    glctx = dr.RasterizeCudaContext()
    name, power = card()
    res = {"device": name, "power_limit": power, "faces": int(f.shape[0]), "ssaa": args.ssaa, "repeats": args.repeats, "sizes": {}}
    for size in args.sizes:
        h = w = size * args.ssaa
        bake_timed(X, t0, v, f, vt, ft, h, w, glctx)                              # warm-up
        runs = []
        for _ in range(args.repeats):
            out = bake_timed(X, t0, v, f, vt, ft, h, w, glctx)
            runs.append(out[0])
        _, _, feats, mask = out
        _, src = X.inpaint(feats, mask, return_source=True)                      # idempotent: only counts the inpaint texels
        n_inpaint = int((src >= 0).sum())
        del src
        med = {k: float(np.median([r[k] for r in runs])) for k in runs[0]}
        covered = int(mask.sum())
        geo_bound_ms = max(2.0 * GEO_MACS * covered / PEAK_FLOPS, GEO_BYTES * covered / PEAK_BYTES) * 1e3
        entry = {"texels": h * w, "covered": covered, "inpaint": n_inpaint, "ms": {k: round(x, 3) for k, x in med.items()},
                 "ms_total": round(sum(med.values()), 3), "geo_feat_bound_ms": round(geo_bound_ms, 3),
                 "geo_feat_share_of_bound": round(geo_bound_ms / med["geo_feat"], 3)}
        del feats, mask, out
        torch.cuda.synchronize(); torch.cuda.empty_cache(); torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        X.bake_features(t0, v, f, vt, ft, size, size, ssaa=args.ssaa)
        torch.cuda.synchronize()
        entry["peak_mem_gib"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 3)
        if size <= args.oracle_max:
            fe, m = X.uv_features(t0, v, f, vt, ft, h, w)
            fe, m = fe.cpu().numpy(), m.cpu().numpy()
            c0 = time.perf_counter()
            out_cpu, *_ = O.reference_inpaint(fe, m)
            O.reference_resize(np.ascontiguousarray(out_cpu[..., :3]), size, size)
            O.reference_resize(np.ascontiguousarray(out_cpu[..., 3:]), size, size)
            entry["reference_cpu_postprocess_s"] = round(time.perf_counter() - c0, 2)
        res["sizes"][str(size)] = entry
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
