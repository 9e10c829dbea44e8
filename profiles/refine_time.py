"""Time the stage-1 step with mesh refinement off and on (Stage1Trainer(refine=...): the per-face error scatter fused into the loss kernel).

    python profiles/refine_time.py [--steps 200] [--rounds 5] [--warmup 17] [--kernel-reps 200]

Setup of bench.py's lego_stage1 workload: icosphere(7) (327,680 faces), 800 x 800 at ssaa 2, antialias, lr_vert 1e-4, 8 views, one CUDA
graph per view.  Two trainers share one Stage0Trainer; after warming both (every view's graph captured), CUDA events time --steps steps
of each, alternating off / on (the order swapped every round) for --rounds rounds.  Every timed run starts from the same model and vertex
state (restored in place, so the captured graphs stay valid): training on random targets moves the vertices and changes the work per
step, which would otherwise drift between runs.  Then the antialiased loss kernel alone, n2m_s1_loss_aa against n2m_s1_loss_aa_err on
the same eagerly rendered view (--kernel-reps launches each, alternating blocks).  Prints one JSON line: the card's name and power limit,
ms/step per round and the medians, the low-res pixels charged per step (each adds to its face with two fp32 atomics when refinement is
on) and the loss-kernel times.

Measured on an NVIDIA H100 80GB HBM3 at a 400 W power limit (defaults, --rounds 6): 276,500 low-res pixels charged per step.  Step
medians 2.522 ms off, 2.537 ms on; the run-to-run spread (about 0.1 ms, set by which run of a pair comes second) hides the difference.
The loss kernel alone: 53.2 us off, 56.1 us on (medians of 12 blocks of 200 launches, every block within 0.3 us of its median), so the
error scatter costs about 3 us per step.
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


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=17)
    ap.add_argument("--kernel-reps", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("refine_time.py: no CUDA device")
    from nerf2mesh_b200 import synthetic as S
    from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
    from nerf2mesh_b200.stage1 import Stage1Trainer
    from nerf2mesh_b200.train_synthetic import full_image_rays
    torch.cuda.set_device(0)
    h0 = w0 = 800
    t0 = Stage0Trainer(Stage0Config(bound=1.0, num_rays=1024, max_samples=1024 * 128), seed=0)
    v, f = S.icosphere(7)
    trainers = {r: Stage1Trainer(t0, torch.from_numpy(v), torch.from_numpy(f), h0, w0, ssaa=2, antialias=True, lr_vert=1e-4, refine=r)
                for r in (False, True)}
    g = torch.Generator().manual_seed(0)
    views = []
    for k in range(8):
        cam = S.orbit_cameras(8, radius=2.35, seed=3)[k, :3, 3].numpy().astype(np.float64)
        pose = torch.from_numpy(S.look_at_pose(cam).astype(np.float32))
        intr = S.lego_intrinsics(h0, w0)
        _, rd = full_image_rays(pose, intr, h0, w0)
        mvp = S.perspective_mvp(cam, fovy=2 * np.arctan(0.5 * h0 / intr[1]), aspect=w0 / h0); mvp[1] *= -1
        gt = torch.rand(h0 * w0, 4, generator=g); gt[:, 3] = 1.0
        views.append((torch.from_numpy(mvp).cuda(), rd.cuda(), gt.cuda(), torch.rand(h0 * w0, 3, generator=g).cuda()))
    W = max(args.warmup, 17)                                # every view's graph is captured during warm-up
    for s1 in trainers.values():
        for it in range(W):
            s1.step(*views[it % 8], use_graph=True)
    vert = ("vertices", "base_vertices", "offsets", "m_vert", "v_vert", "vert_state")
    for n in vert:                                          # both trainers start every run from the same mesh
        getattr(trainers[True], n).copy_(getattr(trainers[False], n))
    torch.cuda.synchronize()
    state = [getattr(t0, n) for n in ("table", "color_master", "mlp", "m_table", "v_table", "m_mlp", "v_mlp", "wpack", "opt_state")]
    state += list(t0.gtables) + [t0.g_mlp]
    for s1 in trainers.values():
        state += [getattr(s1, n) for n in vert]
    snap = [x.clone() for x in state]
    on = trainers[True]
    on.face_errors.zero_(); on.face_counts.zero_()
    ms = {"off": [], "on": []}
    steps_on = 0
    for rnd in range(args.rounds):
        for r in ((False, True) if rnd % 2 == 0 else (True, False)):
            s1 = trainers[r]
            for x, y in zip(state, snap):
                x.copy_(y)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for it in range(args.steps):
                s1.step(*views[it % 8], use_graph=True)
            e1.record()
            torch.cuda.synchronize()
            ms["on" if r else "off"].append(e0.elapsed_time(e1) / args.steps)
            steps_on += args.steps if r else 0
    charged = float(on.face_counts.double().sum().item()) / steps_on
    # the loss kernel alone, with and without the error scatter, on one eagerly rendered view
    from nerf2mesh_b200._lib import call, ptr, stream
    mvp, rd, gt, bg = views[0]
    on.forward(mvp, rd)
    args_aa = (ptr(on.aa), ptr(gt), gt.shape[-1], ptr(bg), h0, w0, on.ssaa, on.lambda_mask, ptr(t0.opt_state), ptr(on.d_aa), ptr(on.image),
               ptr(on.weights_sum), ptr(on.loss_acc))
    err = (ptr(on.rast), ptr(on.face_errors), ptr(on.face_counts), on.triangles.shape[0])
    kern = {"off": [], "on": []}
    for rnd in range(2 * args.rounds):
        for r in (False, True):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for it in range(args.kernel_reps):
                if r:
                    call("n2m_s1_loss_aa_err", *args_aa, *err, stream())
                else:
                    call("n2m_s1_loss_aa", *args_aa, stream())
            e1.record()
            torch.cuda.synchronize()
            kern["on" if r else "off"].append(e0.elapsed_time(e1) * 1e3 / args.kernel_reps)
    name, power = card()
    med = {k: float(np.median(x)) for k, x in ms.items()}
    print(json.dumps({"device": name, "power_limit": power, "faces": int(f.shape[0]), "image": [h0, w0], "ssaa": 2, "antialias": True,
                      "lr_vert": 1e-4, "cuda_graph": True, "steps_per_round": args.steps, "rounds": args.rounds,
                      "ms_per_step": {k: [round(x, 4) for x in v] for k, v in ms.items()},
                      "median_ms_per_step": {k: round(x, 4) for k, x in med.items()},
                      "median_difference_us": round((med["on"] - med["off"]) * 1e3, 2),
                      "charged_pixels_per_step": charged,
                      "loss_aa_kernel_us": {k: round(float(np.median(x)), 2) for k, x in kern.items()},
                      "loss_aa_kernel_us_runs": {k: [round(x, 2) for x in v] for k, v in kern.items()}}))


if __name__ == "__main__":
    main()
