"""Time the stage-1 step with the colour-field vertex gradient off and on (Stage1Trainer(offset_nerf_grad=...), the reference's
--enable_offset_nerf_grad), and the new kernel n2m_s1_offset_grad alone.

    python profiles/offset_grad_time.py [--steps 200] [--rounds 5] [--warmup 17] [--kernel-reps 200]

Setup of bench.py's lego_stage1 workload: icosphere(7) (327,680 faces), 800 x 800 at ssaa 2, antialias, lr_vert 1e-4, 8 views, one CUDA
graph per view.  Two trainers share one Stage0Trainer; after warming both (every view's graph captured), CUDA events time --steps steps
of each, alternating off / on (the order swapped every round) for --rounds rounds; every timed run starts from the same model and vertex
state (restored in place, so the captured graphs stay valid).  Then n2m_s1_offset_grad alone on one eagerly rendered view (--kernel-reps
launches per block, 2 x --rounds blocks).  Prints one JSON line: the card's name and power limit, ms/step per round and the medians, the
covered super-samples of that view and the kernel time.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (defaults, --rounds 4): step medians 2.448 ms off, 2.963 ms on (+0.515 ms,
+21%); n2m_s1_offset_grad alone 458 us for 1,082,749 covered super-samples (every block of 200 launches within 1 us of the median), so
the kernel is nearly all of the option's cost.  Not tuned yet: one thread per super-sampled pixel, a 16-level colour-grid gather per
point and 21 fp32 atomics per point.
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
        raise SystemExit("offset_grad_time.py: no CUDA device")
    from nerf2mesh_b200 import synthetic as S
    from nerf2mesh_b200._lib import call, ptr, stream
    from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
    from nerf2mesh_b200.stage1 import Stage1Trainer
    from nerf2mesh_b200.train_synthetic import full_image_rays
    torch.cuda.set_device(0)
    h0 = w0 = 800
    t0 = Stage0Trainer(Stage0Config(bound=1.0, num_rays=1024, max_samples=1024 * 128), seed=0)
    v, f = S.icosphere(7)
    trainers = {r: Stage1Trainer(t0, torch.from_numpy(v), torch.from_numpy(f), h0, w0, ssaa=2, antialias=True, lr_vert=1e-4,
                                 offset_nerf_grad=r) for r in (False, True)}
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
    ms = {"off": [], "on": []}
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
    # the kernel alone on one eagerly rendered view (it accumulates into grad_vclip / grad_vworld: the sums are not read)
    on = trainers[True]
    mvp, rd, gt, bg = views[0]
    on.forward(mvp, rd)
    on.loss_backward(gt, bg)
    torch.cuda.synchronize()
    covered = int(on.counters[1].item())
    kargs = (on._pp(), ptr(on.rast), ptr(on.vertices), ptr(on.vclip), ptr(on.triangles), ptr(on.inv), on.h, on.w, ptr(on.pts),
             ptr(on.denc_tiles), ptr(t0.table), ptr(t0.offsets), ptr(on.grad_vclip), ptr(on.grad_vworld), ptr(t0.opt_state), stream())
    for _ in range(20):
        call("n2m_s1_offset_grad", *kargs)
    kern = []
    for rnd in range(2 * args.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for it in range(args.kernel_reps):
            call("n2m_s1_offset_grad", *kargs)
        e1.record()
        torch.cuda.synchronize()
        kern.append(e0.elapsed_time(e1) * 1e3 / args.kernel_reps)
    name, power = card()
    med = {k: float(np.median(x)) for k, x in ms.items()}
    print(json.dumps({"device": name, "power_limit": power, "faces": int(f.shape[0]), "image": [h0, w0], "ssaa": 2, "antialias": True,
                      "lr_vert": 1e-4, "cuda_graph": True, "steps_per_round": args.steps, "rounds": args.rounds,
                      "ms_per_step": {k: [round(x, 4) for x in v] for k, v in ms.items()},
                      "median_ms_per_step": {k: round(x, 4) for k, x in med.items()},
                      "median_difference_us": round((med["on"] - med["off"]) * 1e3, 2),
                      "covered_supersamples": covered,
                      "offset_grad_kernel_us": round(float(np.median(kern)), 2),
                      "offset_grad_kernel_us_runs": [round(x, 2) for x in kern]}))


if __name__ == "__main__":
    main()
