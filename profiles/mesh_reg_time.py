"""Time the stage-1 step with the mesh regularisers off and on (Stage1Trainer(lambda_normal=..., lambda_edgelen=...)), and their kernel
alone against the Laplacian's.

    python profiles/mesh_reg_time.py [--steps 200] [--rounds 5] [--warmup 17] [--kernel-reps 200]

Setup of bench.py's lego_stage1 workload (as profiles/refine_time.py): icosphere(7) (327,680 faces), 800 x 800 at ssaa 2, antialias,
lr_vert 1e-4, 8 views, one CUDA graph per view.  Two trainers share one Stage0Trainer: both lambdas 0, and lambda_normal 1e-3 (the
reference's indoor and unbounded recipes) with lambda_edgelen 0.1 (the value its readme lists).  After warming both, CUDA events time
--steps steps of each, alternating off / on (the order swapped every round) for --rounds rounds, every run from the same restored state.
Then, on the same mesh, n2m_s1_mesh_reg alone against the Laplacian's three launches alone (k_s1_laplacian, k_s1_lap_normalize,
k_s1_laplacian: n2m_s1_vert_step's lambda_lap part, timed as n2m_s1_vert_step with lambda_lap on minus with it off), --kernel-reps
launches each in alternating blocks (the latter also includes the Laplacian's memset of its [6V] scratch).  Prints one JSON line with the
card's name and power limit.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (defaults): 491,520 edges, every one with a normal pair.  Step medians
2.441 ms off, 2.548 ms on (+107 us, 4.4 %; every round of each within 0.02 ms of its median except one 2.53 ms "off" round).  The
regulariser kernel alone: 102.7 us (10 blocks of 200 launches, all within 0.4 us); the Laplacian's three launches and memset: 84.2 us
(117.6 us for n2m_s1_vert_step with lambda_lap on minus 33.4 us with it off).  The new walk costs about 20 % more than the two Laplacian
walks together: both make 12 scalar fp32 atomics per edge, but the new one also gathers four vertex rows per slot instead of two and reads
the slot's two opposite vertices, and its step adds a [3V] memset of its own.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from refine_time import card  # noqa: E402

LAMBDA_NORMAL, LAMBDA_EDGELEN = 1e-3, 0.1


def _time(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=17)
    ap.add_argument("--kernel-reps", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_reg_time.py: no CUDA device")
    from nerf2mesh_b200 import synthetic as S
    from nerf2mesh_b200._lib import call, ptr, stream
    from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
    from nerf2mesh_b200.stage1 import Stage1Trainer
    from nerf2mesh_b200.train_synthetic import full_image_rays
    torch.cuda.set_device(0)
    h0 = w0 = 800
    t0 = Stage0Trainer(Stage0Config(bound=1.0, num_rays=1024, max_samples=1024 * 128), seed=0)
    v, f = S.icosphere(7)
    lams = {False: (0.0, 0.0), True: (LAMBDA_NORMAL, LAMBDA_EDGELEN)}
    trainers = {r: Stage1Trainer(t0, torch.from_numpy(v), torch.from_numpy(f), h0, w0, ssaa=2, antialias=True, lr_vert=1e-4,
                                 lambda_normal=lams[r][0], lambda_edgelen=lams[r][1]) for r in (False, True)}
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
            ms["on" if r else "off"].append(_time(lambda: [s1.step(*views[it % 8], use_graph=True) for it in range(args.steps)], 1)
                                            / args.steps / 1e3)
    # the regulariser kernel alone vs the Laplacian's three launches, on the same mesh
    on = trainers[True]
    th = on.topology
    V = on.vertices.shape[0]
    grad = torch.zeros(V, 3, device="cuda")
    loss = torch.zeros(1, device="cuda")
    reg = lambda: call("n2m_s1_mesh_reg", ptr(th.keys), ptr(th.opp), th.slots, on.mesh_edges, on.mesh_pairs, ptr(on.vertices), LAMBDA_NORMAL,
                       LAMBDA_EDGELEN, ptr(grad), ptr(loss), stream())
    # n2m_s1_vert_step on scratch copies of the group (lr 0: the offsets do not move), with and without lambda_lap
    buf = {n: getattr(on, n).clone() for n in ("base_vertices", "offsets", "m_vert", "v_vert", "vertices", "grad_vclip")}
    opt = t0.opt_state.clone(); opt[3] = 0.0; opt[7] = 1.0
    vst = torch.zeros(4, device="cuda")
    scratch = torch.zeros(6 * V, device="cuda")

    def vert_step(lam_lap):
        return lambda: call("n2m_s1_vert_step", ptr(buf["grad_vclip"]), ptr(on.mvp), ptr(th.keys), th.slots, ptr(buf["base_vertices"]),
                            ptr(buf["offsets"]), ptr(buf["m_vert"]), ptr(buf["v_vert"]), ptr(buf["vertices"]), ptr(scratch), None, V, lam_lap,
                            0.0, 0.0, 1e-15, ptr(opt), ptr(vst), ptr(loss), stream())
    kern = {"mesh_reg": [], "vert_step_lap": [], "vert_step_no_lap": []}
    for f_ in (reg, vert_step(1e-3), vert_step(0.0)):
        f_()
    torch.cuda.synchronize()
    for rnd in range(2 * args.rounds):
        for name, fn in (("mesh_reg", reg), ("vert_step_lap", vert_step(1e-3)), ("vert_step_no_lap", vert_step(0.0))):
            kern[name].append(_time(fn, args.kernel_reps))
    name, power = card()
    med = {k: float(np.median(x)) for k, x in ms.items()}
    kmed = {k: float(np.median(x)) for k, x in kern.items()}
    print(json.dumps({"device": name, "power_limit": power, "faces": int(f.shape[0]), "unique_edges": on.mesh_edges, "normal_pairs": on.mesh_pairs,
                      "image": [h0, w0], "ssaa": 2, "antialias": True, "lr_vert": 1e-4, "cuda_graph": True,
                      "lambda_normal": LAMBDA_NORMAL, "lambda_edgelen": LAMBDA_EDGELEN, "steps_per_round": args.steps, "rounds": args.rounds,
                      "ms_per_step": {k: [round(x, 4) for x in v] for k, v in ms.items()},
                      "median_ms_per_step": {k: round(x, 4) for k, x in med.items()},
                      "median_difference_us": round((med["on"] - med["off"]) * 1e3, 2),
                      "kernel_us": {k: round(x, 2) for k, x in kmed.items()},
                      "laplacian_three_launches_us": round(kmed["vert_step_lap"] - kmed["vert_step_no_lap"], 2),
                      "kernel_us_runs": {k: [round(x, 2) for x in v] for k, v in kern.items()}}))


if __name__ == "__main__":
    main()
