"""Cost of the per-image appearance codes (Stage0Config.ind_dim) in the graph-replayed stage-0 step, on bench.py's lego and garden batches.

    python profiles/ind_codes_time.py [--parent DIR] [--rounds 3] [--steps 200] [--warmup 30]

Each measurement runs in a fresh process: a trainer configured as bench.py's (bench.make_trainer: same config, two ray-range parts, fixed
occupancy, the next batch's march prefetched), `warmup` steps, then `steps` graph-replayed steps between two CUDA events.  With codes the
ind_num = 100 code rows are drawn per ray (random_image_batch), one int32 [4096] index tensor per batch, staged with its batch.  Modes:
this tree at ind_dim = 0, 4 and 10 and, with --parent (a built checkout of the parent commit), the parent at ind_dim = 0; all of them
are run in turn, `rounds` times, so that drift of the shared machine spreads over every mode.  Prints one JSON line: the device, its
power limit, and per workload and mode the ms per step of every round.

Measured on an H100 80GB HBM3 at 700 W (2 rounds of 100 steps, ms per step):
    lego   parent 0: 1.0115 1.0079   branch 0: 1.0034 1.0055   branch 4: 1.0315 1.0308   branch 10: 1.0307 1.0297
    garden parent 0: 2.1241 2.1257   branch 0: 2.1302 2.1293   branch 4: 2.1605 2.1689   branch 10: 2.1564 2.1570
Without codes the step is as fast as the parent's, within the spread between rounds (the MLP backward kernel, which gained the
code-column weight-gradient branch, is the only changed kernel that ind_dim = 0 runs).  Codes cost about 0.03 ms per step on both
workloads (+2.6 % lego, +1.5 % garden), the same for D = 4 and D = 10: the per-ray code-gradient pass and the three small optimizer
launches, not the per-sample width of the code columns.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def worker(tree, workload, D, steps, warmup):
    sys.path.insert(0, tree)
    import torch
    import bench
    from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
    w = bench.WORKLOADS[workload]
    batches, grid, bits = bench.make_batches(8, 0, False, workload)
    batches = [{k: v.cuda() for k, v in b.items()} for b in batches]
    kw = dict(ind_dim=D, ind_num=100) if D else {}
    cfg = Stage0Config(bound=w["bound"], dt_gamma=w["dt_gamma"], lambda_entropy=w["lambda_entropy"], num_rays=bench.NUM_RAYS,
                       max_samples=bench.NUM_RAYS * w["cap"], **kw)
    tr = Stage0Trainer(cfg, seed=0)
    tr.use_cam_near_far = w["cam_nf"]
    tr.nparts = 2
    tr.set_occupancy(bits, grid)
    g = torch.Generator(device="cuda").manual_seed(0)
    idx = [torch.randint(0, 100, (bench.NUM_RAYS,), device="cuda", generator=g, dtype=torch.int32) for _ in batches]

    def args_of(i):
        b = batches[i % len(batches)]
        return (b["ro"], b["rd"], b["gt"], b["bg"], b["noises"]), b.get("cnf"), idx[i % len(batches)]

    def step(i):
        a, cnf, ix = args_of(i)
        n, ncnf, nix = args_of(i + 1)
        extra = dict(index=ix, next_index=nix) if D else {}
        tr.step(*a, cam_near_far=cnf, next_batch=n if ncnf is None else (*n, ncnf), use_graph=True, **extra)

    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(warmup, warmup + steps):
        step(i)
    e1.record()
    torch.cuda.synchronize()
    print(json.dumps({"ms_per_step": e0.elapsed_time(e1) / steps}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--worker", nargs=3, default=None)
    a = ap.parse_args()
    if a.worker:
        tree, workload, D = a.worker
        worker(tree, workload, int(D), a.steps, a.warmup)
        return
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    modes = [("branch", ROOT, 0), ("branch", ROOT, 4), ("branch", ROOT, 10)]
    if a.parent:
        modes.insert(0, ("parent", os.path.abspath(a.parent), 0))
    res = {}
    for workload in ("lego_stage0_converged", "garden_stage0"):
        for _ in range(a.rounds):
            for tag, tree, D in modes:
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", tree, workload, str(D), "--steps", str(a.steps),
                                    "--warmup", str(a.warmup)], capture_output=True, text=True, cwd=tree)
                if r.returncode != 0:
                    raise RuntimeError(r.stderr[-2000:])
                ms = json.loads(r.stdout.strip().splitlines()[-1])["ms_per_step"]
                res.setdefault(workload, {}).setdefault(f"{tag}_ind_dim_{D}", []).append(round(ms, 4))
    print(json.dumps({"device": q.stdout.strip(), "steps": a.steps, "rounds": a.rounds, "ms_per_step": res}))


if __name__ == "__main__":
    main()
