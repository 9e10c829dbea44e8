"""How much of the stage-0 table optimizer can hide under the hash-grid scatter, on bench.py's batches.

    python profiles/optimizer_overlap_time.py [--iters 100] [--warmup 10] [--workload lego_stage0_converged garden_stage0]

For each workload: builds bench.py's batch and trainer (bench.make_batches, bench.make_trainer), runs the step's forward stages and
the MLP backward once (so that `denc` holds real gradients), then times with CUDA events over many warm launches
  * "scatter": the two ray-range parts' scatters (n2m_s0_encode_bwd), each on its own stream, fork to join -- as the step runs them;
  * "adam": the table optimizer sweep (n2m_s0_adam_tables_keep) alone;
  * "serial": the scatters, then the sweep, on one fork-join (the order of today's step);
  * "overlapped": the scatters and the sweep at once, each on its own stream.
The sweep reads a snapshot of the gradient table that one scatter left behind, so the two phases share no buffer (the scatter never
reads the parameter table).  `saved_us` = serial - overlapped is the most that updating each level group's rows as soon as the
scatter has finished them could take off the step.
Bytes each phase must move are computed from the shapes: the scatter as in profiles/grid_pass_time.py (records + gradient chunks +
one fill and write-back of every touched 32 B sector of the gradient table), the sweep as 56 B read (gradient 16, moments 24,
table 8, colour master 8) and 40 B written per row.
Prints one JSON line per workload with the device name and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BYTES = 3.35e12          # H100 SXM data-sheet HBM3 bandwidth


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=20)
        return r.stdout.strip() or None
    except Exception:      # noqa: BLE001
        return None


def run(workload, iters, warmup):
    import bench
    from nerf2mesh_b200._lib import call, ptr, stream
    tr = bench.make_trainer(workload)
    host, grid, bits = bench.make_batches(1, 1000, False, workload)
    b = {k: v.cuda() for k, v in host[0].items()}
    tr.set_occupancy(bits, grid)
    tr._fill_params(shading_full=True, gt_has_alpha=bench.WORKLOADS[workload]["alpha"])
    tr.slots[tr.cur].load(b["ro"], b["rd"], b["gt"], b["bg"], b["noises"], b.get("cnf"))
    tr.loss_acc.zero_()
    for s in ("march", "encode_fwd", "tv", "mlp_fwd", "composite_loss", "mlp_bwd"):
        getattr(tr, s)()
    torch.cuda.synchronize()
    M = int(tr.counters[1].item())

    gt = tr.gtables[tr.parity]
    gt.zero_()
    tr.encode_bwd(0, 2)
    tr.encode_bwd(1, 2)
    call("n2m_s0_adam_head", ptr(tr.g_mlp), ptr(tr.opt_state), stream())
    torch.cuda.synchronize()
    found_inf = float(tr.opt_state[3].item())
    tr.opt_state[3] = 0.0                       # a skipped sweep reads the gradients only: time the full one
    snap = gt.clone()
    touched = (snap != 0).any(1)
    R = touched.numel()
    pad = (-R) % 4
    t4 = torch.nn.functional.pad(touched, (0, pad)).view(-1, 4)
    g_sectors = int(t4.view(-1, 2).any(1).sum().item())
    bytes_ = {"scatter": M * (16 + 7 * 16) + g_sectors * 64, "adam": R * (56 + 40)}

    main = torch.cuda.current_stream()
    streams = [torch.cuda.Stream() for _ in range(3)]

    def scatter():
        for s in streams[:2]:
            s.wait_stream(main)
        for k in range(2):
            with torch.cuda.stream(streams[k]):
                tr.encode_bwd(k, 2)
        for s in streams[:2]:
            main.wait_stream(s)

    def adam():
        call("n2m_s0_adam_tables_keep", ptr(tr.table), ptr(tr.color_master), ptr(snap), ptr(tr.m_table), ptr(tr.v_table), tr.rows,
             ptr(tr.opt_state), tr.cfg.eps, stream())

    def serial():
        scatter()
        adam()

    def overlapped():
        # the scatters first, as a step would enqueue them; the block scheduler hands the sweep whatever the scatter grids leave free
        for s in streams:
            s.wait_stream(main)
        for k in range(2):
            with torch.cuda.stream(streams[k]):
                tr.encode_bwd(k, 2)
        with torch.cuda.stream(streams[2]):
            adam()
        for s in streams:
            main.wait_stream(s)

    def timed(fn):
        for _ in range(warmup):
            fn()
        a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        z.record()
        torch.cuda.synchronize()
        return a.elapsed_time(z) * 1e3 / iters

    res = {}
    for rep in range(3):             # alternate the four, three rounds: the spread of each is part of the answer
        for name, fn in (("scatter", scatter), ("adam", adam), ("serial", serial), ("overlapped", overlapped)):
            res.setdefault(name, []).append(round(timed(fn), 2))
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    props = torch.cuda.get_device_properties(0)
    return {"workload": workload, "device": props.name, "power_limit": power_limit(), "M": M, "rows": R, "found_inf": found_inf,
            "bytes": bytes_, "bound_us": {k: round(v / PEAK_BYTES * 1e6, 2) for k, v in bytes_.items()},
            "us": res, "us_median": med, "saved_us": round(med["serial"] - med["overlapped"], 2),
            "iters": iters, "warmup": warmup}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--workload", nargs="+", default=["lego_stage0_converged", "garden_stage0"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("optimizer_overlap_time.py: no CUDA device")
    torch.cuda.set_device(0)
    for w in args.workload:
        print(json.dumps(run(w, args.iters, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
