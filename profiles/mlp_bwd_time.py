"""Time the stand-alone MLP backward (n2m_s0_mlp_bwd, k_mlp_bwd) on bench.py's lego batch, against its bound from shapes.

    python profiles/mlp_bwd_time.py [--iters 200] [--warmup 20] [--shading {full,diffuse}]

Builds bench.py's lego_stage0_converged batch, runs the step's forward stages up to `dout`, then times the MLP backward alone with
CUDA events over many warm launches: the whole batch (one part) and each of the two ray-range parts bench.py's step uses.
--shading diffuse runs the forward and the backward without the specular net (the first part of stage-0 training, and stage 1
when it does not shade fully).  The bound is the larger of the MMA work of full shading as issued (padded shapes) at the
data-sheet dense fp16 rate and the bytes the kernel must move at the data-sheet HBM bandwidth (H100 SXM: 989 TFLOP/s, 3.35 TB/s).
Prints one JSON line.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# multiply-accumulates per sample of the wgmma GEMMs as issued (padded N x K of each layer)
MAC_FWD = 64 * 64 + 32 * 64 + 16 * 32 + 64 * 64 + 16 * 64 + 32 * 16 + 16 * 32            # forward recompute: 12,800
MAC_DGRAD = 32 * 16 + 32 * 16 + 16 * 32 + 64 * 16 + 64 * 64 + 64 * 32 + 64 * 64          # dgrad: 12,800
MAC_WGRAD = 64 * (16 + 16 + 32 + 32 + 16 + 64 + 64)                                       # wgrad (m64 rows): 15,360
BYTES = 128 + 16 + 128                                                                    # enc tile row in, dout in, denc tile row out
PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--shading", choices=("full", "diffuse"), default="full")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mlp_bwd_time.py: no CUDA device")
    import bench
    torch.cuda.set_device(0)
    workload = "lego_stage0_converged"
    tr = bench.make_trainer(workload)
    host, grid, bits = bench.make_batches(1, 1000, False, workload)
    b = {k: v.cuda() for k, v in host[0].items()}
    tr.set_occupancy(bits, grid)
    tr._fill_params(shading_full=args.shading == "full", gt_has_alpha=True)
    tr.slots[tr.cur].load(b["ro"], b["rd"], b["gt"], b["bg"], b["noises"], b.get("cnf"))
    tr.loss_acc.zero_()
    for s in ("march", "encode_fwd", "tv", "mlp_fwd", "composite_loss"):
        getattr(tr, s)()
    torch.cuda.synchronize()
    M = int(tr.counters[1].item())

    def time_launch(part, nparts):
        for _ in range(args.warmup):
            tr.mlp_bwd(part, nparts)
        a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            tr.mlp_bwd(part, nparts)
        z.record()
        torch.cuda.synchronize()
        return a.elapsed_time(z) * 1e3 / args.iters

    flop = 2.0 * (MAC_FWD + MAC_DGRAD + MAC_WGRAD) * M
    bound_us = max(flop / PEAK_FLOPS, BYTES * M / PEAK_BYTES) * 1e6
    whole = time_launch(0, 1)
    parts = [time_launch(p, 2) for p in range(2)]
    props = torch.cuda.get_device_properties(0)
    print(json.dumps({"device": props.name, "M": M, "us_whole": round(whole, 2), "us_part": [round(t, 2) for t in parts],
                      "bound_us": round(bound_us, 2), "bound_share_whole": round(bound_us / whole, 3),
                      "shading": args.shading, "iters": args.iters, "warmup": args.warmup}))


if __name__ == "__main__":
    main()
