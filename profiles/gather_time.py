"""Time the stage-0 forward hash-grid gather (n2m_s0_encode_fwd) on bench.py's batches, cold and warm L2, against the bytes it must move,
and show where it sits in the graph-replayed step.

    python profiles/gather_time.py [--iters 50] [--warmup 5] [--workload lego_stage0_converged garden_stage0] [--no-timeline]

For each workload: builds bench.py's batch (as profiles/grid_pass_time.py does), runs the march once, then times with CUDA events
  * the gather of the whole batch and of each of the two ray-range parts bench.py's step uses,
    "warm": back-to-back launches (the table slices the batch touches stay in L2 from one launch to the next);
    "cold": each launch preceded, on the same stream and outside the timed window, by a write of a 256 MB buffer (five times the
    H100's 50 MB L2), so the table sectors come from HBM.
  * bytes: the compulsory traffic -- march records in (16 B per sample), tile images out (16 KiB per tile), one read of every 32 B
    table sector the batch touches -- next to the table sectors the gather's warp loads ask of L2: for each level and corner, the
    distinct sectors each 32-lane load touches (an L1 hit is counted as a request), summed over the batch.  Both counted with torch from
    the batch's own records (positions restated as sample_of forms them; a sample within an ulp of a cell face may land in the
    neighbouring cell, which does not matter for a count).
  * with the timeline (profiles/step_timeline.py, one graph-replayed step with two parts and TV): when each part's gather and its
    k_mlp_fwd start and end, and which kernels of the step run at the same time as each gather.
Prints per workload one JSON line of kernel times and bytes with the device name and its power limit, and one of the timeline.
"""
import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from grid_pass_time import PEAK_BYTES, power_limit       # noqa: E402

GATHER = "k_s0_encode_fwd"


def table_sectors(tr, M):
    """Per level: distinct 32 B table sectors the batch touches, and the sectors its warp loads request (per load instruction,
    the distinct sectors among the active lanes)."""
    import numpy as np
    p, dev = tr.params, tr.recs.device
    recs = tr.recs[:M]
    n = recs[:, 3].contiguous().view(torch.int32).long()
    x = (tr.rays_o[n].double() + recs[:, :1].double() * tr.rays_d[n].double()).float().clamp(-p.bound, p.bound)
    if p.contract:
        mag = x.abs().amax(-1, keepdim=True)
        x = torch.where(mag > 1, x * ((2 - 1 / mag) / mag), x)
    u = (x + p.grid_bound) * p.inv_2gb
    act = ((u >= 0) & (u <= 1)).all(-1)
    j = torch.arange(M, device=dev)[act]
    u = u[act]
    offs = tr._offsets_host
    touched, requested = [], []
    for l in range(p.num_levels):
        rows = offs[l + 1] - offs[l]
        scale = float(np.float32(np.exp2(np.float32(l) * np.float32(p.S)) * np.float32(p.base_res) - np.float32(1)))
        res = int(np.ceil(scale)) + 1
        b = torch.floor(u * scale + 0.5).long()
        s1, stride, mult = res + 1, 1, []
        for _ in range(3):
            mult.append(stride if stride <= rows else 0)
            if stride <= rows:
                stride *= s1
        hashed = stride > rows
        sec = []
        for k in range(8):
            c = b + torch.tensor([k & 1, (k >> 1) & 1, (k >> 2) & 1], device=dev)
            if hashed:
                raw = (c[:, 0] ^ ((c[:, 1] * 2654435761) & 0xffffffff) ^ ((c[:, 2] * 805459861) & 0xffffffff)) & 0xffffffff
            else:
                raw = c[:, 0] * mult[0] + c[:, 1] * mult[1] + c[:, 2] * mult[2]
            sec.append((offs[l] + raw % rows) >> 2)                  # 8 B entries, 4 per sector
        sec = torch.stack(sec, 1)                                    # [active, 8]
        touched.append(int(torch.unique(sec).numel()))
        inst = (j // 32).unsqueeze(1) * 8 + torch.arange(8, device=dev)  # one warp load instruction per (warp, corner)
        requested.append(int(torch.unique(inst * (offs[-1] // 4 + 1) + sec).numel()))
    return touched, requested


def timed(tr, fn, iters, warmup, flush=None):
    for _ in range(warmup):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, z in ev:
        if flush is not None:
            flush.add_(1)
        a.record()
        fn()
        z.record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(z) * 1e3 for a, z in ev)
    return {"median_us": round(ts[len(ts) // 2], 2), "min_us": round(ts[0], 2), "max_us": round(ts[-1], 2)}


def kernel_timing(workload, iters, warmup):
    import bench
    tr = bench.make_trainer(workload)
    host, grid, bits = bench.make_batches(1, 1000, False, workload)
    b = {k: v.cuda() for k, v in host[0].items()}
    tr.set_occupancy(bits, grid)
    tr._fill_params(shading_full=True, gt_has_alpha=bench.WORKLOADS[workload]["alpha"])
    tr.slots[tr.cur].load(b["ro"], b["rd"], b["gt"], b["bg"], b["noises"], b.get("cnf"))
    tr.march()
    torch.cuda.synchronize()
    M = int(tr.counters[1].item())
    T = (M + 127) // 128
    flush = torch.zeros(64 << 20, dtype=torch.float32, device="cuda")       # 256 MB
    res = {}
    for name, fn in (("whole", lambda: tr.encode_fwd()), ("part0", lambda: tr.encode_fwd(0, 2)), ("part1", lambda: tr.encode_fwd(1, 2))):
        res[name] = {"warm": timed(tr, fn, iters, warmup), "cold": timed(tr, fn, iters, warmup, flush)}
    touched, requested = table_sectors(tr, M)
    nd = 5                                                               # dense levels 0-4, as the scatter groups them
    streamed = M * 16 + T * 128 * 128
    bytes_ = {"records_in": M * 16, "tiles_out": T * 128 * 128,
              "table_sectors_touched": sum(touched), "table_sectors_requested": sum(requested),
              "table_sectors_touched_hashed": sum(touched[nd:]), "table_sectors_requested_hashed": sum(requested[nd:]),
              "compulsory": streamed + 32 * sum(touched), "requested": streamed + 32 * sum(requested),
              "per_level_touched": touched, "per_level_requested": requested}
    w = res["whole"]
    res["bound_us_compulsory"] = round(bytes_["compulsory"] / PEAK_BYTES * 1e6, 2)
    res["bound_us_requested"] = round(bytes_["requested"] / PEAK_BYTES * 1e6, 2)
    res["gb_s_requested_cold"] = round(bytes_["requested"] / (w["cold"]["median_us"] * 1e-6) / 1e9, 1)
    return {"M": M, "tiles": T, "bytes": bytes_, **res}


def timeline(workload, warmup):
    import step_timeline
    with tempfile.TemporaryDirectory() as tmp:
        r = step_timeline.run(workload, warmup, tmp)
    ks = r["graph"]["kernels"]
    out = []
    for g in sorted((k for k in ks if k["name"].startswith(GATHER)), key=lambda k: k["start_us"]):
        fwd = next(k for k in ks if k["stream"] == g["stream"] and k["name"] == "k_mlp_fwd" and k["start_us"] >= g["end_us"])
        beside = sorted({k["name"] for k in ks if k is not g and k["start_us"] < g["end_us"] and k["end_us"] > g["start_us"]})
        out.append({"stream": g["stream"], "gather_start_us": g["start_us"], "gather_end_us": g["end_us"],
                    "gather_us": round(g["end_us"] - g["start_us"], 2), "mlp_fwd_start_us": fwd["start_us"],
                    "mlp_fwd_end_us": fwd["end_us"], "beside": beside})
    return {"parts": out, "step_span_us": r["graph"]["waits"]["step_span_us"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--workload", nargs="+", default=["lego_stage0_converged", "garden_stage0"])
    ap.add_argument("--no-timeline", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gather_time.py: no CUDA device")
    torch.cuda.set_device(0)
    for w in args.workload:
        r = {"workload": w, "device": torch.cuda.get_device_properties(0).name, "power_limit": power_limit(),
             **kernel_timing(w, args.iters, args.warmup)}
        print(json.dumps(r), flush=True)
        if not args.no_timeline:
            print(json.dumps({"workload": w, "timeline": timeline(w, 10)}), flush=True)


if __name__ == "__main__":
    main()
