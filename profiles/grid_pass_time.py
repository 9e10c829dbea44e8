"""Time the per-sample hash-grid passes of the stage-0 step (gather, TV, scatter) on bench.py's batches, against the bytes they must move.

    python profiles/grid_pass_time.py [--iters 100] [--warmup 10] [--workload lego_stage0_converged garden_stage0]

For each workload: builds bench.py's batch, runs the step's forward stages and the MLP backward once (so that `denc` holds real
gradients), then times with CUDA events over many warm launches
  * encode_fwd (n2m_s0_encode_fwd), tv (n2m_s0_tv + the random-point fallback launch) and encode_bwd (n2m_s0_encode_bwd), each for
    the whole batch and for each of the two ray-range parts bench.py's step uses;
  * "concurrent": the passes as the step overlaps them -- the two parts' scatters on their own streams, TV on a third and the
    deferred zeroing of the other gradient table (97.6 MB memset at the default config) on a fourth -- fork to join.
The bytes each pass must move are computed from the shapes: the streamed per-sample data (march records, tile images) plus one pass
over the 32 B sectors of the tables the batch actually touches (a sector of the gradient table is filled and written back once, a
sector of the parameter table is read once).  The touched sectors are counted from the gradient table one scatter leaves behind.
The scatter's RED counts per level ("reds") are computed with torch from the batch's own march records: the 8 corner contributions
of every sample inside the grid, the REDs the same-cell run merge of a warp leaves, and the distinct gradient rows per 32-sample warp
and per 128-sample tile (what a scatter that sums duplicate rows per warp / per tile would issue).
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


def red_counts(tr, M):
    """Per level: corner contributions, REDs left by the warp's same-cell run merge (csrc/stage0.cu encode_bwd_visit), distinct
    gradient rows per warp and per tile, over the whole batch (positions restated from the records as sample_of / corners_of form
    them; a sample within an ulp of a cell face may land in the neighbouring cell, which does not matter for a count)."""
    import numpy as np
    p, dev = tr.params, tr.recs.device
    recs = tr.recs[:M]
    n = recs[:, 3].contiguous().view(torch.int32).long()
    x = (tr.rays_o[n].double() + recs[:, :1].double() * tr.rays_d[n].double()).float().clamp(-p.bound, p.bound)
    if p.contract:
        mag = x.abs().amax(-1, keepdim=True)
        x = torch.where(mag > 1, x * ((2 - 1 / mag) / mag), x)
    u = (x + p.grid_bound) * p.inv_2gb
    T = (M + 127) // 128
    Mt = T * 128
    act = torch.zeros(Mt, dtype=torch.bool, device=dev)
    act[:M] = ((u >= 0) & (u <= 1)).all(-1)
    u = torch.nn.functional.pad(u, (0, 0, 0, Mt - M), value=0.5)
    offs = tr._offsets_host
    out = {"contrib": [], "reds_run_merge": [], "distinct_warp": [], "distinct_tile": []}
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
        corner = []
        for k in range(8):
            c = b + torch.tensor([k & 1, (k >> 1) & 1, (k >> 2) & 1], device=dev)
            if hashed:
                raw = (c[:, 0] ^ ((c[:, 1] * 2654435761) & 0xffffffff) ^ ((c[:, 2] * 805459861) & 0xffffffff)) & 0xffffffff
            else:
                raw = c[:, 0] * mult[0] + c[:, 1] * mult[1] + c[:, 2] * mult[2]
            corner.append(raw % rows)
        corner = torch.stack(corner, 1)
        key = torch.where(act, b[:, 0] | (b[:, 1] << 10) | (b[:, 2] << 20), torch.full_like(b[:, 0], -1)).view(-1, 32)
        heads = torch.ones_like(key, dtype=torch.bool)
        heads[:, 1:] = key[:, 1:] != key[:, :-1]
        tails = torch.ones_like(heads)
        tails[:, :-1] = heads[:, 1:]
        merge = ((heads.sum(1) <= 20) & (res < 1023)).unsqueeze(1)
        a32 = act.view(-1, 32)
        issue = torch.where(merge, tails & a32, a32)
        j = torch.arange(Mt, device=dev).unsqueeze(1).expand(-1, 8)[act]
        rr = corner[act]

        def distinct(width):
            return int(torch.unique((j // width) * rows + rr).numel())
        out["contrib"].append(int(act.sum().item()) * 8)
        out["reds_run_merge"].append(int(issue.sum().item()) * 8)
        out["distinct_warp"].append(distinct(32))
        out["distinct_tile"].append(distinct(128))
    out["per_sample"] = {k: round(sum(v) / max(M, 1), 2) for k, v in out.items()}
    return out


def run(workload, iters, warmup):
    import bench
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

    # sectors of the tables this batch touches: rows the scatter gave a non-zero gradient
    gt = tr.gtables[tr.parity]
    gt.zero_()
    tr.encode_bwd()
    torch.cuda.synchronize()
    touched = (gt != 0).any(1)
    R = touched.numel()
    pad = (-R) % 4
    t4 = torch.nn.functional.pad(touched, (0, pad)).view(-1, 4)
    g_sectors = int(t4.view(-1, 2).any(1).sum().item())            # float4 rows: 2 per 32 B sector
    t_sectors = int(t4.any(1).sum().item())                         # 8 B rows: 4 per 32 B sector
    rows_touched = int(touched.sum().item())

    tile_row = 128                                                  # one sample's 64 fp16 columns
    bytes_ = {
        # records in, tile rows out, parameter-table sectors read once
        "encode_fwd": M * (16 + tile_row) + t_sectors * 32,
        # records in, the 7 gradient chunks of a tile row in, gradient-table sectors filled + written back once
        "encode_bwd": M * (16 + 7 * 16) + g_sectors * 64,
        # records in, parameter-table sectors read once, gradient-table sectors filled + written back once
        "tv": M * 16 + t_sectors * 32 + g_sectors * 64,
    }

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
    for name in ("encode_fwd", "tv", "encode_bwd"):
        fn = getattr(tr, name)
        whole = timed(fn)
        parts = [timed(lambda p=p: fn(p, 2)) for p in range(2)] if name != "tv" else None
        res[name] = {"us_whole": round(whole, 2), "us_part": [round(t, 2) for t in parts] if parts else None,
                     "bytes": bytes_[name], "gb_s_whole": round(bytes_[name] / (whole * 1e-6) / 1e9, 1),
                     "bound_us": round(bytes_[name] / PEAK_BYTES * 1e6, 2)}

    # the step's overlap: both parts' scatters, TV and the zeroing of the other gradient table, each on its own stream
    main = torch.cuda.current_stream()
    streams = [torch.cuda.Stream() for _ in range(4)]
    other = tr.gtables[tr.parity ^ 1]

    def concurrent():
        for s in streams:
            s.wait_stream(main)
        with torch.cuda.stream(streams[0]):
            tr.encode_bwd(0, 2)
        with torch.cuda.stream(streams[1]):
            tr.encode_bwd(1, 2)
        with torch.cuda.stream(streams[2]):
            tr.tv()
        with torch.cuda.stream(streams[3]):
            other.zero_()
        for s in streams:
            main.wait_stream(s)

    def zero_only():
        other.zero_()

    res["concurrent"] = {"us": round(timed(concurrent), 2), "what": "encode_bwd part 0 || part 1 || tv || zero other gtable"}
    res["zero_gtable"] = {"us": round(timed(zero_only), 2), "bytes": other.numel() * 4}
    props = torch.cuda.get_device_properties(0)
    return {"workload": workload, "device": props.name, "power_limit": power_limit(), "M": M, "rows": R,
            "rows_touched": rows_touched, "gtable_sectors_touched": g_sectors, "table_sectors_touched": t_sectors,
            **res, "reds": red_counts(tr, M), "iters": iters, "warmup": warmup}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--workload", nargs="+", default=["lego_stage0_converged", "garden_stage0"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("grid_pass_time.py: no CUDA device")
    torch.cuda.set_device(0)
    for w in args.workload:
        print(json.dumps(run(w, args.iters, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
