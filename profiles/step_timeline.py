"""Kernel timeline of one stage-0 train step: when each kernel of bench.py's step starts and ends, and on which stream.

    python profiles/step_timeline.py [--warmup 10] [--workload lego_stage0_converged garden_stage0] [--trace-dir DIR]

For each workload: builds bench.py's batches and trainer (bench.make_batches, bench.make_trainer) with two ray-range parts and the
TV pass on, as bench.py runs them, warms up with graph-replayed and eager steps, then profiles one eager step and, in a profiler run
of its own, one graph-replayed step (torch.profiler, CUDA activities).  Each step is bench.py's: the next batch's march is prefetched
on a side stream and the other gradient table is zeroed underneath.  Prints, per step, every kernel with its start and end in us
from the step's first kernel, its stream and its launch shape, and then when each part's backward could start and what it waited for.
A part is the chain encode_fwd -> mlp_fwd -> composite -> mlp_bwd -> scatter on one stream (part 0 is launched first):
  * part 0: the end of its composite kernel (k_s0_composite_loss, the last of its forward) -> the start of its k_mlp_bwd, beside
    the end of the TV pass (k_s0_encode_bwd<false, true>);
  * part 1: the same gap, beside the end of part 0's k_mlp_bwd and of part 0's scatter (k_s0_encode_bwd<true, false> or
    k_s0_scatter_walkers);
  * part 0's scatter: the end of its k_mlp_bwd -> its start, beside the end of part 1's k_mlp_bwd.
k_mlp_bwd is one CTA per SM that holds the whole SM (384 threads x 160 registers, 217 KB of shared memory), so it starts on an SM
only once no other CTA runs there, and while it runs nothing else fits beside it.
Prints the device name and its power limit, and one JSON line per workload; with --trace-dir the Chrome traces are kept there.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CHAIN = ["k_s0_encode_fwd<false>", "k_mlp_fwd", "k_s0_composite_loss", "k_mlp_bwd", "scatter"]
SCATTERS = ("k_s0_encode_bwd<true, false>", "k_s0_scatter_walkers")       # per-slot and whole-SM form
TV = "k_s0_encode_bwd<false, true>"


def stage(name):
    if name.startswith("k_s0_composite_loss"):          # k_s0_composite_loss<ADAPTIVE>
        return "k_s0_composite_loss"
    return "scatter" if name in SCATTERS else name


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=20)
        return r.stdout.strip() or None
    except Exception:      # noqa: BLE001
        return None


def short_name(name):
    """'void n2m::(anonymous namespace)::k_s0_encode_bwd<true, false>(n2m_s0_params, ...)' -> 'k_s0_encode_bwd<true, false>'"""
    name = re.sub(r"^void ", "", name)
    depth, cut = 0, len(name)
    for i, ch in enumerate(name):            # the argument list: the first '(' outside template brackets, after the namespaces
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0 and not name.startswith("(anonymous", i):
            cut = i
            break
    return re.sub(r"^(?:\w+::|\(anonymous namespace\)::)+", "", name[:cut])


def kernels_of(trace_path):
    with open(trace_path) as f:
        ks = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    t0 = min(e["ts"] for e in ks)
    out = [{"name": short_name(e["name"]), "stream": e["args"].get("stream"), "start_us": round(e["ts"] - t0, 2),
            "end_us": round(e["ts"] + e["dur"] - t0, 2), "grid": e["args"].get("grid"), "block": e["args"].get("block")} for e in ks]
    return sorted(out, key=lambda k: k["start_us"])


def waits(ks):
    by_stream = {}
    for k in ks:
        if stage(k["name"]) in CHAIN:
            by_stream.setdefault(k["stream"], []).append(k)
    parts = sorted((v for v in by_stream.values() if [stage(k["name"]) for k in v] == CHAIN), key=lambda c: c[0]["start_us"])
    assert len(parts) == 2, {s: [k["name"] for k in v] for s, v in by_stream.items()}
    comp, bwd, sc = 2, 3, 4
    tv_end = max((k["end_us"] for k in ks if k["name"] == TV), default=None)

    def gap(a, b):
        return round(b["start_us"] - a["end_us"], 2)
    return {
        "part0_mlp_bwd": {"composite_end_us": parts[0][comp]["end_us"], "start_us": parts[0][bwd]["start_us"],
                          "gap_us": gap(parts[0][comp], parts[0][bwd]), "tv_end_us": tv_end},
        "part1_mlp_bwd": {"composite_end_us": parts[1][comp]["end_us"], "start_us": parts[1][bwd]["start_us"],
                          "gap_us": gap(parts[1][comp], parts[1][bwd]), "part0_mlp_bwd_end_us": parts[0][bwd]["end_us"],
                          "part0_scatter_end_us": parts[0][sc]["end_us"]},
        "part0_scatter": {"mlp_bwd_end_us": parts[0][bwd]["end_us"], "start_us": parts[0][sc]["start_us"],
                          "gap_us": gap(parts[0][bwd], parts[0][sc]), "part1_mlp_bwd_end_us": parts[1][bwd]["end_us"]},
        "scatters_end_us": max(p[sc]["end_us"] for p in parts),
        "step_span_us": max(k["end_us"] for k in ks),
    }


def run(workload, warmup, trace_dir):
    import bench
    from torch.profiler import ProfilerActivity, profile
    tr = bench.make_trainer(workload)
    tr.nparts = 2
    assert tr.cfg.lambda_tv > 0
    n_batches = 8
    host, grid, bits = bench.make_batches(n_batches, 1000, True, workload)
    dev = [{k: v.cuda(non_blocking=True) for k, v in b.items()} for b in host]
    tr.set_occupancy(bits, grid)

    def tup(b):
        return (b["ro"], b["rd"], b["gt"], b["bg"], b["noises"]) + ((b["cnf"],) if "cnf" in b else ())

    it = [0]

    def one_step(use_graph):
        b = dev[it[0] % n_batches]
        tr.step(b["ro"], b["rd"], b["gt"], b["bg"], b["noises"], shading="full", use_graph=use_graph,
                next_batch=tup(dev[(it[0] + 1) % n_batches]), cam_near_far=b.get("cnf"))
        it[0] += 1

    for i in range(warmup):               # every (slot, parity) graph variant, and the eager launches' first-call costs
        one_step(use_graph=i % 4 < 2)
    torch.cuda.synchronize()
    out = {"workload": workload, "device": torch.cuda.get_device_properties(0).name, "power_limit": power_limit(),
           "nparts": tr.nparts, "lambda_tv": tr.cfg.lambda_tv}
    for mode in ("eager", "graph"):
        path = os.path.join(trace_dir, f"step_timeline_{workload}_{mode}.pt.trace.json")
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            one_step(use_graph=mode == "graph")
            torch.cuda.synchronize()
        prof.export_chrome_trace(path)
        ks = kernels_of(path)
        out[mode] = {"waits": waits(ks), "kernels": ks}
    return out


def report(r):
    print(f"== {r['workload']}  {r['device']}  power limit {r['power_limit']}")
    for mode in ("eager", "graph"):
        print(f"-- {mode} step: kernel, stream, start_us, end_us, grid x block")
        for k in r[mode]["kernels"]:
            print(f"   {k['name'][:40]:<40} {str(k['stream']):>4} {k['start_us']:>9.2f} {k['end_us']:>9.2f}  {k['grid']} x {k['block']}")
        w = r[mode]["waits"]
        a, b, c = w["part0_mlp_bwd"], w["part1_mlp_bwd"], w["part0_scatter"]
        print(f"   part 0 k_mlp_bwd: composite ends {a['composite_end_us']:.2f}, starts {a['start_us']:.2f} (gap {a['gap_us']:.2f} us); "
              f"TV ends {a['tv_end_us']}")
        print(f"   part 1 k_mlp_bwd: composite ends {b['composite_end_us']:.2f}, starts {b['start_us']:.2f} (gap {b['gap_us']:.2f} us); "
              f"part 0's k_mlp_bwd ends {b['part0_mlp_bwd_end_us']:.2f}, part 0's scatter ends {b['part0_scatter_end_us']:.2f}")
        print(f"   part 0 scatter:   its k_mlp_bwd ends {c['mlp_bwd_end_us']:.2f}, starts {c['start_us']:.2f} (gap {c['gap_us']:.2f} us); "
              f"part 1's k_mlp_bwd ends {c['part1_mlp_bwd_end_us']:.2f}")
    print(json.dumps({k: ({"waits": v["waits"]} if k in ("eager", "graph") else v) for k, v in r.items()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--workload", nargs="+", default=["lego_stage0_converged", "garden_stage0"])
    ap.add_argument("--trace-dir", default=None, help="keep the Chrome traces here (default: a temporary directory)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_timeline.py: no CUDA device")
    torch.cuda.set_device(0)
    with tempfile.TemporaryDirectory() as tmp:
        trace_dir = args.trace_dir or tmp
        os.makedirs(trace_dir, exist_ok=True)
        for w in args.workload:
            report(run(w, args.warmup, trace_dir))


if __name__ == "__main__":
    main()
