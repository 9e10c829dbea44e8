"""CPU: profiles/step_timeline.py finds the two parts' chains in a step's kernel list, with the composite kernel under its template
name (k_s0_composite_loss<ADAPTIVE>) as the profiler reports it."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import step_timeline as T  # noqa: E402


def k(name, stream, start, end):
    return {"name": name, "stream": stream, "start_us": start, "end_us": end, "grid": None, "block": None}


def test_waits_of_a_two_part_step():
    ks = [k("k_s0_encode_bwd<false, true>", 3, 1.0, 50.0),
          k("k_s0_encode_fwd<false>", 1, 1.0, 40.0), k("k_s0_encode_fwd<false>", 2, 30.0, 60.0),
          k("k_mlp_fwd", 1, 41.0, 70.0), k("k_mlp_fwd", 2, 70.5, 80.0),
          k("k_s0_composite_loss<false>", 1, 70.2, 90.0), k("k_s0_composite_loss<true>", 2, 80.2, 95.0),
          k("k_mlp_bwd", 1, 90.5, 120.0), k("k_mlp_bwd", 2, 121.0, 150.0),
          k("k_s0_scatter_walkers", 1, 151.0, 300.0), k("k_s0_scatter_walkers", 2, 150.5, 310.0)]
    w = T.waits(sorted(ks, key=lambda x: x["start_us"]))
    assert w["part0_mlp_bwd"] == {"composite_end_us": 90.0, "start_us": 90.5, "gap_us": 0.5, "tv_end_us": 50.0}
    assert w["part1_mlp_bwd"]["gap_us"] == 26.0 and w["part1_mlp_bwd"]["part0_mlp_bwd_end_us"] == 120.0
    assert w["part0_scatter"]["gap_us"] == 31.0 and w["part0_scatter"]["part1_mlp_bwd_end_us"] == 150.0
    assert w["scatters_end_us"] == 310.0 and w["step_span_us"] == 310.0
