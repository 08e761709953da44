#!/usr/bin/env python
"""Algorithmic HBM bytes per input sample of a FIR step as the library runs it, and the roofline fraction of a
measured step time.  bench.py's fir_bytes_model charges every single-level tail plan with a per-block k_fir_mac; on
plans with a folded tail (the default; describe() "l0_parts" > 2) there is none: the fused kernel reads lp filter rows and
lp - 1 FDL rows, and V_j in place of Y_j.  A channel sums lp = l0_parts_min .. l0_parts partitions in turn (the near
tier takes the rest of partitions 3 .. t_batch+1 of the periods it covers), lp is their mean; the near tier reads
l0_parts - l0_parts_min filter rows more than bench.py says, the far tier costs what bench.py says.

    python scripts/fir_bytes.py bench_line.json        # a bench.py result line: its plan, its step time
    python scripts/fir_bytes.py --block 4096 --taps 131072 [--t 4] [--shared-ir] [--unfolded] [--step-us 186]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import HBM_PEAK_GBS, fir_bytes_model   # noqa: E402


def folded_bytes_model(plan, h):
    """-> (bytes per sample, {kernel: bytes per sample}) for a plan dict as describe() reports it."""
    total, parts = fir_bytes_model(plan, 0, 0, h)
    lp_max = int(plan.get("l0_parts", 2))
    lp_min = int(plan.get("l0_parts_min", lp_max))
    if lp_max > 2 and "fir_mac" in parts:
        # in 8, spectrum to the FDL 16, lp - 1 FDL rows, lp filter rows, V_j, carry read + write, out
        lp = (lp_min + lp_max) / 2.0
        parts.pop("fir_mac")
        parts["fir_level0"] = 8 + 16 + 16.0 * (lp - 1) + 16.0 * lp * h + 16 + 8 + 8 + 8
        # the near tier's filter rows H_3 .. H_{t_batch+1}, once per launch of t_batch periods
        parts["fir_mac_batch"] += 16.0 * (lp_max - lp_min) * h / int(plan["t_batch"])
        total = sum(parts.values())
    return total, parts


def plan_from_args(a):
    """The single-level plan FirOp::plan() makes for 2048..8192-frame blocks with the default knobs (no far tier below
    48 partitions, the stagger from 16 tail partitions on)."""
    P = -(-a.taps // a.block)
    t_far = 8 if P >= 48 and 8 > a.t and 8 % a.t == 0 and P >= 2 * 8 + 2 + a.t else 0
    return {"levels": [{"B": a.block, "P": P}], "tail_pf": 2, "t_batch": a.t, "t_far": t_far, "far_e": a.t if t_far else 0,
            "stagger": 1 if not t_far and P - a.t - 2 >= 16 else 0, "merge": 0, "pipe": 0, "pipe_pf": 0,
            "l0_parts": 2 if a.unfolded else a.t + 2, "l0_parts_min": 2 if a.unfolded else 3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("bench_json", nargs="?", help="a bench.py result line (file); its roofline.plan and avg_step_us are used")
    ap.add_argument("--block", type=int, default=4096)
    ap.add_argument("--taps", type=int, default=131072)
    ap.add_argument("--channels", type=int, default=256)
    ap.add_argument("--t", type=int, default=4, help="batch depth (DSP_B200_FIR_T)")
    ap.add_argument("--shared-ir", action="store_true")
    ap.add_argument("--unfolded", action="store_true", help="the per-block MAC form (DSP_B200_FIR_FOLD=0)")
    ap.add_argument("--step-us", type=float, help="measured step time")
    ap.add_argument("--peak-gbs", type=float, default=HBM_PEAK_GBS)
    a = ap.parse_args()
    h = 0 if a.shared_ir else 1
    C, step_us = a.channels, a.step_us
    if a.bench_json:
        line = json.load(open(a.bench_json))
        plan = line["roofline"]["plan"]
        C = plan["n_sel"]
        step_us = step_us or line["roofline"]["avg_step_us"]
    else:
        plan = plan_from_args(a)
    B = plan["levels"][-1]["B"]
    total, parts = folded_bytes_model(plan, h)
    out = {"plan": {k: plan[k] for k in ("levels", "t_batch", "t_far", "stagger", "l0_parts", "l0_parts_min") if k in plan},
           "bytes_per_sample": total, "bytes_per_sample_by_kernel": parts, "bytes_per_step": total * C * B}
    if step_us:
        gbs = total * C * B / (step_us * 1e-6) / 1e9
        out.update(step_us=step_us, achieved_GBs=gbs, peak_GBs=a.peak_gbs, frac=gbs / a.peak_gbs)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
