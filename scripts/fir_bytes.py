#!/usr/bin/env python
"""Algorithmic HBM bytes per input sample of a FIR step as the library runs it, and the roofline fraction of a
measured step time.  bench.py's fir_bytes_model charges every single-level tail plan with a per-block k_fir_mac; on
plans with a folded tail (the default; describe() "l0_parts" > 2) there is none: the fused kernel reads lp filter rows and
lp - 1 FDL rows, and V_j in place of Y_j.  A channel sums lp = l0_parts_min .. l0_parts partitions in turn (the near
tier takes the rest of partitions la .. t_batch+la-2 of the periods it covers, la = the look-ahead), lp is their mean,
la + (t_batch - 1) / 2; the near tier reads P - la FDL rows and P - la filter rows per launch, the far tier costs what
bench.py says.  With the mid-window pass (describe() "pass_m" = m > 0) a channel sums la .. la - 1 + max(m, t_batch - m)
partitions, and the pass reads m FDL rows, t_batch - 1 filter rows and t_batch - m rows of V, which it writes back, once
per t_batch blocks.

    python scripts/fir_bytes.py bench_line.json        # a bench.py result line: its plan, its step time
    python scripts/fir_bytes.py --block 4096 --taps 131072 [--t 4] [--lookahead 3] [--pass-m 4] [--shared-ir] [--unfolded] [--step-us 186]
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
        T, la, m = int(plan["t_batch"]), int(plan.get("lookahead", 3)), int(plan.get("pass_m", 0))
        # in 8, spectrum to the FDL 16, lp - 1 FDL rows, lp filter rows, V_j, carry read + write, out
        lp = (lp_min + lp_max) / 2.0
        if m:
            # with the mid-window pass period t of a launch sums la + t partitions for t < m, la + t - m from t = m on
            lp = la + (m * (m - 1) / 2.0 + (T - m) * (T - m - 1) / 2.0) / T
        parts.pop("fir_mac")
        parts["fir_level0"] = 8 + 16 + 16.0 * (lp - 1) + 16.0 * lp * h + 16 + 8 + 8 + 8
        # bench.py charges the near tier the FDL rows from partition 3 and the filter rows from t_batch + 2.  Its launch
        # streams the FDL rows from partition la (the look-ahead, describe() "lookahead") and the filter rows from
        # lp_min on: X_la .. X_2 and H_{lp_min} .. H_{t_batch+1} more, once per launch of t_batch periods
        parts["fir_mac_batch"] += 16.0 * ((3 - la) + (T + 2 - lp_min) * h) / T
        if m:
            # the pass, once per T blocks: m FDL rows, the filter rows la .. la+T-2, T - m rows of V read and written
            parts["fir_mac_batch_pass"] = 16.0 * (m + (T - 1) * h + 2 * (T - m)) / T
        total = sum(parts.values())
    return total, parts


def plan_from_args(a):
    """The single-level plan fir_schedule() (dsp_b200/csrc/fir_plan.h) makes for 2048..8192-frame blocks at batch depth
    a.t and look-ahead a.lookahead (3 when absent; the full-wave plan uses 2 with one tier) with the default knobs (no far
    tier below 48 partitions, the stagger from 16 tail partitions on); tests/test_fir_schedule_cpu.py holds the two equal."""
    P = -(-a.taps // a.block)
    t_far = 8 if P >= 48 and 8 > a.t and 8 % a.t == 0 and P >= 2 * 8 + 2 + a.t else 0
    la = 3 if a.unfolded or t_far else int(getattr(a, "lookahead", None) or 3)
    stagger = 1 if not t_far and P - a.t - 2 >= 16 else 0
    m = int(getattr(a, "pass_m", None) or 0) if stagger and la == 2 and not a.unfolded else 0
    return {"levels": [{"B": a.block, "P": P}], "tail_pf": 2, "t_batch": a.t, "t_far": t_far, "far_e": a.t if t_far else 0,
            "stagger": stagger, "merge": 0, "pipe": 0, "pipe_pf": 0,
            "l0_parts": 2 if a.unfolded else a.t + la - 1, "l0_parts_min": 2 if a.unfolded else la, "lookahead": la,
            "pass_m": m, "l0_parts_steady": la - 1 + max(m, a.t - m) if m else (2 if a.unfolded else a.t + la - 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("bench_json", nargs="?", help="a bench.py result line (file); its roofline.plan and avg_step_us are used")
    ap.add_argument("--block", type=int, default=4096)
    ap.add_argument("--taps", type=int, default=131072)
    ap.add_argument("--channels", type=int, default=256)
    ap.add_argument("--t", type=int, default=4, help="batch depth (DSP_B200_FIR_T)")
    ap.add_argument("--lookahead", type=int, default=3, choices=[2, 3], help="look-ahead of the folded near tier")
    ap.add_argument("--pass-m", type=int, default=0, help="mid-window pass depth (DSP_B200_FIR_PASS; staggered plans at look-ahead 2)")
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
    out = {"plan": {k: plan[k] for k in ("levels", "t_batch", "t_far", "stagger", "l0_parts", "l0_parts_min", "l0_parts_steady", "lookahead",
                                         "pass_m") if k in plan},
           "bytes_per_sample": total, "bytes_per_sample_by_kernel": parts, "bytes_per_step": total * C * B}
    if step_us:
        gbs = total * C * B / (step_us * 1e-6) / 1e9
        out.update(step_us=step_us, achieved_GBs=gbs, peak_GBs=a.peak_gbs, frac=gbs / a.peak_gbs)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
