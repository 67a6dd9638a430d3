#!/usr/bin/env python
"""Lane margins (lmpc_set_lane_margins): what planning through the derived per-controller rows costs, and whether a controller
that plans inside a tightened lane -- fixed or adapted lap by lap -- leaves the real lane less often late in learning, and at what
lap-time cost.

Leg 1, cost: benchmarks/rollout_mc.run (PID lap, seeding, `laps` LMPC laps), independent and pooled, in alternating rounds in the
same process, with
  none   no lane-margin table (the uniform QP kernel);
  zero   an all-mode-1 table at margin0 = 0: every QP reads its controller's derived row through the SETS kernel.
Per round: ms of the LMPC laps and controller steps/s (device events).  configs[3]'s horizon (N = 12) is one at which the SETS
kernel equals the uniform one bit for bit, so both arms must drive the same closed loop: books, end states, health and solver
reports are asserted identical in the run.
Leg 2, study: the circuit of configs[3], `study-laps` LMPC laps with lap reports, independent mode, on the rollout_mc handle (the
setting of benchmarks/lane_rules.py leg 2).  Margin arms: none; fixed 0.02; fixed 0.05; adaptive (margin0 0, step_up 0.01,
step_down 0.0025, margin_max 0.1), crossed with lane rules off (mode 0) and on (mode 1, lane_tol 0) and with measurement sigma
{0, 0.01} on all six channels (clip 5 sigma): 16 cells in one batch, cell = controller mod 16, noise streams controller // 16
(common random numbers, so the arms pair).  Per cell and lap: mean steps, the share of controllers whose plant state left the
lane (reports, judged against the given lane), unsolved QPs; per cell the final margins (min / mean / max).

  python benchmarks/lane_margins.py [--rounds 3 --batch 8192 --laps 3] [--legs 1,2] [--study-batch 4096 --study-laps 40]
                                    [--out FILE] [--table FILE]
Prints one JSON line per leg (card name and power limit read in the same run); --out appends them to FILE as well, --table writes
leg 2 as a readable table."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "benchmarks")):
    if p not in sys.path:
        sys.path.insert(0, p)
from racinglmpc_b200.reference_params import LaneMarginParams, LaneRuleParams, MeasurementParams   # noqa: E402
from param_sweep import card                                                                      # noqa: E402
from model_sweep import SAME, _spread                                                             # noqa: E402
import rollout_mc                                                                                 # noqa: E402

ARMS = (("none", LaneMarginParams(0)), ("fixed0.02", LaneMarginParams(1, 0.02, 0.02)), ("fixed0.05", LaneMarginParams(1, 0.05, 0.05)),
        ("adaptive", LaneMarginParams(2, 0.0, 0.1, 0.01, 0.0025)))
RULES = (("rules_off", LaneRuleParams(0, 0.0)), ("rules_on", LaneRuleParams(1, 0.0)))
SIGMAS = (0.0, 0.01)


def leg_cost(rounds, batch, laps, dev):
    arms = {"none": {}, "zero": dict(lane_margin_sets=([LaneMarginParams(1, 0.0, 0.0)], np.zeros(batch, np.int32)))}
    out = {"benchmark": "lane_margins leg 1: closed loop without a lane-margin table vs an all-mode-1 table at margin0 = 0",
           **card(dev), "batch": batch, "laps": laps, "rounds": rounds}
    for mode in ("independent", "pooled"):
        ms, rate, first = {n: [] for n in arms}, {n: [] for n in arms}, {}
        for _ in range(rounds):
            for name, kw in arms.items():
                fin = {}
                r = rollout_mc.run(batch=batch, laps=laps, mode=mode, local=dev, final=fin, books=fin, **kw)
                ms[name].append(r["ms_total"])
                rate[name].append(r["controller_steps_per_s"])
                first.setdefault(name, fin)
        fa, fb = first["none"], first["zero"]
        for k in SAME:
            assert np.array_equal(fa[k], fb[k]), k
        assert np.array_equal(fb["lane_margins"], np.zeros(batch))
        a, b = np.array(ms["none"]), np.array(ms["zero"])
        d = 100.0 * (b / a - 1.0)
        out[mode] = {"ms_total": {"none": a.tolist(), "zero": b.tolist()},
                     "controller_steps_per_s": {"none": rate["none"], "zero": rate["zero"]},
                     "zero_over_none_ms_pct_rounds": d.tolist(),
                     "zero_over_none_ms_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
                     "none_round_spread_pct": _spread(a), "zero_round_spread_pct": _spread(b)}
    out["identical"] = list(SAME)
    return out


def study_tables(batch, laps):
    K = len(ARMS) * len(RULES) * len(SIGMAS)
    b = np.arange(batch)
    cell = b % K
    arm, rule, sig = cell % len(ARMS), (cell // len(ARMS)) % len(RULES), cell // (len(ARMS) * len(RULES))
    meas = [MeasurementParams((s,) * 6, (5 * s,) * 6) for s in SIGMAS]
    kw = dict(lane_margin_sets=([r for _, r in ARMS], arm), lane_rule_sets=([r for _, r in RULES], rule),
              measurement_sets=(meas, sig), noise_streams=b // K, lap_reports=laps)
    return K, cell, arm, rule, sig, kw


def leg_study(batch, laps, dev):
    K, cell, arm, rule, sig, kw = study_tables(batch, laps)
    bk = {}
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, books=bk, **kw)
    reps, m_end = bk["lap_reports"], bk["lane_margins"]
    cells = []
    for k in range(K):
        sel = cell == k
        rows = []
        for r in range(laps):
            m = sel & (reps["n"] > r)
            n = int(m.sum())
            rows.append({"lap": r + 1, "controllers": n, "steps_mean": float(reps["steps"][m, r].mean()) if n else 0.0,
                         "violating_share": float((reps["viol_steps"][m, r] > 0).mean()) if n else 0.0,
                         "unsolved": int(reps["unsolved"][m, r].sum())})
        a, u, s = int(arm[sel][0]), int(rule[sel][0]), int(sig[sel][0])
        cells.append({"arm": ARMS[a][0], "rules": RULES[u][0], "meas_sigma": SIGMAS[s], "controllers": int(sel.sum()),
                      "margin_final": {"min": float(m_end[sel].min()), "mean": float(m_end[sel].mean()),
                                       "max": float(m_end[sel].max())},
                      "per_lap": rows})
    keep = ("closed_loop_steps", "ms_total", "controller_steps_per_s", "unsolved_steps_rank0", "instances_with_flags_rank0",
            "flag_bits_rank0", "per_lane_margin_rank0", "lane_margin_final_rank0")
    return {"benchmark": "lane_margins leg 2: no margin / fixed 0.02 / fixed 0.05 / adaptive x lane rules off / on (lane_tol 0) x "
                         "measurement sigma {0, 0.01}, common noise streams (controller // %d), independent mode" % K,
            **card(dev), "batch": batch, "laps": laps, "controllers_per_cell": batch // K, "cells": cells,
            **{k: out[k] for k in keep}}


def summary(study):
    """Leg 2 as a table: per cell, mean steps / violating share (%) / unsolved QPs at a few laps, and the final mean margin."""
    laps = study["laps"]
    pick = sorted({r for r in (1, 5, 10, 20, 30, 40) if r <= laps} | {laps})
    lines = ["%s, %s, power limit %s W: %d controllers per cell" % (study["benchmark"], study["gpu"], study["power_limit_w"],
                                                                    study["controllers_per_cell"]),
             "arm        rules      sigma  m_end  " + "  ".join("lap%-2d steps viol%% unsolv" % r for r in pick)]
    for c in study["cells"]:
        row = ["%-10s %-10s %5.2f %6.4f " % (c["arm"], c["rules"], c["meas_sigma"], c["margin_final"]["mean"])]
        for r in pick:
            e = c["per_lap"][r - 1]
            row.append("%5d %7.1f %5.1f %6d" % (r, e["steps_mean"], 100.0 * e["violating_share"], e["unsolved"]))
        lines.append("  ".join(row))
    return "\n".join(lines) + "\n"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of leg 1")
    ap.add_argument("--batch", type=int, default=8192, help="controllers of leg 1")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps of leg 1")
    ap.add_argument("--study-batch", type=int, default=4096, help="controllers of leg 2 (a multiple of 16)")
    ap.add_argument("--study-laps", type=int, default=40, help="LMPC laps of leg 2")
    ap.add_argument("--legs", default="1,2", help="legs to run")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    ap.add_argument("--table", default="", help="write leg 2's readable table to this file")
    args = ap.parse_args()
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    legs = args.legs.split(",")
    for leg, fn in (("1", lambda: leg_cost(args.rounds, args.batch, args.laps, dev)),
                    ("2", lambda: leg_study(args.study_batch, args.study_laps, dev))):
        if leg not in legs:
            continue
        r = fn()
        print(json.dumps(r), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(r) + "\n")
        if leg == "2" and args.table:
            with open(args.table, "w") as f:
                f.write(summary(r))


if __name__ == "__main__":
    main()
