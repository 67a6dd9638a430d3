#!/usr/bin/env python
"""Lane-safe safe sets (lmpc_set_lane_rules): what judging every filed lap costs, and whether ranking lane-unsafe laps behind the
others lowers the late-learning lane violations and what it costs in lap time.

Leg 1, cost: benchmarks/rollout_mc.run (PID lap, seeding, `laps` LMPC laps, lap reports on), independent and pooled, in
alternating rounds in the same process, with
  none   no lane-rule table;
  judge  an all-mode-1 table with lane_tol = 1e300: every lap is judged, none is unsafe, so the closed loop is the same.
Per round: ms of the LMPC laps and controller steps/s (device events).  Both arms must drive the same closed loop: books, end
states, health, solver reports and lap reports are asserted identical.
Leg 2, study: the circuit of configs[3], `study-laps` LMPC laps with lap reports, independent mode, on the rollout_mc handle.
Arms: reference ranking (mode 0), mode 1 with lane_tol 0, mode 1 with lane_tol 0.02, crossed with measurement sigma {0, 0.01} on
all six channels (clip 5 sigma): 6 cells in one batch, cell = controller mod 6, noise streams controller // 6 (common random
numbers, so the arms pair).  Per cell and lap: mean steps, the share of controllers whose plant state left the lane (reports),
the share whose lap was judged lane-unsafe (report bit), unsolved QPs.
Leg parent, against the parent build (--parent-root: a checkout of the previous commit with its library built): bench.py --config
1, 2 and 3 with --dump-outputs, alternating this tree and the parent's; every dumped array of both trees is compared bit for bit.

  python benchmarks/lane_rules.py [--rounds 5 --batch 8192 --laps 3] [--legs 1,2,parent] [--parent-root DIR]
                                  [--study-batch 1536 --study-laps 40] [--out FILE] [--table FILE]
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
from racinglmpc_b200.reference_params import LaneRuleParams, MeasurementParams   # noqa: E402
from racinglmpc_b200 import _native                                              # noqa: E402
from param_sweep import card                                                     # noqa: E402
from model_sweep import SAME, _spread                                            # noqa: E402
from lap_windows import leg_parent                                               # noqa: E402
import rollout_mc                                                                # noqa: E402

ARMS = (("reference", LaneRuleParams(0, 0.0)), ("tol0", LaneRuleParams(1, 0.0)), ("tol0.02", LaneRuleParams(1, 0.02)))
SIGMAS = (0.0, 0.01)


def leg_cost(rounds, batch, laps, dev):
    arms = {"none": {}, "judge": dict(lane_rule_sets=([LaneRuleParams(1, 1e300)], np.zeros(batch, np.int32)))}
    out = {"benchmark": "lane_rules leg 1: closed loop without a lane-rule table vs an all-mode-1 table at lane_tol 1e300",
           **card(dev), "batch": batch, "laps": laps, "rounds": rounds}
    for mode in ("independent", "pooled"):
        ms, rate, first = {n: [] for n in arms}, {n: [] for n in arms}, {}
        for _ in range(rounds):
            for name, kw in arms.items():
                fin = {}
                r = rollout_mc.run(batch=batch, laps=laps, mode=mode, local=dev, final=fin, books=fin, lap_reports=laps, **kw)
                ms[name].append(r["ms_total"])
                rate[name].append(r["controller_steps_per_s"])
                first.setdefault(name, fin)
        fa, fb = first["none"], first["judge"]
        for k in SAME:
            assert np.array_equal(fa[k], fb[k]), k
        for k in fa["lap_reports"]:
            assert np.array_equal(fa["lap_reports"][k], fb["lap_reports"][k]), k
        a, b = np.array(ms["none"]), np.array(ms["judge"])
        d = 100.0 * (b / a - 1.0)
        out[mode] = {"ms_total": {"none": a.tolist(), "judge": b.tolist()},
                     "controller_steps_per_s": {"none": rate["none"], "judge": rate["judge"]},
                     "judge_over_none_ms_pct_rounds": d.tolist(),
                     "judge_over_none_ms_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
                     "none_round_spread_pct": _spread(a), "judge_round_spread_pct": _spread(b)}
    out["identical"] = list(SAME) + ["lap_reports"]
    return out


def study_tables(batch, laps):
    K = len(ARMS) * len(SIGMAS)
    b = np.arange(batch)
    cell = b % K
    arm, sig = cell % len(ARMS), cell // len(ARMS)
    meas = [MeasurementParams((s,) * 6, (5 * s,) * 6) for s in SIGMAS]
    kw = dict(lane_rule_sets=([r for _, r in ARMS], arm), measurement_sets=(meas, sig), noise_streams=b // K, lap_reports=laps)
    return K, cell, arm, sig, kw


def leg_study(batch, laps, dev):
    K, cell, arm, sig, kw = study_tables(batch, laps)
    bk = {}
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, books=bk, **kw)
    reps = bk["lap_reports"]
    cells = []
    for k in range(K):
        sel = cell == k
        rows = []
        for r in range(laps):
            m = sel & (reps["n"] > r)
            n = int(m.sum())
            rows.append({"lap": r + 1, "controllers": n, "steps_mean": float(reps["steps"][m, r].mean()) if n else 0.0,
                         "violating_share": float((reps["viol_steps"][m, r] > 0).mean()) if n else 0.0,
                         "judged_unsafe_share": float(((reps["flags"][m, r] & _native.REPORT_LANE_UNSAFE) != 0).mean()) if n else 0.0,
                         "unsolved": int(reps["unsolved"][m, r].sum())})
        a, s = int(arm[sel][0]), int(sig[sel][0])
        cells.append({"arm": ARMS[a][0], "mode": ARMS[a][1].mode, "lane_tol": ARMS[a][1].lane_tol, "meas_sigma": SIGMAS[s],
                      "controllers": int(sel.sum()), "per_lap": rows})
    keep = ("closed_loop_steps", "ms_total", "controller_steps_per_s", "unsolved_steps_rank0", "instances_with_flags_rank0",
            "flag_bits_rank0", "per_lane_rule_rank0", "lane_unsafe_selected_share_rank0")
    return {"benchmark": "lane_rules leg 2: reference ranking vs lane rule tol 0 vs tol 0.02 x measurement sigma {0, 0.01}, common "
                         "noise streams (controller // %d), independent mode" % K,
            **card(dev), "batch": batch, "laps": laps, "controllers_per_cell": batch // K, "cells": cells,
            **{k: out[k] for k in keep}}


def summary(study):
    """Leg 2 as a table: per cell, mean steps / violating share (%) / judged-unsafe share (%) / unsolved QPs at a few laps."""
    laps = study["laps"]
    pick = sorted({r for r in (1, 5, 10, 20, 30, 40) if r <= laps} | {laps})
    lines = ["%s, %s, power limit %s W: %d controllers per cell" % (study["benchmark"], study["gpu"], study["power_limit_w"],
                                                                    study["controllers_per_cell"]),
             "arm      sigma  " + "  ".join("lap%-2d steps viol%% unsf%% unsolv" % r for r in pick)]
    for c in study["cells"]:
        row = ["%-8s %5.2f " % (c["arm"], c["meas_sigma"])]
        for r in pick:
            e = c["per_lap"][r - 1]
            row.append("%5d %7.1f %5.1f %5.1f %6d" % (r, e["steps_mean"], 100.0 * e["violating_share"],
                                                      100.0 * e["judged_unsafe_share"], e["unsolved"]))
        lines.append("  ".join(row))
    return "\n".join(lines) + "\n"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of legs 1 and parent")
    ap.add_argument("--batch", type=int, default=8192, help="controllers of leg 1")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps of leg 1")
    ap.add_argument("--study-batch", type=int, default=1536, help="controllers of leg 2 (a multiple of 6)")
    ap.add_argument("--study-laps", type=int, default=40, help="LMPC laps of leg 2")
    ap.add_argument("--legs", default="1,2", help="legs to run; leg parent needs --parent-root")
    ap.add_argument("--parent-root", default="", help="the previous commit's tree with its library built (leg parent)")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    ap.add_argument("--table", default="", help="write leg 2's readable table to this file")
    args = ap.parse_args()
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    legs = args.legs.split(",")
    if "parent" in legs and not args.parent_root:
        ap.error("leg parent needs --parent-root")
    for leg, fn in (("1", lambda: leg_cost(args.rounds, args.batch, args.laps, dev)),
                    ("2", lambda: leg_study(args.study_batch, args.study_laps, dev)),
                    ("parent", lambda: leg_parent(args.rounds, args.parent_root, dev))):
        if leg not in legs:
            continue
        r = fn()
        if leg == "parent":
            r["benchmark"] = "lane_rules leg parent: bench.py configs[1], [2], [3] of this tree against the parent commit's"
        print(json.dumps(r), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(r) + "\n")
        if leg == "2" and args.table:
            with open(args.table, "w") as f:
                f.write(summary(r))


if __name__ == "__main__":
    main()
