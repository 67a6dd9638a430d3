#!/usr/bin/env python
"""Per-controller lap windows (lmpc_set_lap_windows): what a window table costs, and what windows do when the friction drops while
LMPC learns.

Leg 1, cost: benchmarks/rollout_mc.run (PID lap, seeding, `laps` LMPC laps, independent mode, lap reports on) in alternating
rounds in the same process, with
  none       no window table;
  unbounded  a table of all-(0, 0) rows: every book kernel reads the window table, every window unbounded.
Per round: ms of the LMPC laps and controller steps/s (device events).  Both arms must drive the same closed loop: books, end
states, health, solver reports and lap reports are asserted identical.
Leg 2, against the parent build (--parent-root: a checkout of the previous commit with its library built): bench.py --config 1, 2
and 3 with --dump-outputs, alternating this tree and the parent's in `rounds` rounds (odd rounds parent first); every dumped array
of both trees is compared bit for bit.
Leg 3, study: the circuit of configs[3], `study-laps` LMPC laps, lap reports on, independent mode, on the rollout_mc handle
(numSS_it 4, ss_cap 7, trToUse 4, model_cap 5).  Friction arms "drop" (mu 1.0 for LMPC laps 1-7, 0.6 from lap 8 on, a vehicle lap
schedule) and "constant" (1.0 throughout), crossed with ss_window in {0, 4, 7} and model_window in {0, 4}: 12 cells in one batch,
cell = controller mod 12, on noise streams controller // 12 (common random numbers).  Per cell and lap: controllers that filed it,
mean steps, share of controllers with a lane violation, unsolved QPs and flagged controllers (report flags != 0).

  python benchmarks/lap_windows.py [--rounds 5 --batch 8192 --laps 3] [--legs 1,2,3] [--parent-root DIR]
                                   [--study-batch 1536 --study-laps 16] [--out FILE] [--table FILE]
Prints one JSON line per leg (card name and power limit read in the same run); --out appends them to FILE as well, --table writes
leg 3 as a readable table."""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "benchmarks")):
    if p not in sys.path:
        sys.path.insert(0, p)
from racinglmpc_b200.reference_params import LapWindowParams, VehicleParams   # noqa: E402
from param_sweep import card                                                  # noqa: E402
from model_sweep import SAME, _spread, _bench, _same_dumps                    # noqa: E402
import rollout_mc                                                             # noqa: E402

SWITCH_LAP = 8           # the first LMPC lap under the new friction
ARMS = (("drop", 1.0, 0.6), ("constant", 1.0, 1.0))
SS_WINDOWS = (0, 4, 7)
MODEL_WINDOWS = (0, 4)


def leg_cost(rounds, batch, laps, dev):
    arms = {"none": {}, "unbounded": dict(lap_window_sets=([LapWindowParams.unbounded()], np.zeros(batch, np.int32)))}
    ms, rate, first = {n: [] for n in arms}, {n: [] for n in arms}, {}
    for _ in range(rounds):
        for name, kw in arms.items():
            fin = {}
            out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, final=fin, books=fin, lap_reports=laps, **kw)
            ms[name].append(out["ms_total"])
            rate[name].append(out["controller_steps_per_s"])
            first.setdefault(name, fin)
    fa, fb = first["none"], first["unbounded"]
    for k in SAME:
        assert np.array_equal(fa[k], fb[k]), k
    for k in fa["lap_reports"]:
        assert np.array_equal(fa["lap_reports"][k], fb["lap_reports"][k]), k
    a, b = np.array(ms["none"]), np.array(ms["unbounded"])
    d = 100.0 * (b / a - 1.0)
    return {"benchmark": "lap_windows leg 1: closed loop without a window table vs a table of unbounded (0, 0) rows", **card(dev),
            "batch": batch, "laps": laps, "mode": "independent", "rounds": rounds,
            "ms_total": {"none": a.tolist(), "unbounded": b.tolist()},
            "controller_steps_per_s": {"none": rate["none"], "unbounded": rate["unbounded"]},
            "unbounded_over_none_ms_pct_rounds": d.tolist(),
            "unbounded_over_none_ms_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
            "none_round_spread_pct": _spread(a), "unbounded_round_spread_pct": _spread(b),
            "identical": list(SAME) + ["lap_reports"]}


def leg_parent(rounds, parent_root, dev):
    arms = {"parent": os.path.abspath(parent_root), "this": ROOT}
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(rounds):
            order = ["parent", "this"] if r % 2 == 0 else ["this", "parent"]
            row = {"round": r + 1, "order": order}
            dirs = {name: {} for name in order}
            for name in order:
                row[name] = {}
                for cfg in (1, 2, 3):
                    d = os.path.join(tmp, "%s_r%d_c%d" % (name, r, cfg))
                    j = _bench(arms[name], cfg, d)
                    row[name]["config%d_ms_per_step" % cfg] = j["ms_per_step"]
                    dirs[name][cfg] = d
            for cfg in (1, 2, 3):
                names, same = _same_dumps(dirs["parent"][cfg], dirs["this"][cfg])
                row["config%d_dumps_identical" % cfg] = same
                row["config%d_dumped" % cfg] = len(names)
            rows.append(row)
    out = {"benchmark": "lap_windows leg 2: bench.py configs[1], [2], [3] of this tree against the parent commit's", **card(dev),
           "rounds": rows}
    for cfg in (1, 2, 3):
        key = "config%d_ms_per_step" % cfg
        a = np.array([r["parent"][key] for r in rows], float)
        b = np.array([r["this"][key] for r in rows], float)
        d = 100.0 * (b / a - 1.0)
        out[key] = {"parent": a.tolist(), "this": b.tolist(), "this_over_parent_pct_rounds": d.tolist(),
                    "parent_round_spread_pct": _spread(a), "this_round_spread_pct": _spread(b)}
    out["all_dumps_identical"] = all(r["config%d_dumps_identical" % c] for r in rows for c in (1, 2, 3))
    return out


def study_cells(batch, laps):
    """The 12 cells (arm, ss_window, model_window) and the tables of run(): vehicle sets (mu 1.0, 0.6) with their schedule, window
    sets and noise streams."""
    K = len(ARMS) * len(SS_WINDOWS) * len(MODEL_WINDOWS)
    b = np.arange(batch)
    cell = b % K
    arm, sw, mw = cell // 6, (cell // 2) % 3, cell % 2
    mu = {1.0: 0, 0.6: 1}
    sched = np.empty((batch, SWITCH_LAP), np.int32)
    for a, (_, before, after) in enumerate(ARMS):
        sched[arm == a, :SWITCH_LAP - 1] = mu[before]
        sched[arm == a, SWITCH_LAP - 1] = mu[after]
    wins = [LapWindowParams(s, m) for s in SS_WINDOWS for m in MODEL_WINDOWS]
    kw = dict(vehicle_sets=([VehicleParams.from_friction(1.0), VehicleParams.from_friction(0.6)], sched[:, 0].copy()),
              lap_window_sets=(wins, sw * len(MODEL_WINDOWS) + mw), noise_streams=b // K, lap_reports=laps,
              lap_schedules={"vehicle": sched})
    return K, cell, (arm, sw, mw), kw


def leg_study(batch, laps, dev):
    K, cell, (arm, sw, mw), kw = study_cells(batch, laps)
    bk = {}
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, books=bk, **kw)
    reps = bk["lap_reports"]
    cells = []
    for k in range(K):
        sel = cell == k
        a = int(arm[sel][0])
        rows = []
        for r in range(laps):
            m = sel & (reps["n"] > r)
            n = int(m.sum())
            rows.append({"lap": r + 1, "controllers": n, "steps_mean": float(reps["steps"][m, r].mean()) if n else 0.0,
                         "violating_share": float((reps["viol_steps"][m, r] > 0).mean()) if n else 0.0,
                         "unsolved": int(reps["unsolved"][m, r].sum()), "flagged": int((reps["flags"][m, r] != 0).sum())})
        cells.append({"arm": ARMS[a][0], "mu_before": ARMS[a][1], "mu_after": ARMS[a][2], "ss_window": SS_WINDOWS[int(sw[sel][0])],
                      "model_window": MODEL_WINDOWS[int(mw[sel][0])], "controllers": int(sel.sum()), "per_lap": rows})
    keep = ("closed_loop_steps", "ms_total", "controller_steps_per_s", "unsolved_steps_rank0", "instances_with_flags_rank0",
            "flag_bits_rank0", "per_lap_window_rank0")
    return {"benchmark": "lap_windows leg 3: friction drop 1.0 -> 0.6 at LMPC lap %d vs constant 1.0 x ss_window {0,4,7} x "
                         "model_window {0,4}, common noise streams (controller // %d), independent mode" % (SWITCH_LAP, K),
            **card(dev), "batch": batch, "laps": laps, "switch_lap": SWITCH_LAP, "controllers_per_cell": batch // K,
            "cells": cells, **{k: out[k] for k in keep}}


def summary(study):
    """Leg 3 as a table: per cell, mean steps / violating share (%) / unsolved QPs at laps 6 .. 12 and the last."""
    laps = study["laps"]
    pick = sorted({r for r in range(SWITCH_LAP - 2, SWITCH_LAP + 5) if r <= laps} | {laps})
    lines = ["%s, %s, power limit %s W: %d controllers per cell" % (study["benchmark"], study["gpu"], study["power_limit_w"],
                                                                    study["controllers_per_cell"]),
             "arm       ssW mdW  " + "  ".join("lap%-2d steps viol%% unsolv" % r for r in pick)]
    for c in study["cells"]:
        row = ["%-8s %3d %3d " % (c["arm"], c["ss_window"], c["model_window"])]
        for r in pick:
            e = c["per_lap"][r - 1]
            row.append("%5d %7.1f %5.1f %6d" % (r, e["steps_mean"], 100.0 * e["violating_share"], e["unsolved"]))
        lines.append("  ".join(row))
    return "\n".join(lines) + "\n"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of legs 1 and 2")
    ap.add_argument("--batch", type=int, default=8192, help="controllers of leg 1")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps of leg 1")
    ap.add_argument("--study-batch", type=int, default=1536, help="controllers of leg 3 (a multiple of 12)")
    ap.add_argument("--study-laps", type=int, default=16, help="LMPC laps of leg 3")
    ap.add_argument("--legs", default="1,3", help="legs to run; leg 2 needs --parent-root")
    ap.add_argument("--parent-root", default="", help="the previous commit's tree with its library built (leg 2)")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    ap.add_argument("--table", default="", help="write leg 3's readable table to this file")
    args = ap.parse_args()
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    legs = args.legs.split(",")
    if "2" in legs and not args.parent_root:
        ap.error("leg 2 needs --parent-root")
    for leg, fn in (("1", lambda: leg_cost(args.rounds, args.batch, args.laps, dev)),
                    ("2", lambda: leg_parent(args.rounds, args.parent_root, dev)),
                    ("3", lambda: leg_study(args.study_batch, args.study_laps, dev))):
        if leg not in legs:
            continue
        r = fn()
        print(json.dumps(r), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(r) + "\n")
        if leg == "3" and args.table:
            with open(args.table, "w") as f:
                f.write(summary(r))


if __name__ == "__main__":
    main()
