#!/usr/bin/env python
"""Per-lap reports (lmpc_rollout_enable_lap_reports): what they cost, and what they show at the reference's experiment length.

Leg 1, A/B: configs[3] (benchmarks/rollout_mc.run: batch 8192, 3 LMPC laps, pooled mode) without and with reports (L = 3), in
alternating rounds in the same process.  Per round: controller steps/s of the LMPC laps (device events).  Both arms must drive the
same closed loop: lap books, end states, health counters and last solver reports are asserted identical.
Leg 2, study: 40 LMPC laps (main.py's Laps = 40 + numSS_it) over measurement noise sigma {0, 0.01, 0.03, 0.1} (the base set of
benchmarks/measurement_noise.py scaled by 0, 1, 3, 10: sigma on vx, vy, wz, s, ey, half of it on epsi, each clipped at five sigma)
crossed with process noise {reference, 2x} (NoiseParams.scaled(sim, 1)) as 8 cells of batch / 8 controllers in one batch
(cell = controller mod 8), independent mode, common random numbers (stream b // 8: the controllers of one row meet the same
draws in every cell).  Per cell and lap: the learning curve (steps per lap: mean, min, max) beside the safety curve (the share of
controllers that left the lane at some step of the lap, mean violating steps, quantiles 50 / 90 / 99 / max of viol_max), the
unsolved QPs and the interior-point iterations per step.

  python benchmarks/lap_reports.py [--rounds 3 --batch 8192] [--legs 1,2] [--study-laps 40] [--out FILE]
Prints one JSON line per leg (card name and power limit read in the same run); --out appends them to FILE as well."""
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
from racinglmpc_b200.reference_params import MeasurementParams, NoiseParams   # noqa: E402
from param_sweep import card                                              # noqa: E402
from noise_sweep import SAME                                              # noqa: E402
from measurement_noise import BASE                                        # noqa: E402
import rollout_mc                                                         # noqa: E402


def leg_ab(rounds, batch, laps, dev):
    arms = {"off": {}, "on": dict(lap_reports=laps)}
    rate = {name: [] for name in arms}
    first = {}
    for _ in range(rounds):
        for name, kw in arms.items():
            fin = {}
            out = rollout_mc.run(batch=batch, laps=laps, mode="pooled", local=dev, final=fin, books=fin, **kw)
            rate[name].append(out["controller_steps_per_s"])
            if name not in first:
                first[name] = (out["lap_stats_rank0"], out["kernel_launches_rank0"], out["closed_loop_steps"], fin, out)
    (st_a, la, na, fa, _), (st_b, lb, nb, fb, ob) = first["off"], first["on"]
    assert st_a == st_b and na == nb and la == lb, (st_a, st_b, la, lb)
    for k in SAME + ("resid",):
        assert np.array_equal(fa[k], fb[k]), k
    a, b = np.array(rate["off"]), np.array(rate["on"])
    d = 100.0 * (a / b - 1.0)                             # time with reports over time without, per round
    return {"benchmark": "lap_reports leg 1: configs[3] (pooled) without vs with per-lap reports", **card(dev), "batch": batch,
            "laps": laps, "mode": "pooled", "rounds": rounds,
            "controller_steps_per_s": {"off": a.tolist(), "on": b.tolist()},
            "time_on_over_off_pct_rounds": d.tolist(),
            "time_on_over_off_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
            "off_round_spread_pct": float(100.0 * (a.max() - a.min()) / a.mean()),
            "on_round_spread_pct": float(100.0 * (b.max() - b.min()) / b.mean()),
            "kernel_launches_rank0": la, "closed_loop_steps": na, "identical": list(SAME + ("resid",)),
            "lap_stats_rank0": st_a, "lap_reports_rank0": ob["lap_reports_rank0"]}


def curves(reps, sel, laps):
    """Per lap, over the controllers `sel` that drove it: steps and the lane-safety statistics of the reports."""
    out = []
    for r in range(laps):
        m = sel & (reps["n"] > r)
        k = int(m.sum())
        st, vs, vm = reps["steps"][m, r], reps["viol_steps"][m, r], reps["viol_max"][m, r]
        q = np.quantile(vm, [0.5, 0.9, 0.99]).tolist() if k else [0.0, 0.0, 0.0]
        tot = int(st.sum(dtype=np.int64))
        out.append({"lap": r + 1, "controllers": k, "steps_mean": float(st.mean()) if k else 0.0,
                    "steps_min": int(st.min()) if k else 0, "steps_max": int(st.max()) if k else 0,
                    "violating_share": float((vs > 0).mean()) if k else 0.0, "viol_steps_mean": float(vs.mean()) if k else 0.0,
                    "viol_max_q50": q[0], "viol_max_q90": q[1], "viol_max_q99": q[2], "viol_max_max": float(vm.max()) if k else 0.0,
                    "unsolved": int(reps["unsolved"][m, r].sum()),
                    "ipm_iters_per_step": float(reps["ipm_iters"][m, r].sum(dtype=np.int64)) / tot if tot else 0.0})
    return out


def leg_study(batch, laps, dev):
    meas_k, proc_k = (0.0, 1.0, 3.0, 10.0), (1.0, 2.0)
    cell = np.arange(batch) % (len(meas_k) * len(proc_k))
    midx, pidx = cell // len(proc_k), cell % len(proc_k)
    bk = {}
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, books=bk, lap_reports=laps,
                         measurement_sets=([MeasurementParams.scaled(k, BASE) for k in meas_k], midx),
                         noise_sets=([NoiseParams.scaled(k, 1.0) for k in proc_k], pidx),
                         noise_streams=np.arange(batch) // 8)
    reps = bk["lap_reports"]
    cells = []
    for m, km in enumerate(meas_k):
        for p, kp in enumerate(proc_k):
            sel = (midx == m) & (pidx == p)
            cells.append({"measurement_sigma": 0.01 * km, "process_scale": kp, "controllers": int(sel.sum()),
                          "finished_every_lap": bool((reps["n"][sel] >= laps).all()),
                          "flag_bits": int(np.bitwise_or.reduce(bk["flags_or"][sel])), "per_lap": curves(reps, sel, laps)})
    return {"benchmark": "lap_reports leg 2: %d LMPC laps, measurement sigma {0, 0.01, 0.03, 0.1} x process noise {x1, x2}, "
                         "independent mode, common random numbers" % laps, **card(dev), "batch": batch, "laps": laps,
            "controllers_per_cell": batch // len(cells), "base_set": {"sigma": BASE.sigma, "clip": BASE.clip},
            "closed_loop_steps": out["closed_loop_steps"], "controller_steps_per_s": out["controller_steps_per_s"],
            "cells": cells}


def summary(study):
    """A readable table of leg 2: per cell, steps per lap and the violating share at laps 1, 2, 5, 10, 20 and the last."""
    laps = study["laps"]
    pick = sorted({r for r in (1, 2, 5, 10, 20, laps) if r <= laps})
    lines = ["%s, %s, power limit %s W: %d controllers per cell, independent mode, stream b // 8" %
             (study["benchmark"], study["gpu"], study["power_limit_w"], study["controllers_per_cell"]),
             "sigma_meas process  " + "  ".join("lap%-2d steps viol%% q99" % r for r in pick)]
    for c in study["cells"]:
        row = ["%-10.2f x%-7g" % (c["measurement_sigma"], c["process_scale"])]
        for r in pick:
            e = c["per_lap"][r - 1]
            row.append("%5d %7.1f %5.1f %+9.3g" % (r, e["steps_mean"], 100.0 * e["violating_share"], e["viol_max_q99"]))
        lines.append("  ".join(row))
    return "\n".join(lines) + "\n"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of leg 1")
    ap.add_argument("--batch", type=int, default=8192, help="controllers per run")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps of leg 1 (configs[3]: 3)")
    ap.add_argument("--study-laps", type=int, default=40, help="LMPC laps of leg 2 (main.py: 40)")
    ap.add_argument("--legs", default="1,2")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    ap.add_argument("--table", default="", help="write leg 2's readable table to this file")
    args = ap.parse_args()
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    legs = args.legs.split(",")
    for leg, fn in (("1", lambda: leg_ab(args.rounds, args.batch, args.laps, dev)),
                    ("2", lambda: leg_study(args.batch, args.study_laps, dev))):
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
