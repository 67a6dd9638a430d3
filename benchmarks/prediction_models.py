#!/usr/bin/env python
"""Per-controller prediction models (lmpc_set_prediction_models): what the table and the nominal model's kernel cost, and what a
controller that plans with the exact linearisation of a car does that a learned one does not.

Leg 1, identity and cost: benchmarks/rollout_mc.run at configs[3] (8 192 controllers, 3 LMPC laps, lap reports on), independent
and pooled, without a table against an all-mode-0 table, in alternating rounds in one process.  Both arms must drive the same
closed loop: books, end states, health, solver reports and lap reports are asserted identical in the run.  Per round: ms of the
LMPC laps; the difference against the round-to-round spread.
Leg 2, kernel time: the configs[2] controller state (workloads.lmpc_batch: a 5-lap model store, 4-lap safe set, N = 12) at each
batch size, lmpc_step_profile's ms4[0] in alternating rounds under
  none     no table: K1 alone;
  learned  an all-mode-0 table: K1 (NOMINAL instantiation, every CTA regresses) + nominal_model_kernel (every thread returns);
  nominal  an all-mode-2 table: K1 (every CTA returns at once) + nominal_model_kernel (every stage identified).
The nominal kernel's fp64 work is counted from shapes (nominal_flops below: the arithmetic of one sub-step, the transcendental
calls counted apart) and set against the DFMA rate lmpc_probe_fp64 measures on the same card.
Leg 3, study A (lane crossings): the lane-margin study's setting -- the circuit of configs[3], `study-laps` LMPC laps with lap
reports, independent mode, common noise streams (controller // 8) -- over {learned, mode 2} x margin {0, fixed 0.05} x
measurement sigma {0, 0.01} (all six channels, clip 5 sigma), `per-cell` controllers per cell.  Per cell and lap: mean steps,
the share of controllers whose plant state left the lane, unsolved QPs.
Leg 4, study B (friction drop): the lap-schedule drop of the vehicle from mu 1.0 to 0.6 at LMPC lap 8, over 16 laps, with the arms
learned, mode 2 (follows the schedule) and mode 1 on the dry car (mu 1.0 throughout), common noise streams (controller // 3).
Legs 3 and 4 also trace 32 controllers per prediction arm and report the one-step prediction error of (vx, vy, wz),
x_{t+1} - xPred_t[1], over all traced steps and over the last 5 laps (leg 5 of the design).

  python benchmarks/prediction_models.py [--legs 1,2,3,4] [--rounds 3 --batch 8192 --laps 3] [--batches 4096,8192 --reps 20]
                                         [--per-cell 256 --study-laps 40] [--out FILE] [--table FILE]
Prints one JSON line per leg (card name and power limit read in the same run); --out appends them to FILE as well, --table
writes legs 3 and 4 as readable tables."""
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
from racinglmpc_b200 import _native as nat, reference_params as rp, workloads    # noqa: E402
from racinglmpc_b200.controller import BatchedController                          # noqa: E402
from racinglmpc_b200.reference_params import PredictionModelParams as P           # noqa: E402
from racinglmpc_b200.reference_params import LaneMarginParams, MeasurementParams, VehicleParams   # noqa: E402
from param_sweep import card                                                      # noqa: E402
from model_sweep import SAME, _spread                                             # noqa: E402
import rollout_mc                                                                 # noqa: E402

SUBSTEPS = 100            # (i + 1) * 0.001 <= dt = 0.1


def nominal_flops(batch, N):
    """fp64 operations of nominal_model_kernel for batch x N stages, from the code's shapes: per sub-step the rates and their
    derivatives (~45 operations besides the calls), f_z S + f_u E and the update of S (3 x 5 entries, 8 each), the state update
    (14); per stage the constant rows and C (~60).  Transcendental calls (2 atan2, 2 atan, 2 sin, 2 cos per sub-step, 2
    reciprocals) are counted apart: their cost depends on the libdevice path taken."""
    per_sub = 45 + 3 * 5 * 8 + 14
    return {"flops": float(batch * N * (SUBSTEPS * per_sub + 60)), "transcendental_calls": float(batch * N * SUBSTEPS * 10)}


def controller(B):
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(12)
    c = BatchedController(par, B, workloads.track_seg_table(), rp.TRACK_LENGTH, trToUse=5, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1280, ss_cap=6, model_cap=6)
    data = workloads.lmpc_batch(B)
    workloads.restore_lmpc_batch(c, data)
    return c, data


def leg_kernel(batches, rounds, reps, dev):
    out = {"benchmark": "prediction_models leg 2: lmpc_step_profile ms4[0] (K1, plus nominal_model_kernel under a table)",
           **card(dev.index), "rounds": rounds, "reps_per_round": reps, "fp64_probe": nat.probe_fp64(dev.index)}
    arms = {"none": None, "learned": [P.learned()], "nominal": [P.plant()]}
    for B in batches:
        c, data = controller(B)
        try:
            x0 = torch.from_numpy(data["x0"]).to(dev)
            st = c.get_state()
            ms = {a: [] for a in arms}
            for _ in range(rounds):
                for a, rows in arms.items():
                    c.set_prediction_models(rows, None if rows is None else np.zeros(B, int))
                    t = []
                    for _ in range(reps + 2):
                        c.set_state(xLin=st["xLin"], uLin=st["uLin"], zt=st["zt"], OldInput=st["OldInput"], timeStep=st["timeStep"])
                        t.append(c.step_profile(x0.data_ptr())[0])
                    ms[a].append(float(np.median(t[2:])))
            res = {a: {"ms_rounds": v, "ms_median": float(np.median(v))} for a, v in ms.items()}
            fl = nominal_flops(B, 12)
            t_nom = res["nominal"]["ms_median"] * 1e-3
            res["nominal_fp64"] = dict(fl, achieved_tflops=fl["flops"] / t_nom / 1e12,
                                       frac_of_dfma=fl["flops"] / t_nom / 1e12 / out["fp64_probe"]["dfma_tflops"])
            res["nominal_over_k1"] = res["nominal"]["ms_median"] / res["none"]["ms_median"]
            res["learned_over_none_pct"] = 100.0 * (res["learned"]["ms_median"] / res["none"]["ms_median"] - 1.0)
            res["none_round_spread_pct"] = 100.0 * (max(ms["none"]) - min(ms["none"])) / float(np.median(ms["none"]))
            out["batch_%d" % B] = res
        finally:
            c.close()
    return out


def leg_identity(rounds, batch, laps, dev):
    arms = {"none": {}, "learned": dict(prediction_model_sets=([P.learned()], np.zeros(batch, np.int32)))}
    out = {"benchmark": "prediction_models leg 1: closed loop without a table vs an all-mode-0 table", **card(dev), "batch": batch,
           "laps": laps, "rounds": rounds}
    for mode in ("independent", "pooled"):
        ms, first = {n: [] for n in arms}, {}
        for _ in range(rounds):
            for name, kw in arms.items():
                fin = {}
                r = rollout_mc.run(batch=batch, laps=laps, mode=mode, local=dev, final=fin, books=fin, lap_reports=laps, **kw)
                ms[name].append(r["ms_total"])
                first.setdefault(name, fin)
        fa, fb = first["none"], first["learned"]
        for k in SAME:
            assert np.array_equal(fa[k], fb[k]), k
        for k in fa["lap_reports"]:
            assert np.array_equal(fa["lap_reports"][k], fb["lap_reports"][k]), k
        a, b = np.array(ms["none"]), np.array(ms["learned"])
        d = 100.0 * (b / a - 1.0)
        out[mode] = {"ms_total": {"none": a.tolist(), "learned": b.tolist()}, "learned_over_none_ms_pct_rounds": d.tolist(),
                     "learned_over_none_ms_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
                     "none_round_spread_pct": _spread(a), "learned_round_spread_pct": _spread(b)}
    out["identical"] = list(SAME) + ["lap_reports"]
    return out


def _cells(reps, cell, K, laps):
    """Per cell and lap: controllers that filed the lap, their mean steps, the share whose plant state left the lane, unsolved QPs."""
    out = []
    for k in range(K):
        rows = []
        for r in range(laps):
            m = (cell == k) & (reps["n"] > r)
            n = int(m.sum())
            rows.append({"lap": r + 1, "controllers": n, "steps_mean": float(reps["steps"][m, r].mean()) if n else 0.0,
                         "violating_share": float((reps["viol_steps"][m, r] > 0).mean()) if n else 0.0,
                         "unsolved": int(reps["unsolved"][m, r].sum())})
        out.append(rows)
    return out


def _traced(arm_of, n_arms, per_arm=32):
    """The first `per_arm` controllers of every prediction arm."""
    return np.concatenate([np.nonzero(arm_of == a)[0][:per_arm] for a in range(n_arms)])


def prediction_error(tr, inst, arm_of, names, last_laps=5):
    """Per prediction arm: RMS and mean |.| of x_{t+1} - xPred_t[1] on (vx, vy, wz) over the traced steps (consecutive rows of one
    controller), and over the steps of its last `last_laps` laps."""
    out = {}
    for a, name in enumerate(names):
        err, late = [], []
        for t, b in enumerate(inst):
            if arm_of[b] != a:
                continue
            n = tr["steps"][t]
            x, xp, lp = tr["x"][t][:n], tr["xPred"][t][:n], tr["lap"][t][:n]
            e = x[1:, :3] - xp[:-1, 1, :3]
            err.append(e)
            late.append(e[lp[:-1] >= lp.max() - last_laps + 1])
        e, l = np.concatenate(err), np.concatenate(late)
        out[name] = {"controllers": len(err), "steps": int(e.shape[0]), "rms": np.sqrt((e ** 2).mean(0)).tolist(),
                     "mean_abs": np.abs(e).mean(0).tolist(), "rms_last_laps": np.sqrt((l ** 2).mean(0)).tolist() if l.size else None,
                     "last_laps": last_laps}
    return out


PRED = (("learned", P.learned()), ("mode2", P.plant()))
MARGINS = (("margin0", LaneMarginParams(0)), ("fixed0.05", LaneMarginParams(1, 0.05, 0.05)))
SIGMAS = (0.0, 0.01)


def leg_study_a(per_cell, laps, cap, dev):
    K = len(PRED) * len(MARGINS) * len(SIGMAS)
    batch = K * per_cell
    b = np.arange(batch)
    cell = b % K
    pred, marg, sig = cell % 2, (cell // 2) % 2, cell // 4
    meas = [MeasurementParams((s,) * 6, (5 * s,) * 6) for s in SIGMAS]
    inst = _traced(pred, len(PRED))
    tr = {"inst": inst, "cap": cap}
    bk = {}
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, books=bk, lap_reports=laps, noise_streams=b // K,
                         prediction_model_sets=([r for _, r in PRED], pred), lane_margin_sets=([r for _, r in MARGINS], marg),
                         measurement_sets=(meas, sig), trace=tr)
    per = _cells(bk["lap_reports"], cell, K, laps)
    cells = [{"prediction": PRED[k % 2][0], "margin": MARGINS[(k // 2) % 2][0], "meas_sigma": SIGMAS[k // 4],
              "controllers": int((cell == k).sum()), "per_lap": per[k]} for k in range(K)]
    return {"benchmark": "prediction_models leg 3 (study A): {learned, mode 2} x margin {0, fixed 0.05} x measurement sigma {0, 0.01}, "
                         "common noise streams (controller // %d), independent mode" % K,
            **card(dev), "batch": batch, "laps": laps, "controllers_per_cell": per_cell, "cells": cells,
            "prediction_error": prediction_error(tr, inst, pred, [n for n, _ in PRED]),
            **{k: out[k] for k in ("closed_loop_steps", "ms_total", "unsolved_steps_rank0", "instances_with_flags_rank0",
                                   "flag_bits_rank0", "per_prediction_model_rank0")}}


SWITCH_LAP = 8           # the first LMPC lap under the new friction (benchmarks/lap_schedule.py)
DRY, WET = VehicleParams.from_friction(1.0), VehicleParams.from_friction(0.6)
PRED_B = (("learned", P.learned()), ("mode2", P.plant()), ("mode1_dry", P.believes(DRY)))


def leg_study_b(per_cell, laps, cap, dev):
    K = len(PRED_B)
    batch = K * per_cell
    b = np.arange(batch)
    cell = b % K
    sched = np.zeros((batch, SWITCH_LAP), np.int32)
    sched[:, SWITCH_LAP - 1] = 1
    inst = _traced(cell, K)
    tr = {"inst": inst, "cap": cap}
    bk = {}
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, books=bk, lap_reports=laps, noise_streams=b // K,
                         vehicle_sets=([DRY, WET], np.zeros(batch, np.int32)), lap_schedules={"vehicle": sched},
                         prediction_model_sets=([r for _, r in PRED_B], cell), trace=tr)
    per = _cells(bk["lap_reports"], cell, K, laps)
    cells = [{"prediction": PRED_B[k][0], "controllers": int((cell == k).sum()), "per_lap": per[k]} for k in range(K)]
    return {"benchmark": "prediction_models leg 4 (study B): friction 1.0 -> 0.6 at LMPC lap %d; learned, mode 2 (follows the "
                         "schedule), mode 1 on the dry car; common noise streams (controller // %d), independent mode" % (SWITCH_LAP, K),
            **card(dev), "batch": batch, "laps": laps, "controllers_per_cell": per_cell, "cells": cells,
            "prediction_error": prediction_error(tr, inst, cell, [n for n, _ in PRED_B]),
            **{k: out[k] for k in ("closed_loop_steps", "ms_total", "unsolved_steps_rank0", "instances_with_flags_rank0",
                                   "flag_bits_rank0", "per_prediction_model_rank0")}}


def summary(study):
    """A study as a table: per cell, mean steps / violating share (%) / unsolved QPs at a few laps, then the prediction errors."""
    laps = study["laps"]
    pick = sorted({r for r in (1, 5, 7, 8, 9, 10, 16, 20, 30, 40) if r <= laps} | {laps})
    lines = ["%s, %s, power limit %s W: %d controllers per cell" % (study["benchmark"], study["gpu"], study["power_limit_w"],
                                                                    study["controllers_per_cell"]),
             "cell                          " + "  ".join("lap%-2d steps viol%% unsolv" % r for r in pick)]
    for c in study["cells"]:
        name = " ".join(str(c[k]) for k in ("prediction", "margin", "meas_sigma") if k in c)
        row = ["%-29s" % name]
        for r in pick:
            e = c["per_lap"][r - 1]
            row.append("%5d %7.1f %5.1f %6d" % (r, e["steps_mean"], 100.0 * e["violating_share"], e["unsolved"]))
        lines.append("  ".join(row))
    lines.append("one-step prediction error x_{t+1} - xPred_t[1], RMS of (vx, vy, wz): all traced steps | last %d laps"
                 % next(iter(study["prediction_error"].values()))["last_laps"])
    for name, e in study["prediction_error"].items():
        lines.append("  %-10s %2d controllers %6d steps  %s | %s" % (name, e["controllers"], e["steps"],
                                                                    " ".join("%.2e" % v for v in e["rms"]),
                                                                    " ".join("%.2e" % v for v in (e["rms_last_laps"] or []))))
    return "\n".join(lines) + "\n"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="1,2,3,4")
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of legs 1 and 2")
    ap.add_argument("--batch", type=int, default=8192, help="controllers of leg 1")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps of leg 1")
    ap.add_argument("--batches", default="4096,8192", help="batch sizes of leg 2")
    ap.add_argument("--reps", type=int, default=20, help="steps per round of leg 2")
    ap.add_argument("--per-cell", type=int, default=256, help="controllers per cell of legs 3 and 4")
    ap.add_argument("--study-laps", type=int, default=40, help="LMPC laps of leg 3 (leg 4 drives 16)")
    ap.add_argument("--trace-cap", type=int, default=6000, help="traced steps per controller in legs 3 and 4")
    ap.add_argument("--out", default=None)
    ap.add_argument("--table", default=None, help="write legs 3 and 4 as readable tables to this file")
    a = ap.parse_args()
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    legs = a.legs.split(",")
    tables = []
    for leg, fn in (("1", lambda: leg_identity(a.rounds, a.batch, a.laps, dev)),
                    ("2", lambda: leg_kernel([int(b) for b in a.batches.split(",")], a.rounds, a.reps, torch.device("cuda", dev))),
                    ("3", lambda: leg_study_a(a.per_cell, a.study_laps, a.trace_cap, dev)),
                    ("4", lambda: leg_study_b(a.per_cell, 16, a.trace_cap, dev))):
        if leg not in legs:
            continue
        line = json.dumps(fn())
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")
        if leg in ("3", "4"):
            tables.append(summary(json.loads(line)))
    if a.table and tables:
        with open(a.table, "w") as f:
            f.write("\n".join(tables))


if __name__ == "__main__":
    main()
