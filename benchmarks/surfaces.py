#!/usr/bin/env python
"""Track surfaces (lmpc_rollout_set_surfaces): what a surface table costs the closed loop and the plant kernels, and how a learned
and a physics prediction model cope with grip that changes within a lap.

Leg 1, identity and cost: benchmarks/rollout_mc.run at configs[3] (8 192 controllers, 3 LMPC laps, lap reports on), independent
and pooled, in alternating rounds in one process, under
  none     no table;
  dry      an all-dry table (nzone = 0): sim_step_kernel with an empty row;
  ones16   a 16-zone table with every mu = 1 spread over the lap (the worst-case lookup: the cursor walks every zone).
All arms must drive the same closed loop: books, end states, health, solver reports and lap reports are asserted identical in the
run.  Per round: ms of the LMPC laps; each table's difference against the round-to-round spread.
Leg 2, kernel time: torch.profiler CUDA activity of `reps` lmpc_rollout_pid_step launches at each batch size, controllers spread
over the lap, per-launch time of sim_step_kernel under no table, an all-dry table and the 16-zone table; and lmpc_step_profile's
ms4[0] (K1, whose CTAs return at once, + nominal_model_kernel) of the configs[2] controller state under an all-mode-2 prediction
table without and with the 16-zone surface, in alternating rounds.
Leg 3, study (a wet corner): the lane study's setting -- the circuit of configs[3], `study-laps` LMPC laps with lap reports,
independent mode, common noise streams (controller // 6) -- over surface {dry, the first curve wet from the start, the same
curve wet from LMPC lap 8 by schedule} x prediction {learned, mode 2}, `per-cell` controllers per cell.  Wet is mu_f = mu_r = 0.75
on segment 1 (the 4.5 m left-hand curve after the start straight): 0.6 where the dry car has the reference's 0.8.  Per cell and
lap: mean steps, the share of controllers whose plant state left the lane, unsolved QPs.  From traces of 32 controllers per cell:
the RMS one-step prediction error x_{t+1} - xPred_t[1] of (vx, vy, wz) over steps that start inside the curve's s range against
steps outside it (the scheduled arm counts its wet laps only), and the share of lane-violating traced steps whose s lies in the
curve.

  python benchmarks/surfaces.py [--legs 1,2,3] [--rounds 3 --batch 8192 --laps 3] [--batches 4096,8192 --reps 50]
                                [--per-cell 256 --study-laps 40] [--out FILE] [--table FILE]
Prints one JSON line per leg (card name and power limit read in the same run); --out appends them to FILE as well, --table
writes leg 3 as a readable table."""
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
from racinglmpc_b200 import reference_params as rp, workloads                   # noqa: E402
from racinglmpc_b200.controller import BatchedController                         # noqa: E402
from racinglmpc_b200.reference_params import PredictionModelParams as P, SurfaceParams as S   # noqa: E402
from param_sweep import card                                                     # noqa: E402
from model_sweep import SAME, _spread                                            # noqa: E402
import prediction_models as pmb                                                  # noqa: E402
import rollout_mc                                                                # noqa: E402

L = rp.TRACK_LENGTH
HALF_WIDTH = rp.HALF_WIDTH
ONES16 = S.from_zones([(k * L / 16, (k + 0.5) * L / 16, 1.0, 1.0) for k in range(16)])
CURVE_ROW = 1
WET_CURVE = S.on_segment(rp.TrackParams.l_shaped(), CURVE_ROW, 0.75)
SWITCH_LAP = 8                     # the first LMPC lap on the wet curve in the scheduled arm


def _tables(batch):
    return {"none": None, "dry": ([S.dry()], np.zeros(batch, np.int32)), "ones16": ([ONES16], np.zeros(batch, np.int32))}


def leg_identity(rounds, batch, laps, dev):
    arms = _tables(batch)
    out = {"benchmark": "surfaces leg 1: closed loop without a table vs an all-dry and a 16-zone mu = 1 table", **card(dev),
           "batch": batch, "laps": laps, "rounds": rounds}
    for mode in ("independent", "pooled"):
        ms, first = {n: [] for n in arms}, {}
        for _ in range(rounds):
            for name, sets in arms.items():
                fin = {}
                r = rollout_mc.run(batch=batch, laps=laps, mode=mode, local=dev, final=fin, books=fin, lap_reports=laps,
                                   surface_sets=sets)
                ms[name].append(r["ms_total"])
                first.setdefault(name, fin)
        for name in ("dry", "ones16"):
            fa, fb = first["none"], first[name]
            for k in SAME:
                assert np.array_equal(fa[k], fb[k]), (name, k)
            for k in fa["lap_reports"]:
                assert np.array_equal(fa["lap_reports"][k], fb["lap_reports"][k]), (name, k)
        a = np.array(ms["none"])
        res = {"ms_total": {n: v for n, v in ms.items()}, "none_round_spread_pct": _spread(a)}
        for name in ("dry", "ones16"):
            d = 100.0 * (np.array(ms[name]) / a - 1.0)
            res[name + "_over_none_ms_pct_rounds"] = d.tolist()
            res[name + "_over_none_ms_pct"] = {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())}
            res[name + "_round_spread_pct"] = _spread(np.array(ms[name]))
        out[mode] = res
    out["identical"] = list(SAME) + ["lap_reports"]
    return out


def _kernel_ms(prof, name):
    """Mean device time per launch (ms) and the launch count of the kernels whose name holds `name`."""
    ts = [e.device_time for e in prof.events() if name in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
    return (float(np.mean(ts)) * 1e-3 if ts else float("nan")), len(ts)


def leg_kernel(batches, rounds, reps, dev):
    out = {"benchmark": "surfaces leg 2: sim_step_kernel per launch (torch.profiler, lmpc_rollout_pid_step) and lmpc_step_profile "
                        "ms4[0] of an all-mode-2 prediction table", **card(dev.index), "rounds": rounds, "reps_per_round": reps}
    act = [torch.profiler.ProfilerActivity.CUDA]
    for B in batches:
        res = {}
        numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(12)
        c = BatchedController(par, B, workloads.track_seg_table(), L, trToUse=4, numSS_Points=numSS_Points, numSS_it=numSS_it,
                              QterminalSlack=Qts, Tmax=1280, ss_cap=6, model_cap=5)
        try:
            c.enable_rollout(Tcl=3 * (reps + 1) * rounds + 16)   # every launch keeps its record row
            s0 = np.linspace(0.0, L, B, endpoint=False)
            x0 = np.stack([np.full(B, 1.0), np.zeros(B), np.zeros(B), np.zeros(B), s0, np.zeros(B)], 1)
            sim = {a: [] for a in _tables(B)}
            for _ in range(rounds):
                for a, sets in _tables(B).items():
                    c.set_surfaces(*(sets if sets is not None else (None,)))
                    c.rollout_set_state(x0, x0)
                    c.rollout_pid_step(1.0, seed=5)                    # warm-up launch under this table
                    c.sync()
                    with torch.profiler.profile(activities=act) as prof:
                        for _ in range(reps):
                            c.rollout_pid_step(1.0, seed=5)
                        c.sync()
                    ms, n = _kernel_ms(prof, "sim_step_kernel")
                    assert n == reps, (a, n)
                    sim[a].append(ms)
            res["sim_step_ms_per_launch"] = {a: {"rounds": v, "median": float(np.median(v))} for a, v in sim.items()}
            for a in ("dry", "ones16"):
                res["sim_step_%s_over_none_pct" % a] = 100.0 * (res["sim_step_ms_per_launch"][a]["median"] /
                                                                 res["sim_step_ms_per_launch"]["none"]["median"] - 1.0)
            res["sim_step_none_round_spread_pct"] = _spread(np.array(sim["none"]))
        finally:
            c.close()
        c, data = pmb.controller(B)
        try:
            x0d = torch.from_numpy(data["x0"]).to(dev)
            st = c.get_state()
            c.set_prediction_models([P.plant()], np.zeros(B, int))
            nom = {"none": [], "ones16": []}
            for _ in range(rounds):
                for a in nom:
                    c.set_surfaces(*((None,) if a == "none" else ([ONES16], np.zeros(B, int))))
                    t = []
                    for _ in range(reps // 2 + 2):
                        c.set_state(xLin=st["xLin"], uLin=st["uLin"], zt=st["zt"], OldInput=st["OldInput"], timeStep=st["timeStep"])
                        t.append(c.step_profile(x0d.data_ptr())[0])
                    nom[a].append(float(np.median(t[2:])))
            res["nominal_ms4_0"] = {a: {"rounds": v, "median": float(np.median(v))} for a, v in nom.items()}
            res["nominal_ones16_over_none_pct"] = 100.0 * (res["nominal_ms4_0"]["ones16"]["median"] /
                                                           res["nominal_ms4_0"]["none"]["median"] - 1.0)
            res["nominal_none_round_spread_pct"] = _spread(np.array(nom["none"]))
        finally:
            c.close()
        out["batch_%d" % B] = res
    return out


SURF = ("dry", "wet_from_start", "wet_from_lap%d" % SWITCH_LAP)
PRED = (("learned", P.learned()), ("mode2", P.plant()))


def _in_curve(s):
    s = np.where(s > L, s - L, s)
    s0, s1 = WET_CURVE.zones[0][:2]
    return (s >= s0) & (s < s1)


def zone_errors(tr, inst, cell_of, names):
    """Per cell: the RMS one-step prediction error of (vx, vy, wz) over traced steps that start in the curve against steps that
    start outside it (the scheduled arm: its wet laps only), and the share of traced lane-violating steps (|ey| > the half
    width) whose s lies in the curve."""
    out = {}
    for k, name in enumerate(names):
        ins, outs, viol, viol_in = [], [], 0, 0
        for t, b in enumerate(inst):
            if cell_of[b] != k:
                continue
            n = tr["steps"][t]
            x, xp, lp = tr["x"][t][:n], tr["xPred"][t][:n], tr["lap"][t][:n]
            e = x[1:, :3] - xp[:-1, 1, :3]
            curve = _in_curve(x[:-1, 4])
            keep = lp[:-1] >= SWITCH_LAP - 1 if name.startswith("wet_from_lap") else np.ones(n - 1, bool)
            ins.append(e[curve & keep])
            outs.append(e[~curve & keep])
            v = np.abs(x[:, 5]) > HALF_WIDTH
            viol += int(v.sum())
            viol_in += int((v & _in_curve(x[:, 4])).sum())
        ei, eo = np.concatenate(ins), np.concatenate(outs)
        out[name] = {"steps_in_curve": int(ei.shape[0]), "steps_outside": int(eo.shape[0]),
                     "rms_in_curve": np.sqrt((ei ** 2).mean(0)).tolist() if ei.size else None,
                     "rms_outside": np.sqrt((eo ** 2).mean(0)).tolist() if eo.size else None,
                     "violating_steps": viol, "violating_share_in_curve": viol_in / viol if viol else None}
    return out


def leg_study(per_cell, laps, cap, dev):
    K = len(SURF) * len(PRED)
    batch = K * per_cell
    b = np.arange(batch)
    cell = b % K
    surf, pred = cell // 2, cell % 2
    sched = np.zeros((batch, SWITCH_LAP), np.int32)
    sched[surf == 1] = 1
    sched[surf == 2, SWITCH_LAP - 1] = 1
    own = (surf == 1).astype(np.int32)                             # the PID lap ignores schedules: the wet-from-start arm seeds wet
    inst = np.concatenate([np.nonzero(cell == k)[0][:32] for k in range(K)])
    tr = {"inst": inst, "cap": cap}
    bk = {}
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, books=bk, lap_reports=laps, noise_streams=b // K,
                         surface_sets=([S.dry(), WET_CURVE], own), lap_schedules={"surface": sched},
                         prediction_model_sets=([r for _, r in PRED], pred), trace=tr)
    names = ["%s %s" % (SURF[k // 2], PRED[k % 2][0]) for k in range(K)]
    per = pmb._cells(bk["lap_reports"], cell, K, laps)
    cells = [{"surface": SURF[k // 2], "prediction": PRED[k % 2][0], "controllers": int((cell == k).sum()), "per_lap": per[k]}
             for k in range(K)]
    return {"benchmark": "surfaces leg 3 (study): segment %d of the configs[3] circuit at mu 0.75 (dry car 0.8) -- dry, wet from the "
                         "start, wet from LMPC lap %d -- x {learned, mode 2}; common noise streams (controller // %d), independent "
                         "mode" % (CURVE_ROW, SWITCH_LAP, K),
            **card(dev), "batch": batch, "laps": laps, "controllers_per_cell": per_cell, "curve": list(WET_CURVE.zones[0]),
            "cells": cells, "zone_errors": zone_errors(tr, inst, cell, names),
            **{k: out[k] for k in ("closed_loop_steps", "ms_total", "unsolved_steps_rank0", "instances_with_flags_rank0",
                                   "flag_bits_rank0", "per_prediction_model_rank0")}}


def summary(study):
    """The study as a table: per cell, mean steps / violating share (%) / unsolved QPs at a few laps, then the zone errors."""
    laps = study["laps"]
    pick = sorted({r for r in (1, 5, 7, 8, 9, 10, 16, 20, 30, 40) if r <= laps} | {laps})
    lines = ["%s, %s, power limit %s W: %d controllers per cell" % (study["benchmark"], study["gpu"], study["power_limit_w"],
                                                                    study["controllers_per_cell"]),
             "cell                        " + "  ".join("lap%-2d steps viol%% unsolv" % r for r in pick)]
    for c in study["cells"]:
        row = ["%-27s" % ("%s %s" % (c["surface"], c["prediction"]))]
        for r in pick:
            e = c["per_lap"][r - 1]
            row.append("%5d %7.1f %5.1f %6d" % (r, e["steps_mean"], 100.0 * e["violating_share"], e["unsolved"]))
        lines.append("  ".join(row))
    lines.append("one-step prediction error x_{t+1} - xPred_t[1], RMS of (vx, vy, wz): steps starting in the curve | outside it; "
                 "share of traced lane-violating steps in the curve")
    for name, e in study["zone_errors"].items():
        f = lambda v: " ".join("%.2e" % q for q in v) if v else "-"       # noqa: E731
        share = e["violating_share_in_curve"]
        lines.append("  %-27s %5d | %6d steps  %s | %s   %s of %d" % (name, e["steps_in_curve"], e["steps_outside"], f(e["rms_in_curve"]),
                                                                     f(e["rms_outside"]), "-" if share is None else "%.2f" % share,
                                                                     e["violating_steps"]))
    return "\n".join(lines) + "\n"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="1,2,3")
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of legs 1 and 2")
    ap.add_argument("--batch", type=int, default=8192, help="controllers of leg 1")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps of leg 1")
    ap.add_argument("--batches", default="4096,8192", help="batch sizes of leg 2")
    ap.add_argument("--reps", type=int, default=50, help="launches per round of leg 2")
    ap.add_argument("--per-cell", type=int, default=256, help="controllers per cell of leg 3")
    ap.add_argument("--study-laps", type=int, default=40, help="LMPC laps of leg 3")
    ap.add_argument("--trace-cap", type=int, default=8000, help="traced steps per controller in leg 3")
    ap.add_argument("--out", default=None)
    ap.add_argument("--table", default=None, help="write leg 3 as a readable table to this file")
    a = ap.parse_args()
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    legs = a.legs.split(",")
    tables = []
    for leg, fn in (("2", lambda: leg_kernel([int(b) for b in a.batches.split(",")], a.rounds, a.reps, torch.device("cuda", dev))),
                    ("3", lambda: leg_study(a.per_cell, a.study_laps, a.trace_cap, dev)),
                    ("1", lambda: leg_identity(a.rounds, a.batch, a.laps, dev))):
        if leg not in legs:
            continue
        line = json.dumps(fn())
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")
        if leg == "3":
            tables.append(summary(json.loads(line)))
    if a.table and tables:
        with open(a.table, "w") as f:
            f.write("\n".join(tables))


if __name__ == "__main__":
    main()
