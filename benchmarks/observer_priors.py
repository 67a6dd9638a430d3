#!/usr/bin/env python
"""Observer priors in one batch (lmpc_rollout_set_observer_priors): what the model prior costs, and whether an observer whose
prediction does not come from the controller's own plan lets LMPC's learning survive sensor noise.

Every leg drives its own loop as benchmarks/observers.py does (its controller, drive and pilot conventions), with a state
observer table and a prior table on top.
Leg 1, A/B: alternating rounds at `batch` controllers under the base measurement noise, observer uniform 0.5: no prior table,
all source 0 rows (the plan: bit-identical to no table, asserted) and all source 2 rows (the plant prior).  Per round: controller
steps/s of the LMPC laps (device events).
Leg 2, kernel time: observe_kernel<true> with source 2 rows next to sim_step_kernel over many launches under torch.profiler.
Leg 3, study: measurement noise x{0, 1, 3, 10} of the base set crossed with {no observer, own plan uniform 0.5, plant prior
uniform 0.5, plant prior matched}, as 16 cells of `study_batch` / 16 controllers on common streams, `study_laps` LMPC laps.
"Matched" gains are ObserverParams.from_noise with model_sigma the per-channel RMS of y_{k+1} - p of the plant prior measured in
a pilot run of the x0 cell (observer gains 1 - 2^-20, so that x_hat is y to within 2^-20 of the prior's error) and meas_sigma the
cell's sigma.  Per cell: finishers, unsolved QPs, flag counts, the share of lap-`study_laps` laps that left the lane, and per
channel the RMS of x_est - x against y - x at the polls.
Leg 4, friction drop: the car's friction falls from 1.0 to 0.6 at lap 8 (a vehicle lap schedule), measurement noise x3, observer
uniform 0.5, with {no observer, a believed dry car (source 1, friction 1.0), the plant's car (source 2)}.

  python benchmarks/observer_priors.py [--rounds 3 --batch 8192 --laps 3 --study-batch 4096 --study-laps 20] [--legs 1,2,3,4]
                                       [--out F]
Prints one JSON line per leg (card name and power limit read in the same run); --out appends them to F as well."""
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
from racinglmpc_b200 import reference_params as rp                              # noqa: E402
from racinglmpc_b200 import _native as nat                                      # noqa: E402
from racinglmpc_b200.reference_params import (MeasurementParams, ObserverParams, ObserverPrior,   # noqa: E402
                                              VehicleParams)
from param_sweep import card                                                    # noqa: E402
import observers as obs                                                         # noqa: E402

BASE, CHANNELS = obs.BASE, obs.CHANNELS
HALF = ObserverParams.uniform(0.5)


def controller(B, dev, laps, meas, observers=None, priors=None, streams=None):
    c = obs.controller(B, dev, laps, meas, observers, streams=streams)
    if priors is not None:
        c.set_observer_priors(*priors)
    return c


def leg_ab(rounds, batch, laps, dev):
    z = np.zeros(batch, np.int32)
    arms = {"no_prior": None, "plan": ([ObserverPrior.plan()], z), "plant": ([ObserverPrior.plant()], z)}
    rate = {k: [] for k in arms}
    first = {}
    for _ in range(rounds):
        for name, pri in arms.items():
            c = controller(batch, dev, laps, ([BASE], z), ([HALF], z), pri)
            l0 = c.kernel_launches
            steps, secs = obs.drive(c, laps, dev)
            rate[name].append(batch * steps / secs)
            if name not in first:
                first[name] = (steps, c.kernel_launches - l0, obs.result(c))
            c.close()
    (na, la, ra), (nb, lb, rb), (nc, lc, _) = first["no_prior"], first["plan"], first["plant"]
    assert na == nb and la == lb
    obs.same(ra, rb)
    a, b, p = (np.array(rate[k]) for k in ("no_prior", "plan", "plant"))
    d_plan = 100.0 * (b / a - 1.0)
    d_plant = 100.0 * (p / b - 1.0)
    spread = lambda v: float(100.0 * (v.max() - v.min()) / v.mean())     # noqa: E731
    return {"benchmark": "observer priors leg 1: closed loop under base measurement noise, observer uniform 0.5, without a prior "
                         "table vs source 0 rows vs source 2 rows", **card(dev), "batch": batch, "laps": laps,
            "mode": "independent", "rounds": rounds,
            "controller_steps_per_s": {"no_prior": a.tolist(), "plan": b.tolist(), "plant": p.tolist()},
            "plan_over_no_prior_pct_rounds": d_plan.tolist(), "plant_over_plan_pct_rounds": d_plant.tolist(),
            "plan_over_no_prior_pct": {"mean": float(d_plan.mean()), "min": float(d_plan.min()), "max": float(d_plan.max())},
            "plant_over_plan_pct": {"mean": float(d_plant.mean()), "min": float(d_plant.min()), "max": float(d_plant.max())},
            "round_spread_pct": {"no_prior": spread(a), "plan": spread(b), "plant": spread(p)},
            "kernel_launches_with_pid_lap": {"no_prior": la, "plan": lb, "plant": lc},
            "lmpc_steps": {"no_prior": na, "plan": nb, "plant": nc},
            "identical_no_prior_vs_plan": ["books", "state", "health", "solver", "reports"]}


def leg_kernel(batch, dev, steps=400):
    z = np.zeros(batch, np.int32)
    c = controller(batch, dev, 1, ([BASE], z), ([HALF], z), ([ObserverPrior.plant()], z))
    x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (batch, 1))
    c.rollout_set_state(x0, x0)
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(x0, x0)
    for _ in range(20):                                  # warm-up
        c.rollout_step(seed=1)
        c.rollout_commit_laps_dev()
    torch.cuda.synchronize()
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            c.rollout_step(seed=1)
            c.rollout_commit_laps_dev()
        c.sync()
    times = {}
    for ev in prof.events():
        for k in ("observe_kernel", "measure_kernel", "sim_step_kernel", "ftocp"):
            if k in ev.name and ev.device_type.name == "CUDA":
                times.setdefault(k, []).append(ev.device_time if hasattr(ev, "device_time") else ev.cuda_time)
    formed = int(np.sum(np.all(np.isfinite(obs.read(c, "x_prior", (batch, 6))), axis=1)))
    c.close()
    out = {k: {"launches": len(v), "mean_us": float(np.mean(v)), "min_us": float(np.min(v)), "max_us": float(np.max(v))}
           for k, v in times.items()}
    assert out["observe_kernel"]["launches"] == steps
    return {"benchmark": "observer priors leg 2: kernel times under torch.profiler (CUDA activities), observer uniform 0.5 with "
                         "the plant prior (observe_kernel<true>), base measurement noise, LMPC steps", **card(dev),
            "batch": batch, "steps": steps, "priors_formed_last_step": formed, "kernels": out}


def pilot_plant_sigma(batch, laps, dev):
    """Per-channel RMS of y_{k+1} - p of the plant prior in the x0 cell (gains 1 - 2^-20), at the polls, over controllers that
    formed a finite prior."""
    z = np.zeros(batch, np.int32)
    c = controller(batch, dev, laps, ([MeasurementParams.zero()], z), ([ObserverParams.uniform(1.0 - 2.0 ** -20)], z),
                   ([ObserverPrior.plant()], z))
    acc = {"sq": np.zeros(6), "n": 0}

    def at_poll(when, c):
        if when == "before":
            return
        d = obs.read(c, "x_meas", (batch, 6)) - obs.read(c, "x_prior", (batch, 6))
        ok = np.all(np.isfinite(d), axis=1)
        acc["sq"] += np.sum(d[ok] ** 2, axis=0)
        acc["n"] += int(ok.sum())
    obs.drive(c, laps, dev, at_poll=at_poll)
    c.close()
    return np.sqrt(acc["sq"] / max(acc["n"], 1)), acc["n"]


def _cells_out(sel_of, names, meas_k, laps, acc, bk, flags, unsolved, rep, gains_of):
    out = []
    for m, k in enumerate(meas_k):
        for o, name in enumerate(names):
            sel = sel_of(m, o)
            kk = m * len(names) + o
            n_ok = acc["n"][kk]
            last = sel & (rep["n"] >= laps)
            lap_steps = {}
            for lap in (1, 5, 8, 9, 10, 20):
                if lap <= laps:
                    have = sel & (rep["n"] >= lap)
                    lap_steps[str(lap)] = float(rep["steps"][have, lap - 1].mean()) if have.any() else None
            out.append({
                "measurement_scale": k, "observer": name, "gain": gains_of(m, o),
                "controllers": int(sel.sum()), "finished": int((bk["lap_n"][sel] >= laps).sum()),
                "mean_lap_steps": lap_steps, "unsolved_steps": int(unsolved[sel].sum()),
                "with_flag_1": int((flags[sel] & 1 != 0).sum()),
                "with_reset_flag": int((flags[sel] & nat.FLAG_OBSERVER_RESET != 0).sum()),
                "left_lane_last_lap_share": float((rep["viol_steps"][last, laps - 1] > 0).mean()) if last.any() else None,
                "rms_x_est_minus_x": dict(zip(CHANNELS, np.sqrt(acc["est"][kk] / max(n_ok, 1)).tolist())),
                "rms_y_minus_x": dict(zip(CHANNELS, np.sqrt(acc["meas"][kk] / max(n_ok, 1)).tolist())),
                "rms_samples": int(n_ok)})
    return out


def _rms_poll(batch, cell, cells, acc, hold, from_lap=0):
    def at_poll(when, c):
        if when == "before":
            hold["x"] = c.rollout_state()["x"]
            hold["lap"] = c.books()["lap_n"] if from_lap else None
            return
        x = hold["x"]
        e = obs.read(c, "x_est", (batch, 6)) - x
        y = obs.read(c, "x_meas", (batch, 6)) - x
        ok = np.all(np.isfinite(e), axis=1) & np.all(np.isfinite(y), axis=1) & (np.abs(e[:, 4]) < rp.TRACK_LENGTH / 2)
        if from_lap:
            ok &= hold["lap"] >= from_lap
        for k in range(cells):
            s = ok & (cell == k)
            acc["est"][k] += np.sum(e[s] ** 2, axis=0)
            acc["meas"][k] += np.sum(y[s] ** 2, axis=0)
            acc["n"][k] += s.sum()
    return at_poll


def leg_study(batch, laps, dev, pilot_laps=5):
    meas_k = (0.0, 1.0, 3.0, 10.0)
    ms, n_pilot = pilot_plant_sigma(batch // 16, pilot_laps, dev)
    names = ("none", "plan_0.5", "plant_0.5", "plant_matched")
    cells = len(meas_k) * len(names)
    b = np.arange(batch)
    cell = b % cells
    midx, oidx = cell // len(names), cell % len(names)
    streams = b // cells
    meas_rows = [MeasurementParams.scaled(k, BASE) for k in meas_k]
    obs_rows, obs_of = [ObserverParams.off()], np.zeros(batch, np.int32)
    for m in range(len(meas_k)):
        for o, name in enumerate(names):
            if name == "none":
                continue
            row = HALF if name != "plant_matched" else ObserverParams.from_noise(ms, np.asarray(meas_rows[m].sigma))
            obs_of[(midx == m) & (oidx == o)] = len(obs_rows)
            obs_rows.append(row)
    pri_of = np.where(np.isin(oidx, (2, 3)), 1, 0).astype(np.int32)
    c = controller(batch, dev, laps, (meas_rows, midx), (obs_rows, obs_of), ([ObserverPrior.plan(), ObserverPrior.plant()], pri_of),
                   streams=streams)
    acc = {"est": np.zeros((cells, 6)), "meas": np.zeros((cells, 6)), "n": np.zeros(cells)}
    steps, secs = obs.drive(c, laps, dev, at_poll=_rms_poll(batch, cell, cells, acc, {}))
    bk = c.books()
    flags, unsolved = c.rollout_health()
    rep = c.lap_reports()
    c.close()

    def gains_of(m, o):
        row = obs_rows[int(obs_of[(midx == m) & (oidx == o)][0])]
        return list(row.gain) if row.mode == 1 else None
    out_cells = _cells_out(lambda m, o: (midx == m) & (oidx == o), names, meas_k, laps, acc, bk, flags, unsolved, rep, gains_of)
    return {"benchmark": "observer priors leg 3: closed-loop LMPC over measurement noise x{0,1,3,10} x {none, own plan 0.5, "
                         "plant prior 0.5, plant prior matched}, independent mode, common noise streams", **card(dev),
            "batch": batch, "controllers_per_cell": batch // cells, "laps": laps, "lmpc_steps": steps, "seconds": secs,
            "base_set": {"sigma": BASE.sigma, "clip": BASE.clip},
            "matched_model_sigma": dict(zip(CHANNELS, ms.tolist())), "pilot": {"laps": pilot_laps, "samples": n_pilot},
            "cells": out_cells}


def leg_drop(batch, laps, dev, drop_lap=8):
    names = ("none", "believed_dry_car", "plant_car")
    cells = len(names)
    b = np.arange(batch)
    cell = b % cells
    streams = b // cells
    dry, wet = VehicleParams.from_friction(1.0), VehicleParams.from_friction(0.6)
    z = np.zeros(batch, np.int32)
    obs_of = (cell != 0).astype(np.int32)
    c = controller(batch, dev, laps, ([MeasurementParams.scaled(3, BASE)], z), ([ObserverParams.off(), HALF], obs_of),
                   ([ObserverPrior.plan(), ObserverPrior.car(dry), ObserverPrior.plant()], cell.astype(np.int32)),
                   streams=streams)
    c.set_vehicles([dry, wet], z)
    c.set_lap_schedule("vehicle", [0] * drop_lap + [1])
    acc = {"est": np.zeros((cells, 6)), "meas": np.zeros((cells, 6)), "n": np.zeros(cells)}
    steps, secs = obs.drive(c, laps, dev, at_poll=_rms_poll(batch, cell, cells, acc, {}, from_lap=drop_lap))
    bk = c.books()
    flags, unsolved = c.rollout_health()
    rep = c.lap_reports()
    c.close()
    out_cells = _cells_out(lambda m, o: cell == o, names, (3.0,), laps, acc, bk, flags, unsolved, rep,
                           lambda m, o: None if o == 0 else list(HALF.gain))
    return {"benchmark": "observer priors leg 4: friction 1.0 -> 0.6 at lap %d (vehicle lap schedule), measurement noise x3, "
                         "observer uniform 0.5 with a believed dry car (source 1) vs the plant's car (source 2); RMS from lap %d"
                         % (drop_lap, drop_lap), **card(dev), "batch": batch, "controllers_per_cell": batch // cells,
            "laps": laps, "lmpc_steps": steps, "seconds": secs, "cells": out_cells}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of leg 1")
    ap.add_argument("--batch", type=int, default=8192, help="controllers of legs 1 and 2")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps of leg 1")
    ap.add_argument("--study-batch", type=int, default=4096, help="controllers of leg 3 (16 cells)")
    ap.add_argument("--drop-batch", type=int, default=768, help="controllers of leg 4 (3 cells)")
    ap.add_argument("--study-laps", type=int, default=20)
    ap.add_argument("--legs", default="1,2,3,4")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/observer_priors.py needs a GPU")
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    legs = args.legs.split(",")
    for leg, fn in (("1", lambda: leg_ab(args.rounds, args.batch, args.laps, dev)), ("2", lambda: leg_kernel(args.batch, dev)),
                    ("3", lambda: leg_study(args.study_batch, args.study_laps, dev)),
                    ("4", lambda: leg_drop(args.drop_batch, args.study_laps, dev))):
        if leg not in legs:
            continue
        r = fn()
        print(json.dumps(r), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
