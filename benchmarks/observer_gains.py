#!/usr/bin/env python
"""Model-based observer gains in one batch (lmpc_rollout_set_observer_gains): what the frozen-time Kalman gain costs, and whether
it keeps the observer's estimate from running away under sensor noise where fixed gains did not.

Every leg drives its own loop as benchmarks/observers.py does, with observer, prior and gain tables on top
(benchmarks/observer_priors.py's controller and poll conventions).
Leg 1, A/B: alternating rounds at `batch` controllers under the base measurement noise, observer uniform 0.5, plant prior: no
gain table against all mode 0 rows (bit-identical, asserted).  Per round: controller steps/s of the LMPC laps (device events).
Leg 2, kernel time: observer_gain_kernel with mode 1 rows next to observe_kernel<true, true> and sim_step_kernel over many
launches under torch.profiler.
Leg 3, study: measurement noise x{0, 1, 3, 10} of the base set crossed with {no observer, plant prior with gain 0.5, plant prior
with model gains}, `study_batch` / 12 controllers per cell on common streams, `study_laps` LMPC laps.  The model gains are
ObserverGains.from_noise(the reference process noise, the cell's sensor, model_sigma) with model_sigma the per-channel RMS of
y_{k+1} - p of the plant prior in a pilot run without sensor noise (benchmarks/observer_priors.py), floored at 1e-6 so that every
q_j > 0.  The x0 cell has no sensor noise, so from_noise has r = 0 there: it takes r = 1e-12 (K close to I) instead.  Per cell:
finishers, unsolved steps, lap-`study_laps` lane exits and length, per channel RMS of x_est - x, the controllers whose estimate
ran away (at some poll |x_est - x| above 1 m on s or 0.5 m on ey, or not finite), and the controllers with reset and gain flags.
Leg 4, friction drop: the car's friction falls from 1.0 to 0.6 at lap 8, measurement noise x3, model gains of the x3 cell, with a
believed dry car (source 1) against the plant's car (source 2).

  python benchmarks/observer_gains.py [--rounds 3 --batch 8192 --laps 3 --study-batch 3072 --study-laps 20] [--legs 1,2,3,4]
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
from racinglmpc_b200 import _native as nat                                      # noqa: E402
from racinglmpc_b200 import reference_params as rp                              # noqa: E402
from racinglmpc_b200.reference_params import (MeasurementParams, NoiseParams, ObserverGains, ObserverParams,   # noqa: E402
                                              ObserverPrior, VehicleParams)
from param_sweep import card                                                    # noqa: E402
import observers as obs                                                         # noqa: E402
import observer_priors as opb                                                   # noqa: E402

BASE, CHANNELS = obs.BASE, obs.CHANNELS
HALF = ObserverParams.uniform(0.5)
RUNAWAY = (1.0, 0.5)                                     # |x_est - x| on s, on ey


def controller(B, dev, laps, meas, observers, priors, gains=None, streams=None):
    c = opb.controller(B, dev, laps, meas, observers, priors, streams=streams)
    if gains is not None:
        c.set_observer_gains(*gains)
    return c


def model_gains(meas, ms):
    if all(s == 0.0 for s in meas.sigma):
        g = ObserverGains.from_noise(NoiseParams.reference(), BASE, ms)
        return ObserverGains.kalman(g.q, 1e-12)
    return ObserverGains.from_noise(NoiseParams.reference(), meas, ms)


def leg_ab(rounds, batch, laps, dev):
    z = np.zeros(batch, np.int32)
    arms = {"no_table": None, "fixed": ([ObserverGains.fixed()], z)}
    rate = {k: [] for k in arms}
    first = {}
    for _ in range(rounds):
        for name, g in arms.items():
            c = controller(batch, dev, laps, ([BASE], z), ([HALF], z), ([ObserverPrior.plant()], z), g)
            l0 = c.kernel_launches
            steps, secs = obs.drive(c, laps, dev)
            rate[name].append(batch * steps / secs)
            if name not in first:
                first[name] = (steps, c.kernel_launches - l0, obs.result(c))
            c.close()
    (na, la, ra), (nb, lb, rb) = first["no_table"], first["fixed"]
    assert na == nb
    obs.same(ra, rb)
    a, b = (np.array(rate[k]) for k in ("no_table", "fixed"))
    d = 100.0 * (b / a - 1.0)
    spread = lambda v: float(100.0 * (v.max() - v.min()) / v.mean())     # noqa: E731
    return {"benchmark": "observer gains leg 1: closed loop under base measurement noise, observer uniform 0.5, plant prior, "
                         "without a gain table vs mode 0 rows", **card(dev), "batch": batch, "laps": laps,
            "mode": "independent", "rounds": rounds,
            "controller_steps_per_s": {"no_table": a.tolist(), "fixed": b.tolist()},
            "fixed_over_no_table_pct_rounds": d.tolist(),
            "fixed_over_no_table_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
            "round_spread_pct": {"no_table": spread(a), "fixed": spread(b)},
            "kernel_launches_with_pid_lap": {"no_table": la, "fixed": lb}, "lmpc_steps": {"no_table": na, "fixed": nb},
            "identical_no_table_vs_fixed": ["books", "state", "health", "solver", "reports"]}


def leg_kernel(batch, dev, steps=200):
    z = np.zeros(batch, np.int32)
    g = model_gains(BASE, np.full(6, 1e-3))
    c = controller(batch, dev, 1, ([BASE], z), ([HALF], z), ([ObserverPrior.plant()], z), ([g], z))
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
        for k in ("observer_gain_kernel", "observe_kernel", "measure_kernel", "sim_step_kernel", "ftocp"):
            if k in ev.name and ev.device_type.name == "CUDA":
                times.setdefault(k, []).append(ev.device_time if hasattr(ev, "device_time") else ev.cuda_time)
                break
    formed = int(np.sum(np.all(np.isfinite(obs.read(c, "obs_gain", (batch, 36))), axis=1)))
    c.close()
    out = {k: {"launches": len(v), "mean_us": float(np.mean(v)), "min_us": float(np.min(v)), "max_us": float(np.max(v))}
           for k, v in times.items()}
    assert out["observer_gain_kernel"]["launches"] == steps
    return {"benchmark": "observer gains leg 2: kernel times under torch.profiler (CUDA activities), observer uniform 0.5, plant "
                         "prior, model gains (observer_gain_kernel, observe_kernel<true, true>), base measurement noise, LMPC "
                         "steps", **card(dev), "batch": batch, "steps": steps, "gains_formed_last_step": formed, "kernels": out}


def _runaway_poll(batch, inner, worst, hold):
    def at_poll(when, c):
        if when == "before":
            hold["x"] = c.rollout_state()["x"]
        inner(when, c)
        if when == "before":
            return
        e = obs.read(c, "x_est", (batch, 6)) - hold["x"]
        bad = ~np.all(np.isfinite(e), axis=1) | (np.abs(e[:, 4]) > RUNAWAY[0]) | (np.abs(e[:, 5]) > RUNAWAY[1])
        # |e_s| near a lap is the lap wrap of a controller whose estimate crossed the line a step before the plant: not a runaway
        bad &= ~(np.abs(np.abs(e[:, 4]) - rp.TRACK_LENGTH) < 2 * RUNAWAY[0])
        np.logical_or(worst, bad, out=worst)
    return at_poll


def _study_cells(sel_of, names, meas_k, laps, acc, bk, flags, unsolved, rep, gains_of, runaway):
    out = opb._cells_out(sel_of, names, meas_k, laps, acc, bk, flags, unsolved, rep, gains_of)
    k = 0
    for m in range(len(meas_k)):
        for o in range(len(names)):
            sel = sel_of(m, o)
            last = sel & (rep["n"] >= laps)
            out[k]["runaway_estimates"] = int((runaway & sel).sum())
            out[k]["with_gain_flag"] = int((flags[sel] & nat.FLAG_OBSERVER_GAIN != 0).sum())
            out[k]["left_lane_last_lap"] = int((rep["viol_steps"][last, laps - 1] > 0).sum()) if last.any() else 0
            k += 1
    return out


def leg_study(batch, laps, dev, pilot_laps=5):
    meas_k = (0.0, 1.0, 3.0, 10.0)
    ms, n_pilot = opb.pilot_plant_sigma(batch // 12, pilot_laps, dev)
    ms = np.maximum(ms, 1e-6)
    names = ("none", "plant_0.5", "plant_model_gains")
    cells = len(meas_k) * len(names)
    b = np.arange(batch)
    cell = b % cells
    midx, oidx = cell // len(names), cell % len(names)
    streams = b // cells
    meas_rows = [MeasurementParams.scaled(k, BASE) for k in meas_k]
    obs_of = (oidx != 0).astype(np.int32)
    pri_of = np.zeros(batch, np.int32)
    gain_rows = [ObserverGains.fixed()] + [model_gains(m, ms) for m in meas_rows]
    gain_of = np.where(oidx == 2, 1 + midx, 0).astype(np.int32)
    c = controller(batch, dev, laps, (meas_rows, midx), ([ObserverParams.off(), HALF], obs_of), ([ObserverPrior.plant()], pri_of),
                   (gain_rows, gain_of), streams=streams)
    acc = {"est": np.zeros((cells, 6)), "meas": np.zeros((cells, 6)), "n": np.zeros(cells)}
    runaway = np.zeros(batch, bool)
    steps, secs = obs.drive(c, laps, dev, at_poll=_runaway_poll(batch, opb._rms_poll(batch, cell, cells, acc, {}), runaway, {}))
    bk = c.books()
    flags, unsolved = c.rollout_health()
    rep = c.lap_reports()
    c.close()

    def gains_of(m, o):
        if o == 0:
            return None
        if o == 1:
            return list(HALF.gain)
        g = gain_rows[1 + m]
        return {"q": list(g.q), "r": list(g.r)}
    out_cells = _study_cells(lambda m, o: (midx == m) & (oidx == o), names, meas_k, laps, acc, bk, flags, unsolved, rep, gains_of,
                             runaway)
    return {"benchmark": "observer gains leg 3: closed-loop LMPC over measurement noise x{0,1,3,10} x {none, plant prior 0.5, "
                         "plant prior with model gains}, independent mode, common noise streams", **card(dev),
            "batch": batch, "controllers_per_cell": batch // cells, "laps": laps, "lmpc_steps": steps, "seconds": secs,
            "base_set": {"sigma": BASE.sigma, "clip": BASE.clip}, "runaway_threshold_s_ey": RUNAWAY,
            "model_sigma": dict(zip(CHANNELS, ms.tolist())), "pilot": {"laps": pilot_laps, "samples": n_pilot},
            "cells": out_cells}


def leg_drop(batch, laps, dev, ms, drop_lap=8):
    names = ("none", "believed_dry_car", "plant_car")
    cells = len(names)
    b = np.arange(batch)
    cell = b % cells
    streams = b // cells
    dry, wet = VehicleParams.from_friction(1.0), VehicleParams.from_friction(0.6)
    z = np.zeros(batch, np.int32)
    meas = MeasurementParams.scaled(3, BASE)
    obs_of = (cell != 0).astype(np.int32)
    pri_of = np.where(cell == 1, 0, 1).astype(np.int32)
    c = controller(batch, dev, laps, ([meas], z), ([ObserverParams.off(), HALF], obs_of),
                   ([ObserverPrior.car(dry), ObserverPrior.plant()], pri_of), ([model_gains(meas, ms)], z), streams=streams)
    c.set_vehicles([dry, wet], z)
    c.set_lap_schedule("vehicle", [0] * drop_lap + [1])
    acc = {"est": np.zeros((cells, 6)), "meas": np.zeros((cells, 6)), "n": np.zeros(cells)}
    runaway = np.zeros(batch, bool)
    steps, secs = obs.drive(c, laps, dev, at_poll=_runaway_poll(
        batch, opb._rms_poll(batch, cell, cells, acc, {}, from_lap=drop_lap), runaway, {}))
    bk = c.books()
    flags, unsolved = c.rollout_health()
    rep = c.lap_reports()
    c.close()
    out_cells = _study_cells(lambda m, o: cell == o, names, (3.0,), laps, acc, bk, flags, unsolved, rep,
                             lambda m, o: None if o == 0 else "model gains", runaway)
    return {"benchmark": "observer gains leg 4: friction 1.0 -> 0.6 at lap %d (vehicle lap schedule), measurement noise x3, "
                         "observer with model gains, a believed dry car (source 1) vs the plant's car (source 2); RMS from lap "
                         "%d" % (drop_lap, drop_lap), **card(dev), "batch": batch, "controllers_per_cell": batch // cells,
            "laps": laps, "lmpc_steps": steps, "seconds": secs, "model_sigma": dict(zip(CHANNELS, ms.tolist())),
            "cells": out_cells}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of leg 1")
    ap.add_argument("--batch", type=int, default=8192, help="controllers of legs 1 and 2")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps of leg 1")
    ap.add_argument("--study-batch", type=int, default=3072, help="controllers of leg 3 (12 cells)")
    ap.add_argument("--drop-batch", type=int, default=768, help="controllers of leg 4 (3 cells)")
    ap.add_argument("--study-laps", type=int, default=20)
    ap.add_argument("--legs", default="1,2,3,4")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/observer_gains.py needs a GPU")
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    legs = args.legs.split(",")
    ms = {}

    def study():
        r = leg_study(args.study_batch, args.study_laps, dev)
        ms["v"] = np.array([r["model_sigma"][k] for k in CHANNELS])
        return r

    def drop():
        if "v" not in ms:
            ms["v"] = np.maximum(opb.pilot_plant_sigma(args.study_batch // 12, 5, dev)[0], 1e-6)
        return leg_drop(args.drop_batch, args.study_laps, dev, ms["v"])
    for leg, fn in (("1", lambda: leg_ab(args.rounds, args.batch, args.laps, dev)), ("2", lambda: leg_kernel(args.batch, dev)),
                    ("3", study), ("4", drop)):
        if leg not in legs:
            continue
        r = fn()
        print(json.dumps(r), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
