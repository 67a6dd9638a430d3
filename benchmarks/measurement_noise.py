#!/usr/bin/env python
"""Measurement noise in one batch (lmpc_rollout_set_measurement_noise): what the measurement kernel costs, how much sensor noise
LMPC's learning from its own laps absorbs, and whether common random numbers still pair two tunings when the controllers see
noisy measurements.

Leg 1, A/B: benchmarks/rollout_mc.run (PID lap, seeding, `laps` LMPC laps; independent mode) in alternating rounds in the same
process, with
  no_table  no measurement table (no kernel is launched, every controller reads the plant state);
  zero_set  an all-zero measurement set installed for every controller: the measurement kernel runs every step and copies the
            plant state, so this is the whole cost of the feature.
Per round: controller steps/s of the LMPC laps (device events).  Both arms must drive the same closed loop: their lap books, end
states, health counters and last solver reports are asserted identical.
Leg 2, grid: measurement noise x{0, 1, 10, 100} of the base set crossed with process noise x{1, 10} (NoiseParams.scaled(sim, 1))
as 8 cells of batch / 8 controllers in one batch (cell = controller mod 8), independent mode: per cell, mean / minimum length of
every LMPC lap (n = controllers that finished it), unsolved steps, flagged controllers and how many carry flag bit 1 (K1: a
regression lookup failed) and bit 2 (K2: the safe-set selection found no point), which a measured s < 0 near the start line sets.
The base set (BASE): sigma 0.01 on vx, vy, wz (m/s, rad/s), on s and ey (m), 0.005 rad on epsi, each clipped at five sigma: a
wheel-speed / IMU and a centimetre-class position sensor, the size of the reference's process noise on the velocities
(sigma 0.01, 0.01, 0.005 before its gain).
Leg 3, common random numbers under measurement noise: the two QP tunings of noise_sweep.py leg 3 (dR x0.5 and x2) interleaved,
the base measurement set on every controller, run twice: unpaired (streams b) and paired (streams b // 2, which pairs the
measurement draws as well).  Per LMPC lap: the mean lap-length difference, its unpaired and paired standard errors and the
correlation of the pair's lap lengths (noise_sweep.pair_stats).

  python benchmarks/measurement_noise.py [--rounds 5 --batch 8192 --laps 3] [--legs 1,2,3] [--out FILE]
Prints one JSON line per leg (card name and power limit read in the same run); --out appends them to FILE as well."""
import argparse
import copy
import json
import os
import sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "benchmarks")):
    if p not in sys.path:
        sys.path.insert(0, p)
from racinglmpc_b200 import reference_params as rp                        # noqa: E402
from racinglmpc_b200.reference_params import MeasurementParams, NoiseParams   # noqa: E402
from param_sweep import card                                              # noqa: E402
from noise_sweep import SAME, pair_stats                                  # noqa: E402
import rollout_mc                                                         # noqa: E402

BASE = MeasurementParams((0.01, 0.01, 0.01, 0.005, 0.01, 0.01), (0.05, 0.05, 0.05, 0.025, 0.05, 0.05))


def leg_ab(rounds, batch, laps, dev):
    arms = {"no_table": {}, "zero_set": dict(measurement_sets=([MeasurementParams.zero()], np.zeros(batch, np.int32)))}
    rate = {name: [] for name in arms}
    first = {}
    for _ in range(rounds):
        for name, kw in arms.items():
            fin = {}
            out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, final=fin, books=fin, **kw)
            rate[name].append(out["controller_steps_per_s"])
            if name not in first:
                first[name] = (out["lap_stats_rank0"], out["kernel_launches_rank0"], out["closed_loop_steps"], fin)
    (st_a, la, na, fa), (st_b, lb, nb, fb) = first["no_table"], first["zero_set"]
    assert st_a == st_b and na == nb, (st_a, st_b)
    assert lb - la == nb, (la, lb, nb)                     # one measurement launch per closed-loop step, nothing else
    for k in SAME + ("resid",):
        assert np.array_equal(fa[k], fb[k]), k
    a, b = np.array(rate["no_table"]), np.array(rate["zero_set"])
    d = 100.0 * (b / a - 1.0)
    return {"benchmark": "measurement_noise leg 1: closed loop without a measurement table vs an all-zero set for every controller",
            **card(dev), "batch": batch, "laps": laps, "mode": "independent", "rounds": rounds,
            "controller_steps_per_s": {"no_table": a.tolist(), "zero_set": b.tolist()},
            "zero_set_over_no_table_pct_rounds": d.tolist(),
            "zero_set_over_no_table_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
            "no_table_round_spread_pct": float(100.0 * (a.max() - a.min()) / a.mean()),
            "zero_set_round_spread_pct": float(100.0 * (b.max() - b.min()) / b.mean()),
            "kernel_launches_rank0": {"no_table": la, "zero_set": lb}, "closed_loop_steps": na,
            "identical": list(SAME + ("resid",)), "lap_stats_rank0": st_a}


def leg_grid(batch, laps, dev):
    meas_k, proc_k = (0.0, 1.0, 10.0, 100.0), (1.0, 10.0)
    cell = np.arange(batch) % (len(meas_k) * len(proc_k))
    midx, pidx = cell // len(proc_k), cell % len(proc_k)
    bk = {}
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, books=bk,
                         measurement_sets=([MeasurementParams.scaled(k, BASE) for k in meas_k], midx),
                         noise_sets=([NoiseParams.scaled(k, 1.0) for k in proc_k], pidx))
    cells = []
    for m, km in enumerate(meas_k):
        for p, kp in enumerate(proc_k):
            sel = (midx == m) & (pidx == p)
            s = rollout_mc._set_stats(bk, bk["flags_or"], bk["unsolved"], sel, laps)
            s.update(measurement_scale=km, process_scale=kp, finished_every_lap=all(l["n"] == s["controllers"] for l in s["laps"]),
                     with_flag_1=int((bk["flags_or"][sel] & 1 != 0).sum()), with_flag_2=int((bk["flags_or"][sel] & 2 != 0).sum()),
                     flag_bits=int(np.bitwise_or.reduce(bk["flags_or"][sel])))
            cells.append(s)
    for k in ("benchmark", "per_measurement_rank0", "per_noise_rank0"):
        out.pop(k)
    return {"benchmark": "measurement_noise leg 2: closed-loop LMPC over measurement noise x{0,1,10,100} x process noise x{1,10}, "
                         "independent mode", **card(dev), "base_set": {"sigma": BASE.sigma, "clip": BASE.clip},
            "cells": cells, "controllers_per_cell": batch // len(cells), **out}


def leg_crn(batch, laps, dev):
    _, _, _, _, _, base = rp.lmpc_params(rollout_mc.N_HORIZON)
    ps = []
    for s in (0.5, 2.0):
        p = copy.deepcopy(base)
        p.dR = s * np.asarray(base.dR, float)
        ps.append(p)
    pidx = np.arange(batch) % 2
    meas = ([BASE], np.zeros(batch, np.int32))
    out = {"benchmark": "measurement_noise leg 3: two QP tunings (dR x0.5, x2) interleaved under the base measurement noise, "
                        "unpaired (streams b) vs paired (streams b // 2)",
           **card(dev), "batch": batch, "laps": laps, "mode": "independent", "tunings": ["dR x0.5", "dR x2"],
           "base_set": {"sigma": BASE.sigma, "clip": BASE.clip}}
    for name, streams in (("unpaired", None), ("paired", np.arange(batch) // 2)):
        bk = {}
        o = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, books=bk, param_sets=(ps, pidx, None),
                           noise_streams=streams, measurement_sets=meas)
        out[name] = {"per_lap": pair_stats(bk, laps), "per_set_rank0": o["per_set_rank0"],
                     "controller_steps_per_s": o["controller_steps_per_s"]}
    for arm in ("unpaired", "paired"):
        for p in out[arm]["per_lap"]:
            p["se_ratio_paired_over_unpaired"] = p["se_paired"] / p["se_unpaired"] if p["se_unpaired"] > 0 else None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of leg 1")
    ap.add_argument("--batch", type=int, default=8192, help="controllers per run")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps every controller drives")
    ap.add_argument("--legs", default="1,2,3")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args()
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    legs = args.legs.split(",")
    for leg, fn in (("1", lambda: leg_ab(args.rounds, args.batch, args.laps, dev)), ("2", lambda: leg_grid(args.batch, args.laps, dev)),
                    ("3", lambda: leg_crn(args.batch, args.laps, dev))):
        if leg not in legs:
            continue
        r = fn()
        print(json.dumps(r), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
