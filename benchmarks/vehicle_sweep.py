#!/usr/bin/env python
"""Plant sweeps in one batch (lmpc_rollout_set_vehicles): what per-controller vehicles cost, and a closed-loop friction x mass grid.

Leg 1, A/B: benchmarks/rollout_mc.run (PID lap, seeding, `laps` LMPC laps; independent mode) in alternating rounds in the same
process, with
  no_sets   no vehicle table installed (the simulator reads the reference vehicle from the handle's one-row default table);
  one_set   the reference vehicle installed as the only set, with an index for every controller.
Per round: controller steps/s of the LMPC laps (device events).  Both arms must drive the same closed loop: their lap books, end
states and health counters are asserted identical.
Leg 2, grid: 4 friction coefficients x 4 masses (Iz scaled with the mass) as one batch of `batch` controllers (vehicle = controller
mod 16): per vehicle, mean / minimum length of every LMPC lap, unsolved steps and controllers with health flags.
Both legs run in the independent mode: the pooled exchange hands laps between controllers whatever their car, and a lap another car
drove is not a feasible trajectory of this one.

  python benchmarks/vehicle_sweep.py [--rounds 5 --batch 8192 --laps 3] [--out FILE]
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
from racinglmpc_b200.reference_params import VehicleParams      # noqa: E402
from param_sweep import card                                    # noqa: E402
import rollout_mc                                               # noqa: E402

SAME = ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt",
        "flags_or", "unsolved", "status", "iters")


def leg_ab(rounds, batch, laps, dev):
    arms = {"no_sets": None, "one_set": ([VehicleParams.reference()], np.zeros(batch, np.int32))}
    rate = {name: [] for name in arms}
    first = {}
    for _ in range(rounds):
        for name, vs in arms.items():
            fin = {}
            out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, final=fin, books=fin, vehicle_sets=vs)
            rate[name].append(out["controller_steps_per_s"])
            if name not in first:
                first[name] = (out["lap_stats_rank0"], fin)
    (st_a, fa), (st_b, fb) = first["no_sets"], first["one_set"]
    assert st_a == st_b, (st_a, st_b)
    for k in SAME:
        assert np.array_equal(fa[k], fb[k]), k
    a, b = np.array(rate["no_sets"]), np.array(rate["one_set"])
    d = 100.0 * (b / a - 1.0)
    return {"benchmark": "vehicle_sweep leg 1: closed loop without vehicle sets vs the reference vehicle as one set", **card(dev),
            "batch": batch, "laps": laps, "mode": "independent", "rounds": rounds,
            "controller_steps_per_s": {"no_sets": a.tolist(), "one_set": b.tolist()},
            "one_set_over_no_sets_pct_rounds": d.tolist(),
            "one_set_over_no_sets_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
            "no_sets_round_spread_pct": float(100.0 * (a.max() - a.min()) / a.mean()),
            "identical": list(SAME), "lap_stats_rank0": st_a}


def vehicle_grid():
    """4 friction coefficients x 4 masses around the reference's car; the yaw inertia scales with the mass."""
    vs, labels = [], []
    for mu in (0.4, 0.6, 0.8, 1.0):
        for s in (0.8, 1.0, 1.2, 1.4):
            vs.append(VehicleParams.from_friction(mu, m=s * 1.98, Iz=s * 0.024))
            labels.append({"mu": mu, "m": s * 1.98, "Iz": s * 0.024})
    return vs, labels


def leg_grid(batch, laps, dev):
    vs, labels = vehicle_grid()
    idx = np.arange(batch) % len(vs)
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, vehicle_sets=(vs, idx))
    for s, lab in zip(out["per_vehicle_rank0"], labels):
        s.update(lab)
    out.pop("benchmark")
    return {"benchmark": "vehicle_sweep leg 2: closed-loop LMPC over a 4 friction x 4 mass vehicle grid, independent mode", **card(dev),
            "vehicles": len(vs), "controllers_per_vehicle": batch // len(vs), **out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of leg 1")
    ap.add_argument("--batch", type=int, default=8192, help="controllers per run")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps every controller drives")
    ap.add_argument("--legs", default="1,2")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args()
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    lines = []
    if "1" in args.legs.split(","):
        lines.append(leg_ab(args.rounds, args.batch, args.laps, dev))
    if "2" in args.legs.split(","):
        lines.append(leg_grid(args.batch, args.laps, dev))
    for r in lines:
        print(json.dumps(r), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
