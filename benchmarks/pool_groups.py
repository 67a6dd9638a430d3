#!/usr/bin/env python
"""Pooled safe-set exchange within pool groups (lmpc_set_pool_groups): what grouping costs, and fleet learning per circuit.

Leg 1, A/B: benchmarks/rollout_mc.run in the pooled mode (PID lap, seeding, `laps` LMPC laps, one exchange per lap) in
alternating rounds in the same process, with
  no_groups  no pool groups installed (every controller in group 0);
  one_group  one group holding every controller, installed through lmpc_set_pool_groups.
Per round: controller steps/s of the LMPC laps (device events) and milliseconds per exchange.  Both arms must drive the same
closed loop: their lap books, end states and health counters are asserted identical.
Leg 2, grid: the three circuits of Track.py (L-shaped, goggle, oval) x 3 friction coefficients as one batch of `batch`
controllers (track = controller mod 3, friction = (controller // 3) mod 3), pooled per cell (sharding.design_groups: 9 groups)
against the same batch in the independent mode: per cell, mean / minimum length of every LMPC lap, unsolved steps and
controllers with health flags in both modes, laps filed per group, and the exchange time and bytes with 9 groups.  The exchange
waits for the slowest controller of the whole batch, so the groups on shorter circuits ship a lap from further on
(benchmarks/pool_readiness.py runs the same grid with each group exchanging on its own schedule).

  python benchmarks/pool_groups.py [--rounds 5 --batch 8192 --laps 3] [--out FILE]
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
from racinglmpc_b200 import sharding                                          # noqa: E402
from racinglmpc_b200.reference_params import TrackParams, VehicleParams      # noqa: E402
from param_sweep import card                                                 # noqa: E402
from vehicle_sweep import SAME                                               # noqa: E402
from track_sweep import TRACKS, FRICTION                                     # noqa: E402
import rollout_mc                                                            # noqa: E402


def leg_ab(rounds, batch, laps, dev):
    arms = {"no_groups": None, "one_group": (np.zeros(batch, np.int32), 1)}
    rate = {name: [] for name in arms}
    xms = {name: [] for name in arms}
    first = {}
    for _ in range(rounds):
        for name, pg in arms.items():
            fin = {}
            out = rollout_mc.run(batch=batch, laps=laps, mode="pooled", local=dev, final=fin, books=fin, pool_groups=pg)
            rate[name].append(out["controller_steps_per_s"])
            xms[name].append(out["exchange_ms_each"])
            if name not in first:
                first[name] = (out["lap_stats_rank0"], out["laps_filed_rank0"], fin)
    (st_a, fl_a, fa), (st_b, fl_b, fb) = first["no_groups"], first["one_group"]
    assert st_a == st_b and fl_a == fl_b, (st_a, st_b, fl_a, fl_b)
    for k in SAME:
        assert np.array_equal(fa[k], fb[k]), k
    a, b = np.array(rate["no_groups"]), np.array(rate["one_group"])
    d = 100.0 * (b / a - 1.0)
    return {"benchmark": "pool_groups leg 1: pooled closed loop without groups vs one group holding every controller", **card(dev),
            "batch": batch, "laps": laps, "mode": "pooled", "rounds": rounds,
            "controller_steps_per_s": {"no_groups": a.tolist(), "one_group": b.tolist()},
            "one_group_over_no_groups_pct_rounds": d.tolist(),
            "one_group_over_no_groups_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
            "no_groups_round_spread_pct": float(100.0 * (a.max() - a.min()) / a.mean()),
            "exchange_ms_each": xms, "laps_filed_rank0": fl_a, "identical": list(SAME), "lap_stats_rank0": st_a}


def grid_design(batch):
    """The circuits x frictions grid of leg 2: (tracks, vehicles, track index, vehicle index, pool group per cell, G)."""
    ts = [make() for _, make in TRACKS]
    vs = [VehicleParams.from_friction(mu) for mu in FRICTION]
    b = np.arange(batch)
    t_idx, v_idx = b % len(ts), (b // len(ts)) % len(vs)
    groups, G = sharding.design_groups(t_idx, v_idx)
    return ts, vs, t_idx, v_idx, groups, G


def leg_grid(batch, laps, dev):
    ts, vs, t_idx, v_idx, groups, G = grid_design(batch)
    runs = {}
    for mode in ("independent", "pooled"):
        fin = {}
        out = rollout_mc.run(batch=batch, laps=laps, mode=mode, local=dev, books=fin, track_sets=(ts, t_idx), vehicle_sets=(vs, v_idx),
                             pool_groups=(groups, G) if mode == "pooled" else None)
        runs[mode] = (out, fin)
    pooled = runs["pooled"][0]
    cells = []
    for i, (name, _) in enumerate(TRACKS):
        for j, mu in enumerate(FRICTION):
            sel = (t_idx == i) & (v_idx == j)
            g = int(groups[np.nonzero(sel)[0][0]])
            cell = {"track": name, "TrackLength": ts[i].TrackLength, "mu": mu, "group": g,
                    "laps_filed": pooled["laps_filed_per_group_rank0"][g]}
            for mode, (_, fin) in runs.items():
                cell[mode] = rollout_mc._set_stats(fin, fin["flags_or"], fin["unsolved"], sel, laps)
            cells.append(cell)
    keep = ("controller_steps_per_s", "closed_loop_steps", "exchanges", "exchange_ms_each", "allgather_bytes_per_rank",
            "laps_filed_rank0", "unsolved_steps_rank0", "instances_with_flags_rank0", "late_accepts_rank0", "lap_stats_rank0")
    return {"benchmark": "pool_groups leg 2: 3 circuits x 3 friction coefficients, pooled per cell (%d groups) vs independent" % G,
            **card(dev), "batch": batch, "laps": laps, "pool_groups": G, "cells": cells,
            **{mode: {k: out[k] for k in keep} for mode, (out, _) in runs.items()}}


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
