#!/usr/bin/env python
"""Horizon and safe-set size sweeps in one batch (lmpc_set_shapes): what per-controller shapes cost, how LMPC's laps depend on the
horizon N and the safe-set size numSS_Points (the trade-off of Rosolia & Borrelli, TCST 2019), and what one mixed batch saves
over one handle per shape.

Leg 1, A/B: benchmarks/rollout_mc.run (PID lap, seeding, `laps` LMPC laps; independent mode) in alternating rounds in the same
process, with
  no_table   no shape table (the uniform QP kernel at the handle's (12, 48));
  one_shape  (12, 48) installed as the only shape, with an index for every controller (the shaped QP kernel, the handle's
             parameters read from a one-row table).
Per round: controller steps/s of the LMPC laps (device events).  Both arms must drive the same closed loop: their lap books, end
states and health counters are asserted identical.
Leg 2, grid: N in {6, 8, 10, 12, 14} at 48 points and numSS_Points in {24, 32, 64, 96} at N in {12, 14} (13 shapes, handle
(14, 96)), then a 48-point horizon arm N in {6, 8, 10, 12, 14, 16, 20, 24, 32, 48} (handle (48, 48)); shape = controller mod
shapes, noise streams controller // shapes, so the shapes meet the same noise (common random numbers), independent mode: per
shape, mean / minimum length of every LMPC lap, unsolved steps, flagged controllers and the mean interior-point iterations
sampled at the polls.
Leg 3, payoff: the wall time (host clock around rollout_mc.run, PID lap and seeding included) of the grid's 13 shapes as one
mixed batch against one run per shape, one after the other, with the same controllers (batch / 13 each, same noise streams).

  python benchmarks/shape_sweep.py [--rounds 3 --batch 4096 --laps 3] [--legs 1,2,3] [--out FILE]
Prints one JSON line per leg (card name and power limit read in the same run); --out appends them to FILE as well."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "benchmarks")):
    if p not in sys.path:
        sys.path.insert(0, p)
from param_sweep import card                                     # noqa: E402
import rollout_mc                                                # noqa: E402

SAME = ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt",
        "flags_or", "unsolved", "status", "iters")
GRID = [(n, 48) for n in (6, 8, 10, 12, 14)] + [(n, m) for n in (12, 14) for m in (24, 32, 64, 96)]
HORIZONS_48 = [(n, 48) for n in (6, 8, 10, 12, 14, 16, 20, 24, 32, 48)]


def _spread(a):
    return float(100.0 * (a.max() - a.min()) / a.mean())


def leg_ab(rounds, batch, laps, dev):
    arms = {"no_table": {}, "one_shape": dict(shape_sets=([(12, 48)], np.zeros(batch, np.int32)))}
    rate = {name: [] for name in arms}
    first = {}
    for _ in range(rounds):
        for name, kw in arms.items():
            fin = {}
            out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, final=fin, books=fin, **kw)
            rate[name].append(out["controller_steps_per_s"])
            if name not in first:
                first[name] = (out["lap_stats_rank0"], fin)
    (st_a, fa), (st_b, fb) = first["no_table"], first["one_shape"]
    assert st_a == st_b, (st_a, st_b)
    for k in SAME:
        assert np.array_equal(fa[k], fb[k]), k
    a, b = np.array(rate["no_table"]), np.array(rate["one_shape"])
    d = 100.0 * (b / a - 1.0)
    return {"benchmark": "shape_sweep leg 1: closed loop without a shape table vs the handle's (12, 48) as one shape",
            **card(dev), "batch": batch, "laps": laps, "mode": "independent", "rounds": rounds,
            "controller_steps_per_s": {"no_table": a.tolist(), "one_shape": b.tolist()},
            "one_shape_over_no_table_pct_rounds": d.tolist(),
            "one_shape_over_no_table_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
            "no_table_round_spread_pct": _spread(a), "one_shape_round_spread_pct": _spread(b),
            "identical": list(SAME), "lap_stats_rank0": st_a}


def _grid_run(shapes, batch, laps, dev):
    K = len(shapes)
    b = np.arange(batch)
    t0 = time.perf_counter()
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, shape_sets=(shapes, b % K), noise_streams=b // K)
    wall = time.perf_counter() - t0
    for s in out["per_shape_rank0"]:
        s["finished_every_lap"] = all(l["n"] == s["controllers"] for l in s["laps"])
    out.pop("benchmark")
    return out, wall


def leg_grid(batch, laps, dev):
    res = {"benchmark": "shape_sweep leg 2: closed-loop LMPC over N x numSS_Points in one batch, common noise streams "
                        "(controller // shapes), independent mode", **card(dev), "batch": batch, "laps": laps}
    for name, shapes in (("grid", GRID), ("horizons_48_points", HORIZONS_48)):
        out, wall = _grid_run(shapes, batch, laps, dev)
        res[name] = {"shapes": len(shapes), "wall_s": wall, **out}
    return res


def leg_payoff(batch, laps, dev):
    K = len(GRID)
    b = np.arange(batch)
    mixed, wall_mixed = _grid_run(GRID, batch, laps, dev)
    sep, walls = [], []
    for k, shape in enumerate(GRID):
        streams = (b // K)[b % K == k]
        t0 = time.perf_counter()
        out = rollout_mc.run(batch=streams.size, laps=laps, mode="independent", local=dev,
                             shape_sets=([shape], np.zeros(streams.size, np.int32)), noise_streams=streams)
        walls.append(time.perf_counter() - t0)
        sep.append(out["per_shape_rank0"][0])
    same = all(m["laps"] == s["laps"] and m["unsolved_steps"] == s["unsolved_steps"] for m, s in zip(mixed["per_shape_rank0"], sep))
    return {"benchmark": "shape_sweep leg 3: the grid's shapes as one mixed batch vs one run per shape, one after the other",
            **card(dev), "batch": batch, "laps": laps, "shapes": K, "mixed_wall_s": wall_mixed, "separate_wall_s": walls,
            "separate_wall_s_total": float(sum(walls)), "separate_over_mixed": float(sum(walls) / wall_mixed),
            "mixed_closed_loop_ms": mixed["ms_total"], "per_shape_lap_stats_equal": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of leg 1")
    ap.add_argument("--batch", type=int, default=4096, help="controllers per run")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps every controller drives")
    ap.add_argument("--legs", default="1,2,3", help="legs to run")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args()
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    for leg, fn in (("1", lambda: leg_ab(args.rounds, args.batch, args.laps, dev)),
                    ("2", lambda: leg_grid(args.batch, args.laps, dev)),
                    ("3", lambda: leg_payoff(args.batch, args.laps, dev))):
        if leg not in args.legs.split(","):
            continue
        r = fn()
        print(json.dumps(r), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
