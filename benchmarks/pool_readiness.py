#!/usr/bin/env python
"""Per-group readiness of the pooled exchange (rollout_mc.run(readiness="group")): what it costs, and what it does for
circuits that lap at different speeds.

Leg 1, A/B: benchmarks/rollout_mc.run in the pooled mode without pool groups, readiness "batch" against "group", in alternating
rounds in the same process.  Without groups both make the same decisions at the same steps: lap books, end states and health
counters are asserted identical.  Per round: controller steps/s of the LMPC laps (device events); then the host time of one
progress poll in each form (the stats call, the readiness rule and, for "group", the agreement vector) on a seeded handle,
without groups and with the 9 groups of leg 2.
Leg 2, grid: the three circuits of Track.py x 3 friction coefficients of benchmarks/pool_groups.py leg 2, pooled per cell
(9 groups), run with "batch" readiness (every group exchanges round r once the slowest controller of the whole batch is
`ship_after` steps into lap r + 1), with "group" readiness (each group once its own slowest controller is) and in the
independent mode.  Per cell: mean / minimum length of every LMPC lap, the closed-loop steps at which the group exchanged, laps
filed, unsolved steps and controllers with health flags.

  python benchmarks/pool_readiness.py [--rounds 5 --batch 8192 --laps 3] [--out FILE]
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
from racinglmpc_b200 import workloads, sharding, reference_params as rp      # noqa: E402
from racinglmpc_b200.controller import BatchedController                      # noqa: E402
from param_sweep import card                                                 # noqa: E402
from vehicle_sweep import SAME                                               # noqa: E402
from track_sweep import TRACKS, FRICTION                                     # noqa: E402
from pool_groups import grid_design                                          # noqa: E402
import rollout_mc                                                            # noqa: E402


def poll_cost(batch, dev, groups=None, reps=400, laps=3, ship_after=40):
    """Host microseconds per progress poll on a seeded handle of `batch` controllers (reps polls each, after a warm-up):
    "batch" = rollout_stats + the rule on its row, "group" = rollout_group_stats + the rule per row + the agreement vector."""
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(12)
    c = BatchedController(par, batch, workloads.track_seg_table(), rp.TRACK_LENGTH, trToUse=4, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=Qts, device=dev, Tmax=1280, ss_cap=7, model_cap=5)
    if groups is not None:
        c.set_pool_groups(*groups)
    x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (batch, 1))
    c.enable_rollout(Tcl=1024)
    c.rollout_set_state(x0, x0)
    for _ in range(100):                                 # the polls read the books and the record: a short PID lap will do
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.sync()
    nxt = np.ones(c.pool_groups, np.int64)
    live = np.ones(c.pool_groups, bool)
    gpu = torch.device("cuda", dev)

    def batch_poll():
        st = np.array([c.rollout_stats()])
        return sharding.ready_groups(st, 1, laps, ship_after)[0], st[0, 0] >= laps

    def group_poll():
        st = c.rollout_group_stats()
        return sharding.agree_groups(sharding.ready_groups(st, nxt, laps, ship_after) & live, st[:, 0].min() >= laps, gpu)
    us = {}
    for name, f in (("batch", batch_poll), ("group", group_poll)):
        for _ in range(20):
            f()
        t = time.perf_counter()
        for _ in range(reps):
            f()
        us[name] = 1e6 * (time.perf_counter() - t) / reps
    c.close()
    return us


def leg_ab(rounds, batch, laps, dev):
    arms = ("batch", "group")
    rate = {name: [] for name in arms}
    first = {}
    for _ in range(rounds):
        for name in arms:
            fin = {}
            out = rollout_mc.run(batch=batch, laps=laps, mode="pooled", local=dev, final=fin, books=fin, readiness=name)
            rate[name].append(out["controller_steps_per_s"])
            if name not in first:
                first[name] = (out, fin)
    (oa, fa), (ob, fb) = first["batch"], first["group"]
    for k in ("lap_stats_rank0", "laps_filed_rank0", "exchanges", "closed_loop_steps"):
        assert oa[k] == ob[k], (k, oa[k], ob[k])
    for k in SAME:
        assert np.array_equal(fa[k], fb[k]), k
    a, b = np.array(rate["batch"]), np.array(rate["group"])
    d = 100.0 * (b / a - 1.0)
    *_, groups, G = grid_design(batch)
    polls = {"no_groups": poll_cost(batch, dev), "9_groups": poll_cost(batch, dev, groups=(groups, G))}
    return {"benchmark": "pool_readiness leg 1: pooled closed loop without groups, readiness batch vs group", **card(dev),
            "batch": batch, "laps": laps, "mode": "pooled", "rounds": rounds,
            "controller_steps_per_s": {"batch": a.tolist(), "group": b.tolist()},
            "group_over_batch_pct_rounds": d.tolist(),
            "group_over_batch_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
            "batch_round_spread_pct": float(100.0 * (a.max() - a.min()) / a.mean()),
            "group_round_spread_pct": float(100.0 * (b.max() - b.min()) / b.mean()),
            "poll_us": polls, "polls_per_run": oa["closed_loop_steps"] // oa["poll_every"], "exchanges": oa["exchanges"],
            "identical": list(SAME) + ["lap_stats_rank0", "laps_filed_rank0", "exchanges", "closed_loop_steps"],
            "lap_stats_rank0": oa["lap_stats_rank0"]}


def leg_grid(batch, laps, dev):
    ts, vs, t_idx, v_idx, groups, G = grid_design(batch)
    runs = {}
    for name, mode, readiness in (("batch", "pooled", "batch"), ("group", "pooled", "group"), ("independent", "independent", "batch")):
        fin = {}
        out = rollout_mc.run(batch=batch, laps=laps, mode=mode, local=dev, books=fin, track_sets=(ts, t_idx), vehicle_sets=(vs, v_idx),
                             pool_groups=(groups, G) if mode == "pooled" else None, readiness=readiness)
        runs[name] = (out, fin)
    cells = []
    for i, (tname, _) in enumerate(TRACKS):
        for j, mu in enumerate(FRICTION):
            sel = (t_idx == i) & (v_idx == j)
            g = int(groups[np.nonzero(sel)[0][0]])
            cell = {"track": tname, "TrackLength": ts[i].TrackLength, "mu": mu, "group": g}
            for name, (out, fin) in runs.items():
                cell[name] = rollout_mc._set_stats(fin, fin["flags_or"], fin["unsolved"], sel, laps)
                if name != "independent":
                    cell[name]["exchange_steps"] = out["exchange_steps_per_group_rank0"][g]
                    cell[name]["laps_filed"] = out["laps_filed_per_group_rank0"][g]
            cells.append(cell)
    keep = ("controller_steps_per_s", "closed_loop_steps", "exchanges", "exchange_ms_each", "allgather_bytes_per_rank",
            "laps_filed_rank0", "unsolved_steps_rank0", "instances_with_flags_rank0", "late_accepts_rank0", "lap_stats_rank0")
    return {"benchmark": "pool_readiness leg 2: 3 circuits x 3 friction coefficients pooled per cell (%d groups), readiness batch "
                         "vs group, and independent" % G,
            **card(dev), "batch": batch, "laps": laps, "pool_groups": G, "cells": cells,
            **{name: {k: out[k] for k in keep} for name, (out, _) in runs.items()}}


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
