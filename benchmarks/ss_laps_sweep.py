#!/usr/bin/env python
"""Safe-set lap-count sweeps in one batch (lmpc_set_ss_laps): what per-controller lap counts cost, how LMPC's laps depend on how
the safe set is split between laps (numSS_it) and points per lap at each safe-set size, and what one mixed batch saves over one
handle per lap count.

Leg 1, A/B: benchmarks/rollout_mc.run (PID lap, seeding, `laps` LMPC laps; independent mode) in alternating rounds in the same
process, with
  no_table   no lap-count table (the handle's numSS_it = 4 everywhere);
  one_value  4 installed as the only lap count, with an index for every controller (K2's table instantiation and the
             lap-book kernels that read the table).
Per round: controller steps/s of the LMPC laps (device events).  Both arms must drive the same closed loop: their lap books, end
states, health counters and interior-point iterations are asserted identical.
Leg 2, grid: numSS_it in {1, 2, 3, 4} x numSS_Points in {24, 48, 96} at N = 12 (12 cells, one (12, 96) handle, the safe-set size
through shape_sets, the lap count through ss_laps_sets); cell = controller mod 12, noise streams controller // 12, so the cells
meet the same noise (common random numbers), independent mode: per cell, mean / minimum length of every LMPC lap, unsolved
steps, flagged controllers and the mean interior-point iterations sampled at the polls.
Leg 3, payoff: the wall time (host clock around rollout_mc.run, PID lap and seeding included) of the four lap counts at the
handle's (12, 48) as one mixed batch against one run per lap count, one after the other, with the same controllers (batch / 4
each, same noise streams).

  python benchmarks/ss_laps_sweep.py [--rounds 3 --batch 2048 --laps 3] [--legs 1,2,3] [--out FILE]
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

SAME = ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt", "sel",
        "is_prev", "prev_slot", "used", "flags_or", "unsolved", "status", "iters")
VALUES = (1, 2, 3, 4)
POINTS = (24, 48, 96)
CELLS = [(v, m) for v in VALUES for m in POINTS]


def _spread(a):
    return float(100.0 * (a.max() - a.min()) / a.mean())


def leg_ab(rounds, batch, laps, dev):
    arms = {"no_table": {}, "one_value": dict(ss_laps_sets=([4], np.zeros(batch, np.int32)))}
    rate = {name: [] for name in arms}
    first = {}
    for _ in range(rounds):
        for name, kw in arms.items():
            fin = {}
            out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, final=fin, books=fin, **kw)
            rate[name].append(out["controller_steps_per_s"])
            if name not in first:
                first[name] = (out["lap_stats_rank0"], fin)
    (st_a, fa), (st_b, fb) = first["no_table"], first["one_value"]
    assert st_a == st_b, (st_a, st_b)
    for k in SAME:
        assert np.array_equal(fa[k], fb[k]), k
    a, b = np.array(rate["no_table"]), np.array(rate["one_value"])
    d = 100.0 * (b / a - 1.0)
    return {"benchmark": "ss_laps_sweep leg 1: closed loop without a lap-count table vs the handle's numSS_it = 4 as one value",
            **card(dev), "batch": batch, "laps": laps, "mode": "independent", "rounds": rounds,
            "controller_steps_per_s": {"no_table": a.tolist(), "one_value": b.tolist()},
            "one_value_over_no_table_pct_rounds": d.tolist(),
            "one_value_over_no_table_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
            "no_table_round_spread_pct": _spread(a), "one_value_round_spread_pct": _spread(b),
            "identical": list(SAME), "lap_stats_rank0": st_a}


def leg_grid(batch, laps, dev):
    K = len(CELLS)
    b = np.arange(batch)
    cell = b % K
    shapes = [(12, m) for m in POINTS]
    sidx = np.array([POINTS.index(CELLS[k][1]) for k in cell])
    lidx = np.array([VALUES.index(CELLS[k][0]) for k in cell])
    t0 = time.perf_counter()
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, shape_sets=(shapes, sidx),
                         ss_laps_sets=(list(VALUES), lidx), noise_streams=b // K)
    wall = time.perf_counter() - t0
    per = out["per_shape_ss_laps_rank0"]
    for st in per:
        st.update(points_per_lap=st["numSS_Points"] // st["numSS_it"],
                  finished_every_lap=all(l["n"] == st["controllers"] for l in st["laps"]))
    res = {"benchmark": "ss_laps_sweep leg 2: closed-loop LMPC over numSS_it x numSS_Points at N = 12 in one batch, common noise "
                        "streams (controller // cells), independent mode", **card(dev), "batch": batch, "laps": laps,
           "wall_s": wall, "per_cell": per}
    res.update({k: out[k] for k in ("closed_loop_steps", "ms_total", "controller_steps_per_s", "handle_shape", "lap_stats_rank0",
                                    "instances_with_flags_rank0", "flag_bits_rank0", "unsolved_steps_rank0")})
    return res


def leg_payoff(batch, laps, dev):
    K = len(VALUES)
    b = np.arange(batch)
    t0 = time.perf_counter()
    mixed = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, ss_laps_sets=(list(VALUES), b % K),
                           noise_streams=b // K)
    wall_mixed = time.perf_counter() - t0
    sep, walls = [], []
    for k, v in enumerate(VALUES):
        streams = (b // K)[b % K == k]
        t0 = time.perf_counter()
        out = rollout_mc.run(batch=streams.size, laps=laps, mode="independent", local=dev,
                             ss_laps_sets=([v], np.zeros(streams.size, np.int32)), noise_streams=streams)
        walls.append(time.perf_counter() - t0)
        sep.append(out["per_ss_laps_rank0"][0])
    same = all(m["laps"] == s["laps"] and m["unsolved_steps"] == s["unsolved_steps"]
               for m, s in zip(mixed["per_ss_laps_rank0"], sep))
    return {"benchmark": "ss_laps_sweep leg 3: four lap counts at (12, 48) as one mixed batch vs one run per lap count, one after "
                         "the other", **card(dev), "batch": batch, "laps": laps, "values": list(VALUES), "mixed_wall_s": wall_mixed,
            "separate_wall_s": walls, "separate_wall_s_total": float(sum(walls)), "separate_over_mixed": float(sum(walls) / wall_mixed),
            "mixed_closed_loop_ms": mixed["ms_total"], "per_value_lap_stats_equal": same,
            "per_ss_laps": mixed["per_ss_laps_rank0"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of leg 1")
    ap.add_argument("--batch", type=int, default=2048, help="controllers per run")
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
