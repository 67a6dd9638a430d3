#!/usr/bin/env python
"""Circuit sweeps in one batch (lmpc_set_tracks): what per-controller tracks cost, and a closed-loop track x friction grid.

Leg 1, A/B: benchmarks/rollout_mc.run (PID lap, seeding, `laps` LMPC laps; independent mode) in alternating rounds in the same
process, with
  no_sets   no track table installed (every kernel reads the track of lmpc_store_create from the handle's one-row table);
  one_set   the reference's L-shaped track installed as the only set, with an index for every controller.
Per round: controller steps/s of the LMPC laps (device events).  Both arms must drive the same closed loop: their lap books, end
states and health counters are asserted identical.
Leg 2, grid: the three circuits of Track.py (L-shaped, goggle, oval) x 3 friction coefficients as one batch of `batch`
controllers (track = controller mod 3, friction = (controller // 3) mod 3): per cell, mean / minimum length of every LMPC lap,
unsolved steps and controllers with health flags.
Both legs run in the independent mode: a lap of another circuit is not a trajectory of this one.

  python benchmarks/track_sweep.py [--rounds 5 --batch 8192 --laps 3] [--out FILE]
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
from racinglmpc_b200.reference_params import TrackParams, VehicleParams      # noqa: E402
from param_sweep import card                                                 # noqa: E402
from vehicle_sweep import SAME                                               # noqa: E402
import rollout_mc                                                            # noqa: E402

TRACKS = (("L-shaped", TrackParams.l_shaped), ("goggle", TrackParams.goggle), ("oval", TrackParams.oval))
FRICTION = (0.6, 0.8, 1.0)


def leg_ab(rounds, batch, laps, dev):
    arms = {"no_sets": None, "one_set": ([TrackParams.l_shaped()], np.zeros(batch, np.int32))}
    rate = {name: [] for name in arms}
    first = {}
    for _ in range(rounds):
        for name, ts in arms.items():
            fin = {}
            out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, final=fin, books=fin, track_sets=ts)
            rate[name].append(out["controller_steps_per_s"])
            if name not in first:
                first[name] = (out["lap_stats_rank0"], fin)
    (st_a, fa), (st_b, fb) = first["no_sets"], first["one_set"]
    assert st_a == st_b, (st_a, st_b)
    for k in SAME:
        assert np.array_equal(fa[k], fb[k]), k
    a, b = np.array(rate["no_sets"]), np.array(rate["one_set"])
    d = 100.0 * (b / a - 1.0)
    return {"benchmark": "track_sweep leg 1: closed loop without track sets vs the reference track as one set", **card(dev),
            "batch": batch, "laps": laps, "mode": "independent", "rounds": rounds,
            "controller_steps_per_s": {"no_sets": a.tolist(), "one_set": b.tolist()},
            "one_set_over_no_sets_pct_rounds": d.tolist(),
            "one_set_over_no_sets_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
            "no_sets_round_spread_pct": float(100.0 * (a.max() - a.min()) / a.mean()),
            "identical": list(SAME), "lap_stats_rank0": st_a}


def leg_grid(batch, laps, dev):
    ts = [make() for _, make in TRACKS]
    vs = [VehicleParams.from_friction(mu) for mu in FRICTION]
    b = np.arange(batch)
    t_idx, v_idx = b % len(ts), (b // len(ts)) % len(vs)
    fin = {}
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, books=fin, track_sets=(ts, t_idx),
                         vehicle_sets=(vs, v_idx))
    cells = []
    for i, (name, _) in enumerate(TRACKS):
        for j, mu in enumerate(FRICTION):
            s = rollout_mc._set_stats(fin, fin["flags_or"], fin["unsolved"], (t_idx == i) & (v_idx == j), laps)
            s.update({"track": name, "TrackLength": ts[i].TrackLength, "mu": mu})
            cells.append(s)
    for k in ("benchmark", "per_track_rank0", "per_vehicle_rank0"):
        out.pop(k)
    return {"benchmark": "track_sweep leg 2: closed-loop LMPC over 3 circuits x 3 friction coefficients, independent mode", **card(dev),
            "cells": cells, **out}


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
