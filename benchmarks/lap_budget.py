#!/usr/bin/env python
"""Lap budgets (lmpc_rollout_set_lap_budget): what the feature costs when it does nothing, and what it saves on batches whose
controllers need different numbers of steps.  Every leg runs benchmarks/rollout_mc.run (PID lap, seeding, `laps` LMPC laps;
independent mode) in alternating rounds in one process; times are device events around the LMPC laps.

Leg 1, cost: `batch` controllers on one circuit, no budget against a budget of 16 laps (never reached, so every kernel reads the
  budget and retires nobody): controller steps/s per round; lap books, end states, health counters and the last solver report are
  asserted identical between the arms.
Leg 2, gain on circuits of different length: the L-shaped, goggle and oval circuits x friction 0.6 / 0.8 / 1.0 of
  benchmarks/track_sweep.py, no budget against lap_budget = laps: wall time of the run, batch x steps / s, driven steps / s and
  the steps really driven; the first `laps` laps of every controller are asserted identical between the arms.
Leg 3, gain with cells that never finish: the regression grid of benchmarks/model_sweep.py (the run goes to its 900-step limit).
Leg 4, this tree against another (--parent-root: e.g. the previous commit's tree with its library built): bench.py
  (configs[1], [2], [3], outputs dumped) of each tree, alternating, every dumped array compared bit for bit.

  python benchmarks/lap_budget.py [--legs 1,2,3 --rounds 5 --batch 8192 --laps 3] [--parent-root DIR] [--out FILE]
Prints one JSON line per leg (card name and power limit read in the same run); --out appends them to FILE as well."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "benchmarks")):
    if p not in sys.path:
        sys.path.insert(0, p)
from racinglmpc_b200.reference_params import VehicleParams      # noqa: E402
from param_sweep import card                                     # noqa: E402
from model_sweep import SAME, model_grid                         # noqa: E402
from track_sweep import TRACKS, FRICTION                         # noqa: E402
import rollout_mc                                                # noqa: E402


def _summary(name, a, b, higher_is_better):
    """Arm b against arm a over the rounds: means, per-round ratio and each arm's round-to-round spread."""
    a, b = np.asarray(a, float), np.asarray(b, float)
    d = 100.0 * (b / a - 1.0)
    return {name: {"a": a.tolist(), "b": b.tolist(), "b_over_a_pct_rounds": d.tolist(),
                   "b_over_a_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
                   "a_round_spread_pct": float(100.0 * (a.max() - a.min()) / a.mean()),
                   "b_round_spread_pct": float(100.0 * (b.max() - b.min()) / b.mean()), "higher_is_better": higher_is_better}}


def leg_cost(rounds, batch, laps, dev):
    arms = {"no_budget": None, "budget_16": 16}
    rate, first = {n: [] for n in arms}, {}
    for _ in range(rounds):
        for name, bud in arms.items():
            fin = {}
            out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, final=fin, books=fin, lap_budget=bud)
            rate[name].append(out["controller_steps_per_s"])
            first.setdefault(name, (out["lap_stats_rank0"], out["closed_loop_steps"], fin))
    (st_a, n_a, fa), (st_b, n_b, fb) = first["no_budget"], first["budget_16"]
    assert st_a == st_b and n_a == n_b, (st_a, st_b, n_a, n_b)
    for k in SAME:
        assert np.array_equal(fa[k], fb[k]), k
    return {"benchmark": "lap_budget leg 1: closed loop without a budget (a) vs a budget of 16 laps that is never reached (b)", **card(dev),
            "batch": batch, "laps": laps, "mode": "independent", "rounds": rounds, "closed_loop_steps": n_a,
            **_summary("controller_steps_per_s", rate["no_budget"], rate["budget_16"], True), "identical": list(SAME), "lap_stats_rank0": st_a}


def _gain(title, rounds, batch, laps, dev, kw, cell_of, cell_names, max_steps=0):
    """Alternating rounds of run(**kw) without a budget (a) and with lap_budget = laps (b)."""
    keys = ("ms_total", "controller_steps_per_s")
    got, first = {n: {k: [] for k in keys} for n in ("a", "b")}, {}
    for _ in range(rounds):
        for name, bud in (("a", None), ("b", laps)):
            bk = {}
            out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, books=bk, lap_budget=bud, max_steps=max_steps, **kw)
            for k in keys:
                got[name][k].append(out[k])
            if name == "b":
                got[name].setdefault("driven_steps_per_s", []).append(out["driven_steps_per_s"])
            first.setdefault(name, (out, bk))
    (oa, ba), (ob, bb) = first["a"], first["b"]
    firstlaps = np.where(np.arange(16)[None, :] < np.minimum(ba["lap_n"], laps)[:, None], ba["lap_hist"], -1)[:, :laps]
    assert np.array_equal(firstlaps, np.where(np.arange(16)[None, :] < bb["lap_n"][:, None], bb["lap_hist"], -1)[:, :laps])
    assert bb["lap_n"].max() <= laps
    driven_a = rollout_mc._driven_steps(ba, dict(cl_len=np.zeros(batch, np.int64)))      # laps handed over (the lap under way not read back)
    cells = []
    for i, nm in enumerate(cell_names):
        sel = cell_of == i
        cells.append({"cell": nm, "controllers": int(sel.sum()), "finished_%d_laps" % laps: int((bb["lap_n"][sel] >= laps).sum()),
                      "laps_driven_without_budget_max": int(ba["lap_n"][sel].max()),
                      "filed_lap_steps_mean_with_budget": float(np.where(np.arange(16)[None, :] < bb["lap_n"][sel][:, None],
                                                                  bb["lap_hist"][sel], 0).sum(1).mean()),
                      "first_laps_identical": True})
    return {"benchmark": title, **card(dev), "batch": batch, "laps": laps, "mode": "independent", "rounds": rounds,
            "closed_loop_steps": {"a": oa["closed_loop_steps"], "b": ob["closed_loop_steps"]},
            "controller_steps_stepped": batch * ob["closed_loop_steps"], "driven_controller_steps_with_budget": ob["driven_controller_steps_rank0"],
            "filed_lap_steps_without_budget": driven_a,
            **_summary("ms_total", got["a"]["ms_total"], got["b"]["ms_total"], False),
            **_summary("controller_steps_per_s", got["a"]["controller_steps_per_s"], got["b"]["controller_steps_per_s"], True),
            "driven_steps_per_s_with_budget": got["b"]["driven_steps_per_s"], "cells": cells}


def leg_circuits(rounds, batch, laps, dev):
    ts = [make() for _, make in TRACKS]
    vs = [VehicleParams.from_friction(mu) for mu in FRICTION]
    b = np.arange(batch)
    t_idx, v_idx = b % len(ts), (b // len(ts)) % len(vs)
    names = ["%s, mu %.1f" % (t, mu) for mu in FRICTION for t, _ in TRACKS]
    return _gain("lap_budget leg 2: 3 circuits x 3 friction coefficients, no budget (a) vs lap_budget = laps (b)", rounds, batch, laps, dev,
                 dict(track_sets=(ts, t_idx), vehicle_sets=(vs, v_idx)), v_idx * len(ts) + t_idx, names)


def leg_models(rounds, batch, laps, dev):
    regs, labels = model_grid()
    K = len(regs)
    b = np.arange(batch)
    return _gain("lap_budget leg 3: regression grid of model_sweep (cells that never finish; 900-step limit), no budget (a) vs lap_budget = laps (b)",
                 rounds, batch, laps, dev, dict(regression_sets=(regs, b % K), noise_streams=b // K), b % K, [json.dumps(l) for l in labels],
                 max_steps=300 * laps)


def _bench(root, dump):
    """One default bench.py run (configs[1], [2], [3]) of `root`'s tree: its JSON line."""
    cmd = [sys.executable, os.path.join(root, "bench.py"), "--gpus", "1", "--steps", "20", "--warmup", "3", "--no-cpu-baseline",
           "--dump-outputs", dump]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=1800)
    if r.returncode != 0:
        raise RuntimeError("bench.py failed in %s:\n%s\n%s" % (root, r.stdout[-3000:], r.stderr[-3000:]))
    d = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    return {"c1_ms": d["ms_per_step"], "c2_ms": d["configs"]["configs[2]"]["ms_per_step"],
            "c3_steps_s": d["configs"]["configs[3]"]["controller_steps_per_s"]}


def leg_parent(rounds, parent_root, dev):
    arms = {"parent": os.path.abspath(parent_root), "this": ROOT}
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(rounds):
            order = ["parent", "this"] if r % 2 == 0 else ["this", "parent"]
            row = {"round": r + 1, "order": order}
            for name in order:
                row[name] = _bench(arms[name], os.path.join(tmp, "%s_%d" % (name, r)))
            da, db = (os.path.join(tmp, "%s_%d" % (n, r)) for n in ("parent", "this"))
            names = sorted(f for f in os.listdir(da) if f.endswith(".npy"))
            assert names and names == sorted(f for f in os.listdir(db) if f.endswith(".npy"))
            row["dumped_arrays"] = len(names)
            row["bit_identical"] = all(np.array_equal(np.load(os.path.join(da, f)), np.load(os.path.join(db, f))) for f in names)
            rows.append(row)
    out = {"benchmark": "lap_budget leg 4: bench.py configs[1], [2], [3] of this tree (b) against the parent tree (a)", **card(dev),
           "rounds": rows, "all_dumps_identical": all(r["bit_identical"] for r in rows)}
    for key, hib in (("c1_ms", False), ("c2_ms", False), ("c3_steps_s", True)):
        out.update(_summary(key, [r["parent"][key] for r in rows], [r["this"][key] for r in rows], hib))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of every leg")
    ap.add_argument("--batch", type=int, default=8192, help="controllers per run")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps every controller drives")
    ap.add_argument("--legs", default="1,2,3", help="legs to run; leg 4 needs --parent-root")
    ap.add_argument("--parent-root", default="", help="the tree to compare this one against, with its library built (leg 4)")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args()
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    legs = args.legs.split(",")
    if "4" in legs and not args.parent_root:
        ap.error("leg 4 needs --parent-root")
    for leg, fn in (("1", lambda: leg_cost(args.rounds, args.batch, args.laps, dev)),
                    ("2", lambda: leg_circuits(args.rounds, args.batch, args.laps, dev)),
                    ("3", lambda: leg_models(args.rounds, args.batch, args.laps, dev)),
                    ("4", lambda: leg_parent(args.rounds, args.parent_root, dev))):
        if leg not in legs:
            continue
        r = fn()
        print(json.dumps(r), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
