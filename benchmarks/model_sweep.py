#!/usr/bin/env python
"""Regression-model sweeps in one batch (lmpc_set_regression_sets): what per-controller regression constants cost, and how LMPC's
learning depends on the k-NN bandwidth, the neighbour count and the laps the model regresses on.

Leg 1, A/B: benchmarks/rollout_mc.run (PID lap, seeding, `laps` LMPC laps; independent mode) in alternating rounds in the same
process, with
  no_sets   no regression table installed (K1 reads the store's one-row table of the constants of lmpc_store_create);
  one_set   the reference's constants (RegressionParams.reference(4)) installed as the only set, with an index for every controller.
Per round: controller steps/s of the LMPC laps (device events).  Both arms must drive the same closed loop: their lap books, end
states and health counters are asserted identical.
Leg 2, against the parent build (--parent-root: a checkout of the previous commit with its library built): bench.py --config 2
(K1 time from lmpc_step_profile's events, step time) and --config 3 (closed-loop controller steps/s), each with --dump-outputs,
alternating this tree and the parent's in `rounds` rounds (odd rounds parent first); every dumped array of both trees is compared
bit for bit.
Leg 3, grid: h in {0.5, 1, 5, 50} x MaxNumPoint in {3, 7} at trToUse 4, plus trToUse in {1, 2, 4} at the reference's constants,
as 11 cells in one batch (cell = controller mod 11) on noise streams controller // 11, so the cells meet the same noise (common
random numbers), independent mode: per cell, mean / minimum length of every LMPC lap (n = controllers that finished it), unsolved
steps and flagged controllers.

  python benchmarks/model_sweep.py [--rounds 5 --batch 8192 --laps 3] [--legs 1,2,3] [--parent-root DIR] [--out FILE]
Prints one JSON line per leg (card name and power limit read in the same run); --out appends them to FILE as well."""
import argparse
import dataclasses
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
from racinglmpc_b200.reference_params import RegressionParams   # noqa: E402
from param_sweep import card                                     # noqa: E402
import rollout_mc                                                # noqa: E402

SAME = ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt",
        "flags_or", "unsolved", "status", "iters")


def _spread(a):
    return float(100.0 * (a.max() - a.min()) / a.mean())


def leg_ab(rounds, batch, laps, dev):
    arms = {"no_sets": {}, "one_set": dict(regression_sets=([RegressionParams.reference(rollout_mc.TR_TO_USE)],
                                                            np.zeros(batch, np.int32)))}
    rate = {name: [] for name in arms}
    first = {}
    for _ in range(rounds):
        for name, kw in arms.items():
            fin = {}
            out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, final=fin, books=fin, **kw)
            rate[name].append(out["controller_steps_per_s"])
            if name not in first:
                first[name] = (out["lap_stats_rank0"], fin)
    (st_a, fa), (st_b, fb) = first["no_sets"], first["one_set"]
    assert st_a == st_b, (st_a, st_b)
    for k in SAME:
        assert np.array_equal(fa[k], fb[k]), k
    a, b = np.array(rate["no_sets"]), np.array(rate["one_set"])
    d = 100.0 * (b / a - 1.0)
    return {"benchmark": "model_sweep leg 1: closed loop without regression tables vs the reference constants as one set",
            **card(dev), "batch": batch, "laps": laps, "mode": "independent", "rounds": rounds,
            "controller_steps_per_s": {"no_sets": a.tolist(), "one_set": b.tolist()},
            "one_set_over_no_sets_pct_rounds": d.tolist(),
            "one_set_over_no_sets_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
            "no_sets_round_spread_pct": _spread(a), "one_set_round_spread_pct": _spread(b),
            "identical": list(SAME), "lap_stats_rank0": st_a}


def _bench(root, config, dump):
    """One bench.py run of `root`'s tree: its JSON line."""
    cmd = [sys.executable, os.path.join(root, "bench.py"), "--gpus", "1", "--steps", "20", "--warmup", "3", "--config", str(config),
           "--no-cpu-baseline", "--dump-outputs", dump]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=1800)
    if r.returncode != 0:
        raise RuntimeError("bench.py failed in %s:\n%s\n%s" % (root, r.stdout[-3000:], r.stderr[-3000:]))
    return json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])


def _same_dumps(a, b):
    names = sorted(f for f in os.listdir(a) if f.endswith(".npy"))
    assert names and names == sorted(f for f in os.listdir(b) if f.endswith(".npy")), (a, b)
    return names, all(np.array_equal(np.load(os.path.join(a, f)), np.load(os.path.join(b, f))) for f in names)


def leg_parent(rounds, parent_root, dev):
    arms = {"parent": os.path.abspath(parent_root), "this": ROOT}
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(rounds):
            order = ["parent", "this"] if r % 2 == 0 else ["this", "parent"]
            row = {"round": r + 1, "order": order}
            dirs = {}
            for name in order:
                d2, d3 = (os.path.join(tmp, "%s_r%d_c%d" % (name, r, c)) for c in (2, 3))
                j2, j3 = _bench(arms[name], 2, d2), _bench(arms[name], 3, d3)
                c3 = j3["configs"]["configs[3]"] if "configs" in j3 else j3
                row[name] = {"k1_ms": j2["kernels"]["knn_ltv_regress_kernel"]["ms"], "config2_ms_per_step": j2["ms_per_step"],
                             "config3_controller_steps_per_s": c3.get("value")}
                dirs[name] = (d2, d3)
            n2, same2 = _same_dumps(dirs["parent"][0], dirs["this"][0])
            n3, same3 = _same_dumps(dirs["parent"][1], dirs["this"][1])
            row.update(config2_dumps_identical=same2, config3_dumps_identical=same3, config2_dumped=n2, config3_dumped=n3)
            rows.append(row)
    out = {"benchmark": "model_sweep leg 2: bench.py configs[2] (K1 time) and configs[3] of this tree against the parent commit's",
           **card(dev), "rounds": rows}
    for key in ("k1_ms", "config2_ms_per_step", "config3_controller_steps_per_s"):
        a = np.array([r["parent"][key] for r in rows], float)
        b = np.array([r["this"][key] for r in rows], float)
        d = 100.0 * (b / a - 1.0)
        out[key] = {"parent_mean": float(a.mean()), "this_mean": float(b.mean()), "this_over_parent_pct_rounds": d.tolist(),
                    "this_over_parent_pct": float(100.0 * (b.mean() / a.mean() - 1.0)),
                    "parent_round_spread_pct": _spread(a), "this_round_spread_pct": _spread(b)}
    out["all_dumps_identical"] = all(r["config2_dumps_identical"] and r["config3_dumps_identical"] for r in rows)
    return out


def model_grid():
    """h x{0.5, 1, 5, 50} x MaxNumPoint {3, 7} at trToUse 4, then trToUse {1, 2, 4} at the reference's constants."""
    ref = RegressionParams.reference(4)
    regs, labels = [], []
    for h in (0.5, 1.0, 5.0, 50.0):
        for k in (3, 7):
            regs.append(dataclasses.replace(ref, h=h, MaxNumPoint=k))
            labels.append({"h": h, "MaxNumPoint": k, "trToUse": 4})
    for tr in (1, 2, 4):
        regs.append(RegressionParams.reference(tr))
        labels.append({"h": ref.h, "MaxNumPoint": ref.MaxNumPoint, "trToUse": tr})
    return regs, labels


def leg_grid(batch, laps, dev):
    regs, labels = model_grid()
    K = len(regs)
    b = np.arange(batch)
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, regression_sets=(regs, b % K), noise_streams=b // K)
    for s, lab in zip(out["per_regression_rank0"], labels):
        s.update(lab)
        s["finished_every_lap"] = all(l["n"] == s["controllers"] for l in s["laps"])
    out.pop("benchmark")
    return {"benchmark": "model_sweep leg 3: closed-loop LMPC over h x MaxNumPoint (trToUse 4) and trToUse {1,2,4}, common noise "
                         "streams (controller // cells), independent mode",
            **card(dev), "cells": K, "noise_streams": "controller // %d" % K, **out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of legs 1 and 2")
    ap.add_argument("--batch", type=int, default=8192, help="controllers per run")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps every controller drives")
    ap.add_argument("--legs", default="1,3", help="legs to run; leg 2 needs --parent-root")
    ap.add_argument("--parent-root", default="", help="the previous commit's tree with its library built (leg 2)")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args()
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    legs = args.legs.split(",")
    if "2" in legs and not args.parent_root:
        ap.error("leg 2 needs --parent-root")
    for leg, fn in (("1", lambda: leg_ab(args.rounds, args.batch, args.laps, dev)),
                    ("2", lambda: leg_parent(args.rounds, args.parent_root, dev)),
                    ("3", lambda: leg_grid(args.batch, args.laps, dev))):
        if leg not in legs:
            continue
        r = fn()
        print(json.dumps(r), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
