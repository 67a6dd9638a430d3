#!/usr/bin/env python
"""Noise sweeps in one batch (lmpc_rollout_set_noise, lmpc_rollout_set_noise_streams): what per-controller noise costs, how LMPC's
learning depends on the noise of the plant and of the PID lap, and how much pairing common random numbers buy.

Leg 1, A/B: benchmarks/rollout_mc.run (PID lap, seeding, `laps` LMPC laps; independent mode) in alternating rounds in the same
process, with
  no_sets   no noise table and no streams installed (the kernels read the handle's one-row default table, stream b = b);
  one_set   the reference's noise installed as the only set, with an index for every controller, plus identity streams.
Per round: controller steps/s of the LMPC laps (device events).  Both arms must drive the same closed loop: their lap books, end
states and health counters are asserted identical.
Leg 2, grid: simulator noise x{0, 1, 10, 100} x PID noise x{0.5, 1} (NoiseParams.scaled) as 8 cells of batch / 8 controllers in
one batch (cell = controller mod 8), independent mode: per cell, mean / minimum length of every LMPC lap (n = controllers that
finished it; a cell whose n falls short did not finish within the run's step limit), unsolved steps and flagged controllers.
Leg 3, common random numbers: two QP tunings (dR x0.5 and x2) interleaved (tuning = controller mod 2), run twice:
  unpaired  streams b (every controller its own noise);
  paired    streams b // 2 (controllers 2i and 2i + 1 share their noise: PID lap, seeded stores and every later draw).
Per LMPC lap: mean lap-length difference tuning 1 - tuning 0 over the pairs (2i, 2i + 1) that finished it, its unpaired
standard error sqrt(var0 / n + var1 / n), its paired standard error std(d) / sqrt(n), and the correlation of the pair's lap lengths.
Every leg runs in the independent mode: the pooled exchange would couple the pairs.

  python benchmarks/noise_sweep.py [--rounds 5 --batch 8192 --laps 3] [--legs 1,2,3] [--out FILE]
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
from racinglmpc_b200 import reference_params as rp               # noqa: E402
from racinglmpc_b200.reference_params import NoiseParams         # noqa: E402
from param_sweep import card                                     # noqa: E402
import rollout_mc                                                # noqa: E402

SAME = ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt",
        "flags_or", "unsolved", "status", "iters")


def leg_ab(rounds, batch, laps, dev):
    arms = {"no_sets": {}, "one_set": dict(noise_sets=([NoiseParams.reference()], np.zeros(batch, np.int32)),
                                           noise_streams=np.arange(batch, dtype=np.int32))}
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
    return {"benchmark": "noise_sweep leg 1: closed loop without noise tables vs the reference noise as one set + identity streams",
            **card(dev), "batch": batch, "laps": laps, "mode": "independent", "rounds": rounds,
            "controller_steps_per_s": {"no_sets": a.tolist(), "one_set": b.tolist()},
            "one_set_over_no_sets_pct_rounds": d.tolist(),
            "one_set_over_no_sets_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
            "no_sets_round_spread_pct": float(100.0 * (a.max() - a.min()) / a.mean()),
            "one_set_round_spread_pct": float(100.0 * (b.max() - b.min()) / b.mean()),
            "identical": list(SAME), "lap_stats_rank0": st_a}


def noise_grid():
    """Simulator noise x{0, 1, 10, 100} x PID noise x{0.5, 1}: sigma and clip scaled, the gain kept."""
    ns, labels = [], []
    for sim in (0.0, 1.0, 10.0, 100.0):
        for pid in (0.5, 1.0):
            ns.append(NoiseParams.scaled(sim, pid))
            labels.append({"sim_scale": sim, "pid_scale": pid})
    return ns, labels


def leg_grid(batch, laps, dev):
    ns, labels = noise_grid()
    idx = np.arange(batch) % len(ns)
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, noise_sets=(ns, idx))
    for s, lab in zip(out["per_noise_rank0"], labels):
        s.update(lab)
        s["finished_every_lap"] = all(l["n"] == s["controllers"] for l in s["laps"])
    out.pop("benchmark")
    return {"benchmark": "noise_sweep leg 2: closed-loop LMPC over simulator noise x{0,1,10,100} x PID noise x{0.5,1}, independent mode",
            **card(dev), "cells": len(ns), "controllers_per_cell": batch // len(ns), **out}


def pair_stats(bk, laps):
    """Per LMPC lap, over the pairs (2i, 2i + 1) that both finished it: mean of d = lap(2i + 1) - lap(2i), its unpaired and paired
    standard errors, and the correlation of the two lap lengths."""
    h, n = bk["lap_hist"], bk["lap_n"]
    rows = []
    for r in range(laps):
        ok = (n[0::2] > r) & (n[1::2] > r)
        a, b = h[0::2, r][ok].astype(float), h[1::2, r][ok].astype(float)
        d = b - a
        k = int(ok.sum())
        rows.append({"lap": r + 1, "pairs": k, "mean_tuning0": float(a.mean()), "mean_tuning1": float(b.mean()),
                     "mean_diff": float(d.mean()),
                     "se_unpaired": float(np.sqrt(a.var(ddof=1) / k + b.var(ddof=1) / k)),
                     "se_paired": float(d.std(ddof=1) / np.sqrt(k)),
                     "pair_correlation": float(np.corrcoef(a, b)[0, 1])})
    return rows


def leg_crn(batch, laps, dev):
    _, _, _, _, _, base = rp.lmpc_params(rollout_mc.N_HORIZON)
    ps = []
    for s in (0.5, 2.0):
        p = copy.deepcopy(base)
        p.dR = s * np.asarray(base.dR, float)
        ps.append(p)
    pidx = np.arange(batch) % 2
    out = {"benchmark": "noise_sweep leg 3: two QP tunings (dR x0.5, x2) interleaved, unpaired (streams b) vs paired (streams b // 2)",
           **card(dev), "batch": batch, "laps": laps, "mode": "independent", "tunings": ["dR x0.5", "dR x2"]}
    for name, streams in (("unpaired", None), ("paired", np.arange(batch) // 2)):
        bk = {}
        o = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, books=bk, param_sets=(ps, pidx, None),
                           noise_streams=streams)
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
