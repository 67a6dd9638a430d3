#!/usr/bin/env python
"""Controller snapshots (BatchedController.snapshot / restore, rollout_mc.run(capture=, start=)): what they cost at size and what
they make possible.

Leg 1, cost: pack and unpack every controller of a configs[3]-sized handle (8 192 controllers, Tmax 1280, ss_cap 7, model_cap 5,
Tcl 1024).  Device-event milliseconds per call over --calls calls after a warm-up; the bytes each call reads and writes
(computed from the record layout); the rate against the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM (a bound, not a
target).  An unpack's time includes its check kernel and the host's read of the verdict.
Leg 2, resume at size: a pooled run to 5 laps against a run to 3 laps that is captured, destroyed and resumed to 5 on a fresh
handle.  Whether books, end states, health and exchange steps are identical, and the capture and restore times.
Leg 3, learn once, evaluate many: 64 learners drive 3 pooled LMPC laps on the reference car; each is restored into 128
controllers of an 8 192-controller handle, those split over friction 0.6 / 0.8 / 1.0 (set_vehicles), and all drive 2 more laps
in the independent mode under fresh Philox noise.  Per friction: mean lap 4 and 5, the spread among the clones of one learner
(standard deviation within a learner, averaged over learners) and between learners (standard deviation of the learners' means).

  python benchmarks/snapshot.py [--calls 20] [--out FILE]
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
from racinglmpc_b200 import workloads, reference_params as rp                 # noqa: E402
from racinglmpc_b200 import _native as nat                                    # noqa: E402
from racinglmpc_b200.controller import BatchedController                      # noqa: E402
from param_sweep import card                                                 # noqa: E402
from vehicle_sweep import SAME                                               # noqa: E402
import rollout_mc                                                            # noqa: E402

HBM_TBPS = 3.35        # H100 SXM data sheet
FRICTION = (0.6, 0.8, 1.0)


def configs3(B, dev):
    """Controllers of rollout_mc.run's layout (configs[3] sizes), with a rollout."""
    rm = rollout_mc
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(rm.N_HORIZON)
    c = BatchedController(par, B, workloads.track_seg_table(), rp.TRACK_LENGTH, trToUse=rm.TR_TO_USE, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=Qts, device=dev, Tmax=rm.TMAX, ss_cap=rm.SS_CAP, model_cap=rm.MODEL_CAP)
    c.enable_rollout(Tcl=rm.TCL)
    return c


def leg_cost(B, calls, dev):
    c = configs3(B, dev)
    x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (B, 1))
    c.rollout_set_state(x0, x0)
    for _ in range(1000):                               # the records hold a learned state: PID lap and seeding
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    nbytes = c.snapshot_bytes
    rec = torch.empty((B, nbytes), dtype=torch.uint8, device=torch.device("cuda", dev))
    hdr = nat.decode_snapshot_header(c.snapshot(out=rec)[0, :1024].cpu().numpy())
    payload = sum(nb for _, nb in hdr["sections"].values())
    stream = torch.cuda.ExternalStream(c.stream, device=torch.device("cuda", dev))
    out = {"record_bytes": nbytes, "payload_bytes_per_record": payload, "sections": len(hdr["sections"])}
    for name, call in (("pack", lambda: c.snapshot(out=rec)), ("unpack", lambda: c.restore(rec))):
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        ms = []
        for _ in range(calls):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            call()
            e1.record(stream)
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        # bytes each call reads and writes: every section once each way, plus the header and track row the pack writes (the
        # unpack's check reads the header words and the index fields: counted as part of the payload read, a slight undercount)
        moved = 2 * B * (payload + (784 if name == "pack" else 0))
        best, med = min(ms), float(np.median(ms))
        out[name] = {"ms_median": med, "ms_min": best, "ms_max": max(ms), "calls": calls, "bytes_moved": moved,
                     "gb_s_median": moved / (med * 1e-3) / 1e9, "share_of_hbm_bound_median": moved / (HBM_TBPS * 1e12) / (med * 1e-3),
                     "hbm_bound_ms": moved / (HBM_TBPS * 1e12) * 1e3}
    c.close()
    return out


def leg_resume(B, dev):
    fin5, bk5, cap5 = {}, {}, {}
    o5 = rollout_mc.run(batch=B, laps=5, local=dev, final=fin5, books=bk5, capture=cap5)     # capture: the exchange steps
    cap = {}
    o3 = rollout_mc.run(batch=B, laps=3, local=dev, capture=cap)
    fin, bk, capr = {}, {}, {}
    o = rollout_mc.run(batch=B, laps=5, local=dev, start=cap, final=fin, books=bk, capture=capr)
    same = [k for k in SAME if k in bk5 or k in fin5]
    ident = {k: bool(np.array_equal((bk5 if k in bk5 else fin5)[k], (bk if k in bk else fin)[k])) for k in same}
    ident["closed_loop_steps"] = o5["closed_loop_steps"] == o["closed_loop_steps"]
    ident["exchange_steps"] = cap5["exchange_steps"] == capr["exchange_steps"]
    ident["records"] = bool(torch.equal(cap5["records"], capr["records"]))
    return {"batch": B, "mode": "pooled", "captured_at_step": cap["steps"], "steps_uninterrupted": o5["closed_loop_steps"],
            "steps_resumed": o["closed_loop_steps"], "identical": ident, "all_identical": all(ident.values()),
            "exchange_steps_uninterrupted": cap5["exchange_steps"], "exchange_steps_resumed": capr["exchange_steps"],
            "resume_exact": o["resume_exact"], "capture_s": cap["capture_s"], "restore_s": o["restore_s"],
            "record_bytes": int(cap["records"].shape[1]), "lap_stats_uninterrupted": o5["lap_stats_rank0"],
            "lap_stats_resumed": o["lap_stats_rank0"], "controller_steps_per_s_3_laps": o3["controller_steps_per_s"]}


def leg_evaluate(learners, clones, dev, seed=98765):
    cap = {}
    rollout_mc.run(batch=learners, laps=3, local=dev, capture=cap)
    B = learners * clones
    c = configs3(B, dev)
    learner = np.repeat(np.arange(learners), clones).astype(np.int32)
    mu_idx = np.tile(np.arange(clones) % len(FRICTION), learners).astype(np.int32)
    c.set_vehicles([rp.VehicleParams.from_friction(m) for m in FRICTION], mu_idx)
    t0 = time.perf_counter()
    c.restore(cap["records"], np.arange(B, dtype=np.int32), learner)
    c.rollout_clock = int(cap["clock"])
    c.sync()
    restore_s = time.perf_counter() - t0
    start_laps = c.books()["lap_n"].copy()
    steps = 0
    while steps < 900:
        c.rollout_step(seed=seed)
        c.rollout_commit_laps_dev()
        steps += 1
        if steps % 8 == 0 and c.rollout_stats()[0] >= 5:
            break
    bk = c.books()
    flags, unsolved = c.rollout_health()
    rows = []
    for k, mu in enumerate(FRICTION):
        cell = {"mu": mu, "controllers": int((mu_idx == k).sum())}
        for lap in (4, 5):
            ok = (mu_idx == k) & (bk["lap_n"] >= lap)
            t = bk["lap_hist"][:, lap - 1].astype(float)
            means, within = [], []
            for l in range(learners):
                m = ok & (learner == l)
                if m.sum() >= 2:
                    means.append(t[m].mean())
                    within.append(t[m].std())
            cell["lap%d" % lap] = {"n": int(ok.sum()), "mean": float(t[ok].mean()) if ok.any() else None,
                                   "spread_within_learner": float(np.mean(within)) if within else None,
                                   "spread_between_learners": float(np.std(means)) if means else None}
        cell["unsolved_steps"] = int(unsolved[mu_idx == k].sum())
        cell["instances_with_flags"] = int((flags[mu_idx == k] != 0).sum())
        rows.append(cell)
    c.close()
    return {"learners": learners, "clones_per_learner": clones, "batch": B, "learner_laps": 3, "laps_at_restore_min": int(start_laps.min()),
            "laps_at_restore_max": int(start_laps.max()), "steps_after_restore": steps, "restore_s": restore_s, "per_friction": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--learners", type=int, default=64)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = 0
    torch.cuda.set_device(dev)
    lines = []
    info = card(dev)
    lines.append(dict(benchmark="snapshot leg 1: pack / unpack cost at configs[3] sizes", batch=args.batch, **info,
                      **leg_cost(args.batch, args.calls, dev)))
    print(json.dumps(lines[-1]), flush=True)
    lines.append(dict(benchmark="snapshot leg 2: 3 laps captured and resumed to 5 against a run to 5", **info,
                      **leg_resume(args.batch, dev)))
    print(json.dumps(lines[-1]), flush=True)
    lines.append(dict(benchmark="snapshot leg 3: learn once, evaluate many", **info,
                      **leg_evaluate(args.learners, args.batch // args.learners, dev)))
    print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, "a") as f:
            for l in lines:
                f.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
