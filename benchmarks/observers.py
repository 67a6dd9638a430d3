#!/usr/bin/env python
"""State observers in one batch (lmpc_rollout_set_observers): what the observer kernel costs, and whether filtering the noisy
measurement with the controller's own one-step prediction lets LMPC's learning survive sensor noise.

Every leg drives its own loop on BatchedController (independent mode, the controllers and constants of rollout_mc): PID lap,
rollout_seed_from_record_dev, then rollout_step + rollout_commit_laps_dev until every controller has driven `laps` LMPC laps
(polled every 8 steps) or 300 steps per lap have passed, with lap reports on.
Leg 1, A/B: alternating rounds of no observer table against a table of all-ones rows (the observer kernel runs every step and
copies y) under the base measurement noise.  Per round: controller steps/s of the LMPC laps (device events).  Both arms must drive
the same closed loop: books, end states, health counters, the last solver report and the lap reports are asserted identical.
Leg 2, kernel time: observe_kernel (and measure_kernel beside it) over many launches under torch.profiler with CUDA activities,
uniform gain 0.5, at the batch of leg 1.
Leg 3, study: measurement noise x{0, 1, 3, 10} of the base set (measurement_noise.py) crossed with four observers -- none,
uniform 0.5, uniform 0.2 and "matched" (ObserverParams.from_noise with model_sigma the per-channel RMS of y_{k+1} - p measured in
a pilot run of the x0 cell without observer, meas_sigma the cell's sigma) -- as 16 cells of `study_batch` / 16 controllers,
controller j of every cell on noise stream j.  Per cell: controllers that finished every lap, mean steps of laps 1, 5, 10 and 20,
unsolved QPs, controllers with flag bit 1 and with LMPC_FLAG_OBSERVER_RESET, the share whose last lap left the lane, and per
channel the RMS of x_est - x against that of y - x sampled at the polls.

  python benchmarks/observers.py [--rounds 3 --batch 8192 --laps 3 --study-batch 4096 --study-laps 20] [--legs 1,2,3] [--out F]
Prints one JSON line per leg (card name and power limit read in the same run); --out appends them to F as well."""
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
from racinglmpc_b200 import reference_params as rp, workloads                  # noqa: E402
from racinglmpc_b200 import _native as nat                                      # noqa: E402
from racinglmpc_b200.controller import BatchedController                        # noqa: E402
from racinglmpc_b200.reference_params import MeasurementParams, ObserverParams  # noqa: E402
from param_sweep import card                                                    # noqa: E402
import rollout_mc as rm                                                         # noqa: E402

BASE = MeasurementParams((0.01, 0.01, 0.01, 0.005, 0.01, 0.01), (0.05, 0.05, 0.05, 0.025, 0.05, 0.05))
CHANNELS = ("vx", "vy", "wz", "epsi", "s", "ey")
POLL = 8


def controller(B, dev, laps, meas, obs=None, streams=None):
    """rollout_mc's controller with reports for `laps` laps, measurement table meas = (rows, index) and observer table obs."""
    N, M, numSS_it = rm.N_HORIZON, rp.lmpc_params(rm.N_HORIZON)[1], rp.lmpc_params(rm.N_HORIZON)[0]
    _, _, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, B, workloads.track_seg_table(), rp.TRACK_LENGTH, trToUse=rm.TR_TO_USE, numSS_Points=M,
                          numSS_it=numSS_it, QterminalSlack=Qts, device=dev, Tmax=rm.TMAX, ss_cap=rm.SS_CAP,
                          model_cap=rm.MODEL_CAP)
    c.enable_rollout(Tcl=rm.TCL)
    c.enable_lap_reports(max(int(laps), 1))
    if streams is not None:
        c.set_noise_streams(streams)
    c.set_measurement_noise(*meas)
    if obs is not None:
        c.set_observers(*obs)
    return c


def read(c, name, shape, dtype=np.float64):
    out = np.zeros(shape, dtype)
    nat.check(c._lib.lmpc_read_buffer(c._h, name.encode(), 0, nat.ptr(out), out.nbytes))
    return out


def drive(c, laps, dev, seed=1234, at_poll=None):
    """PID lap, seeding, LMPC steps until every controller drove `laps` laps (or 300 steps per lap).  at_poll(c, step) runs
    around every POLL-th step: it gets ("before", c) and ("after", c).  Returns (steps, seconds of the LMPC steps)."""
    B = c.B
    x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (B, 1))
    c.rollout_set_state(x0, x0)
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(x0, x0)
    stream = torch.cuda.ExternalStream(c.stream, device=torch.device("cuda", dev))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(stream)
    steps = 0
    while steps < 300 * laps:
        poll = at_poll is not None and steps % POLL == 0
        if poll:
            at_poll("before", c)
        c.rollout_step(seed=seed)
        c.rollout_commit_laps_dev()
        if poll:
            at_poll("after", c)
        steps += 1
        if steps % POLL == 0 and c.rollout_stats()[0] >= laps:
            break
    e1.record(stream)
    e1.synchronize()
    return steps, e0.elapsed_time(e1) / 1e3


def result(c):
    return dict(books=c.books(), state=c.rollout_state(), health=c.rollout_health(), solver=c.step_results(),
                reports=c.lap_reports())


def same(a, b, path=()):
    if isinstance(a, dict):
        return all(same(a[k], b[k], path + (k,)) for k in a)
    if isinstance(a, (tuple, list)):
        return all(same(p, q, path) for p, q in zip(a, b))
    ok = np.asarray(a).tobytes() == np.asarray(b).tobytes()
    assert ok, path
    return ok


def leg_ab(rounds, batch, laps, dev):
    z = np.zeros(batch, np.int32)
    arms = {"no_table": None, "all_ones": ([ObserverParams.uniform(1.0)], z)}
    rate = {k: [] for k in arms}
    first = {}
    for _ in range(rounds):
        for name, obs in arms.items():
            c = controller(batch, dev, laps, ([BASE], z), obs)
            l0 = c.kernel_launches
            steps, secs = drive(c, laps, dev)
            rate[name].append(batch * steps / secs)
            if name not in first:
                first[name] = (steps, c.kernel_launches - l0, result(c))
            c.close()
    (na, la, ra), (nb, lb, rb) = first["no_table"], first["all_ones"]
    assert na == nb
    same(ra, rb)
    assert lb - la == na + 1000, (la, lb, na)            # one observer launch per LMPC and per PID step, nothing else
    a, b = np.array(rate["no_table"]), np.array(rate["all_ones"])
    d = 100.0 * (b / a - 1.0)
    return {"benchmark": "observers leg 1: closed loop under base measurement noise without an observer table vs all-ones rows "
                         "for every controller", **card(dev), "batch": batch, "laps": laps, "mode": "independent",
            "rounds": rounds, "controller_steps_per_s": {"no_table": a.tolist(), "all_ones": b.tolist()},
            "all_ones_over_no_table_pct_rounds": d.tolist(),
            "all_ones_over_no_table_pct": {"mean": float(d.mean()), "min": float(d.min()), "max": float(d.max())},
            "no_table_round_spread_pct": float(100.0 * (a.max() - a.min()) / a.mean()),
            "all_ones_round_spread_pct": float(100.0 * (b.max() - b.min()) / b.mean()),
            "kernel_launches_with_pid_lap": {"no_table": la, "all_ones": lb}, "lmpc_steps": na,
            "identical": ["books", "state", "health", "solver", "reports"]}


def leg_kernel(batch, dev, steps=400):
    z = np.zeros(batch, np.int32)
    c = controller(batch, dev, 1, ([BASE], z), ([ObserverParams.uniform(0.5)], z))
    x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (batch, 1))
    c.rollout_set_state(x0, x0)
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(x0, x0)
    for _ in range(20):                                  # warm-up
        c.rollout_step(seed=1)
        c.rollout_commit_laps_dev()
    torch.cuda.synchronize()
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            c.rollout_step(seed=1)
            c.rollout_commit_laps_dev()
        c.sync()
    times = {}
    for ev in prof.events():
        for k in ("observe_kernel", "measure_kernel", "sim_step_kernel", "ftocp"):
            if k in ev.name and ev.device_type.name == "CUDA":
                times.setdefault(k, []).append(ev.device_time if hasattr(ev, "device_time") else ev.cuda_time)
    c.close()
    out = {k: {"launches": len(v), "mean_us": float(np.mean(v)), "min_us": float(np.min(v)), "max_us": float(np.max(v))}
           for k, v in times.items()}
    assert out["observe_kernel"]["launches"] == steps
    return {"benchmark": "observers leg 2: kernel times under torch.profiler (CUDA activities), uniform gain 0.5, base "
                         "measurement noise, LMPC steps", **card(dev), "batch": batch, "steps": steps, "kernels": out}


def pilot_model_sigma(batch, laps, dev):
    """Per-channel RMS of y_{k+1} - p (p = xPred[1] of the previous step, s wrapped) in the x0 cell without observer, at the
    polls, over controllers with a prior and finite values."""
    z = np.zeros(batch, np.int32)
    c = controller(batch, dev, laps, ([MeasurementParams.zero()], z))
    acc = {"sq": np.zeros(6), "n": 0}
    hold = {}
    N = rm.N_HORIZON

    def at_poll(when, c):
        if when == "before":
            hold["hp"] = read(c, "has_pred", batch, np.int32)
            hold["p"] = read(c, "xPredPrev", (batch, N + 1, 6))[:, 1].copy()
            return
        y = read(c, "x_meas", (batch, 6))
        p = hold["p"]
        wrap = p[:, 4] - y[:, 4] > rp.TRACK_LENGTH / 2
        p[wrap, 4] = np.fmax(p[wrap, 4] - rp.TRACK_LENGTH, 0.0)
        d = y - p
        ok = (hold["hp"] == 1) & np.all(np.isfinite(d), axis=1)
        acc["sq"] += np.sum(d[ok] ** 2, axis=0)
        acc["n"] += int(ok.sum())
    drive(c, laps, dev, at_poll=at_poll)
    c.close()
    return np.sqrt(acc["sq"] / max(acc["n"], 1)), acc["n"]


def leg_study(batch, laps, dev, pilot_laps=5):
    meas_k = (0.0, 1.0, 3.0, 10.0)
    ms, n_pilot = pilot_model_sigma(batch // 16, pilot_laps, dev)
    names = ("none", "uniform_0.5", "uniform_0.2", "matched")
    cells = len(meas_k) * len(names)
    b = np.arange(batch)
    cell = b % cells
    midx, oidx = cell // len(names), cell % len(names)
    streams = b // cells                                 # controller j of every cell on stream j
    meas_rows = [MeasurementParams.scaled(k, BASE) for k in meas_k]
    obs_rows, obs_of = [ObserverParams.off()], np.zeros(batch, np.int32)
    for m, k in enumerate(meas_k):
        for o, name in enumerate(names):
            if name == "none":
                continue
            row = (ObserverParams.uniform(0.5) if name == "uniform_0.5" else ObserverParams.uniform(0.2) if name == "uniform_0.2"
                   else ObserverParams.from_noise(ms, np.asarray(meas_rows[m].sigma)))
            obs_of[(midx == m) & (oidx == o)] = len(obs_rows)
            obs_rows.append(row)
    c = controller(batch, dev, laps, (meas_rows, midx), (obs_rows, obs_of), streams=streams)
    acc = {"est": np.zeros((cells, 6)), "meas": np.zeros((cells, 6)), "n": np.zeros(cells)}
    hold = {}

    def at_poll(when, c):
        if when == "before":
            hold["x"] = c.rollout_state()["x"]
            return
        x = hold["x"]
        e = read(c, "x_est", (batch, 6)) - x
        y = read(c, "x_meas", (batch, 6)) - x
        ok = np.all(np.isfinite(e), axis=1) & np.all(np.isfinite(y), axis=1) & (np.abs(e[:, 4]) < rp.TRACK_LENGTH / 2)
        for k in range(cells):
            s = ok & (cell == k)
            acc["est"][k] += np.sum(e[s] ** 2, axis=0)
            acc["meas"][k] += np.sum(y[s] ** 2, axis=0)
            acc["n"][k] += s.sum()
    steps, secs = drive(c, laps, dev, at_poll=at_poll)
    bk = c.books()
    flags, unsolved = c.rollout_health()
    rep = c.lap_reports()
    c.close()
    out_cells = []
    for m, k in enumerate(meas_k):
        for o, name in enumerate(names):
            sel = (midx == m) & (oidx == o)
            kk = m * len(names) + o
            n_ok = acc["n"][kk]
            row = obs_rows[int(obs_of[sel][0])]
            lap_steps = {}
            for lap in (1, 5, 10, 20):
                if lap <= laps:
                    have = sel & (rep["n"] >= lap)
                    lap_steps[str(lap)] = float(rep["steps"][have, lap - 1].mean()) if have.any() else None
            last = sel & (rep["n"] >= laps)
            out_cells.append({
                "measurement_scale": k, "observer": name, "gain": list(row.gain) if row.mode == 1 else None,
                "controllers": int(sel.sum()), "finished": int((bk["lap_n"][sel] >= laps).sum()),
                "mean_lap_steps": lap_steps, "unsolved_steps": int(unsolved[sel].sum()),
                "with_flag_1": int((flags[sel] & 1 != 0).sum()),
                "with_reset_flag": int((flags[sel] & nat.FLAG_OBSERVER_RESET != 0).sum()),
                "left_lane_last_lap_share": float((rep["viol_steps"][last, laps - 1] > 0).mean()) if last.any() else None,
                "rms_x_est_minus_x": dict(zip(CHANNELS, np.sqrt(acc["est"][kk] / max(n_ok, 1)).tolist())),
                "rms_y_minus_x": dict(zip(CHANNELS, np.sqrt(acc["meas"][kk] / max(n_ok, 1)).tolist())),
                "rms_samples": int(n_ok)})
    return {"benchmark": "observers leg 3: closed-loop LMPC over measurement noise x{0,1,3,10} x observers {none, uniform 0.5, "
                         "uniform 0.2, matched}, independent mode, common noise streams", **card(dev), "batch": batch,
            "controllers_per_cell": batch // cells, "laps": laps, "lmpc_steps": steps, "seconds": secs,
            "base_set": {"sigma": BASE.sigma, "clip": BASE.clip},
            "matched_model_sigma": dict(zip(CHANNELS, ms.tolist())), "pilot": {"laps": pilot_laps, "samples": n_pilot},
            "cells": out_cells}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of leg 1")
    ap.add_argument("--batch", type=int, default=8192, help="controllers of legs 1 and 2")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps of leg 1")
    ap.add_argument("--study-batch", type=int, default=4096, help="controllers of leg 3 (16 cells)")
    ap.add_argument("--study-laps", type=int, default=20)
    ap.add_argument("--legs", default="1,2,3")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/observers.py needs a GPU")
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    legs = args.legs.split(",")
    for leg, fn in (("1", lambda: leg_ab(args.rounds, args.batch, args.laps, dev)), ("2", lambda: leg_kernel(args.batch, dev)),
                    ("3", lambda: leg_study(args.study_batch, args.study_laps, dev))):
        if leg not in legs:
            continue
        r = fn()
        print(json.dumps(r), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
