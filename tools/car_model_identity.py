#!/usr/bin/env python
"""tools/car_model_identity.py OLD.so NEW.so — do two builds compute the same nominal model and observer gains, bit for bit?

Runs each build in its own process (LMPC_B200_SO) on the same closed loop, a PID lap and then LMPC steps until every controller
has driven three LMPC laps, and hashes after every step what the kernels under test wrote:
  nominal_mode1    abc of an all-mode-1 prediction table (nominal_model_kernel<false>)
  nominal_mode2    abc of an all-mode-2 table (the plant's own car)
  nominal_surface  abc of an all-mode-2 table with a 16-zone surface (nominal_model_kernel<true>)
  observer_gain    obs_jac, obs_cov, obs_gain and x_est of a plant-prior Kalman observer under measurement noise
                   (observer_gain_kernel, observe_kernel<true, true>)
Prints one line per case: the number of steps hashed and whether every step's hash agrees.  Run on the GPU box.

  python tools/car_model_identity.py OLD.so NEW.so [--batch 1024]"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ("nominal_mode1", "nominal_mode2", "nominal_surface", "observer_gain")
LAPS = 3


def _read(c, name, shape):
    from racinglmpc_b200 import _native as nat                    # run_case put the tree on sys.path
    out = np.zeros(shape)
    nat.check(c._lib.lmpc_read_buffer(c._h, name.encode(), 0, nat.ptr(out), out.nbytes))
    return out


def run_case(case, B):
    """[hex digest per step] of the case's buffers over the PID lap's seeding and three LMPC laps"""
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests", "support")]
    import closed_loop as cl
    from racinglmpc_b200.reference_params import (MeasurementParams, ObserverGains, ObserverParams, ObserverPrior,
                                                  PredictionModelParams as P, SurfaceParams, TrackParams,
                                                  VehicleParams)
    L = TrackParams.l_shaped().TrackLength                        # closed_loop.controller's track
    z = np.zeros(B, np.int32)
    c = cl.controller(B)
    try:
        c.enable_rollout(Tcl=1024)
        if case == "nominal_mode1":
            c.set_prediction_models([P(1, VehicleParams.reference())], z)
        elif case in ("nominal_mode2", "nominal_surface"):
            c.set_prediction_models([P(2)], z)
        if case == "nominal_surface":
            c.set_surfaces([SurfaceParams.from_zones([(k * L / 16, (k + 0.5) * L / 16, 0.9, 0.8) for k in range(16)])], z)
        if case == "observer_gain":
            c.set_measurement_noise([MeasurementParams((1e-3,) * 6, (3e-3,) * 6)], z)
            c.set_observers([ObserverParams.uniform(0.5)], z)
            c.set_observer_priors([ObserverPrior.plant()], z)
            c.set_observer_gains([ObserverGains.kalman((1e-4, 1e-5, 1e-4, 1e-6, 1e-6, 1e-6), (1e-6,) * 6)], z)
        c.rollout_set_state(np.tile(cl.X0, (B, 1)), np.tile(cl.X0, (B, 1)))
        for _ in range(1000):
            c.rollout_pid_step(0.8, seed=4321)
        c.rollout_seed_from_record_dev(copies=4)
        c.rollout_set_state(np.tile(cl.X0, (B, 1)), np.tile(cl.X0, (B, 1)))
        names = [("obs_jac", (B, 36)), ("obs_cov", (B, 36)), ("obs_gain", (B, 36)), ("x_est", (B, 6))] \
            if case == "observer_gain" else [("abc", (B, cl.N, 54))]
        digests = []
        for n in range(6000):
            c.rollout_step(seed=1234)
            h = hashlib.sha256()
            for name, shape in names:
                h.update(_read(c, name, shape).tobytes())
            digests.append(h.hexdigest())
            c.rollout_commit_laps_dev()
            if n % 8 == 0 and c.books()["lap_n"].min() >= LAPS:
                break
        return digests
    finally:
        c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old", nargs="?")
    ap.add_argument("new", nargs="?")
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--case", help=argparse.SUPPRESS)          # one build, one case: the child process
    a = ap.parse_args()
    if a.case:
        print(json.dumps(run_case(a.case, a.batch)))
        return
    ok = True
    for case in CASES:
        out = []
        for so in (a.old, a.new):
            env = dict(os.environ, LMPC_B200_SO=os.path.abspath(so))
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--case", case, "--batch", str(a.batch)], env=env,
                               stdout=subprocess.PIPE, text=True, check=True, cwd=ROOT)
            out.append(json.loads(r.stdout.strip().splitlines()[-1]))
        same = out[0] == out[1]
        ok = ok and same
        print("%-16s batch %d  %d / %d steps  %s" % (case, a.batch, len(out[0]), len(out[1]),
                                                     "bit-identical" if same else "DIFFER at step %d" % next(
                                                         (i for i, (p, q) in enumerate(zip(*out)) if p != q), -1)))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
