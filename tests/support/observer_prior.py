"""Exact restatement of the observer's model prior (lmpc_rollout_set_observer_priors; observe_kernel<true> in csrc/observer.cuh;
DESIGN.md, "Observer priors"), for tests.

  back_laps      how many laps before lap_n a source 2 prior reads its rows at: 1 when a hand-over came between the previous
                 step and this one (x_hat_{k-1}.s - y.s > TrackLength / 2), else 0
  scheduled_row  the row of a lap schedule [L] at lap lap_n - back, clamped to [0, L - 1]
  prior_exact    Phi_car(x_prev, u): plant_exact.dyn_model with zero draws and no global frame, its curvilinear state (mpf)
  blend          the observer's lap-wrap fix and blend of one controller from a given prior (observer.observe_one)

The device prior runs the simulator's own sub-step code, so with process noise off it equals the plant state bit for bit; against
prior_exact it is judged by plant_exact.SIM_BOUND, like the simulator.
"""
from types import SimpleNamespace

import numpy as np

import observer as ob
import plant_exact as pe

NO_NOISE = SimpleNamespace(sim_sigma=(0.0, 0.0, 0.0), sim_clip=(0.0, 0.0, 0.0), sim_gain=0.0)


def back_laps(prev_s, y_s, L):
    """1 when the previous estimate's s lies more than half a lap ahead of the measured s (the plant's s was moved back by L at
    a hand-over in between, and lap_n moved on), else 0."""
    return 1 if np.float64(prev_s) - np.float64(y_s) > np.float64(L) / np.float64(2.0) else 0


def scheduled_row(rows, lap_n, back):
    """The row a lap schedule ``rows`` [L] gives lap lap_n - back (clamped to the schedule)."""
    rows = np.asarray(rows).reshape(-1)
    return int(rows[min(max(int(lap_n) - int(back), 0), rows.shape[0] - 1)])


def prior_exact(vehicle, track, x_prev, u, dt=0.1, surface=None):
    """The exact noise-free control period of ``vehicle`` (an object with the ten vehicle fields) from the curvilinear state
    x_prev under u = (delta, a), with ``surface`` (plant_exact.ExactSurface) or none, on ``track`` (plant_exact.ExactTrack).
    Returns the dyn_model result: x (six mpf), margin, failed (a sub-step's lookup failed) and, with a surface, zone_margin."""
    return pe.dyn_model(vehicle, track, x_prev, np.zeros(6), u, z=(0.0, 0.0, 0.0), noise=NO_NOISE, dt=dt, on_fail="zero",
                        surface=surface)


def blend(y, p, gain, L):
    """(x_hat [6], reset) of a mode 1 row from the prior p [6], before or after the lap-wrap fix (the device's x_prior is after
    it; a wrapped prior lies within half a lap of y_s, so the fix leaves it as it is)."""
    x, _, reset = ob.observe_one(y, p, 1, 1, gain, L)
    return x, reset
