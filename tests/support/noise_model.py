"""Test-side noise of the closed loop for any noise set (lmpc_rollout_set_noise; reference_params.NoiseParams fields).

``dyn_model`` is tests/support/vehicle_model.dyn_model with the simulator's noise constants (SysModel.py:139-145) taken from a
noise set: the dynamics come from vehicle_model with its noise held at zero, then the set's noise is added in the reference's
form, gain * clip(z * sigma, +-clip) per channel on the curvilinear copy, with the same three draws (vx, vy, wz) in the same
order.  With the reference's set it equals vehicle_model.dyn_model, and so tests/golden/vehicle_golden.npz, bit for bit.
``PIDFollower`` is the oracle's PID path follower (Utilities.py:42-68) with the set's PID noise.  ``with_draws`` makes
closed_loop.run drive one controller with other Philox seeds, or with host-given draws of zeros.
"""
import numpy as np

import vehicle_model as vm


class _Zeros:
    def standard_normal(self):
        return 0.0


def dyn_model(track, x, x_glob, u, vehicle, noise, dt=0.1, rng=None):
    """One control period of SysModel.py:56-147 with ``vehicle`` and the simulator noise of ``noise`` (sim_sigma[3],
    sim_clip[3], sim_gain).  ``rng`` None => global np.random."""
    randn = np.random.randn if rng is None else rng.standard_normal
    xn, gn = vm.dyn_model(track, x, x_glob, u, vehicle, dt=dt, rng=_Zeros())     # adds 0.01 * 0.0: x unchanged
    sig, clip, gain = noise.sim_sigma, noise.sim_clip, noise.sim_gain
    n = [np.max([-clip[j], np.min([randn() * sig[j], clip[j]])]) for j in range(3)]
    for j in range(3):
        xn[j] += gain * n[j]
    return xn, gn


class PIDFollower:
    """Utilities.py:42-68 (oracle.vehicle.PIDFollower) with the PID noise of ``noise`` (pid_sigma[2], pid_clip[2]) in place of
    the reference's constants, in the same form and order of draws."""

    def __init__(self, vt, noise, rng=None):
        self.vt = vt
        self.noise = noise
        self.uPred = np.zeros([1, 2])
        self._randn = np.random.randn if rng is None else rng.standard_normal

    def solve(self, x0):
        r, s, c = self._randn, self.noise.pid_sigma, self.noise.pid_clip
        self.uPred[0, 0] = -0.6 * x0[5] - 0.9 * x0[3] + np.max([-c[0], np.min([r() * s[0], c[0]])])
        self.uPred[0, 1] = 1.5 * (self.vt - x0[0]) + np.max([-c[1], np.min([r() * s[1], c[1]])])


def closed_loop(track, x_start, controller, vehicle, noise, *, max_steps, dt=0.1, rng=None):
    """vehicle_model.closed_loop with the simulator noise of ``noise``.  Returns x_cl[T,6], u_cl[T,2], x_glob[T,6] and the state
    after the last step (both frames)."""
    xs = [np.asarray(x_start[0], dtype=float)]
    gs = [np.asarray(x_start[1], dtype=float)]
    us = []
    for _ in range(max_steps):
        controller.solve(xs[-1])
        us.append(controller.uPred[0, :].copy())
        xt, gt = dyn_model(track, xs[-1], gs[-1], us[-1], vehicle, noise, dt=dt, rng=rng)
        xs.append(xt)
        gs.append(gt)
    last = (xs.pop(), gs.pop())
    return np.array(xs), np.array(us), np.array(gs), last


def with_draws(c, seeds=None, zeros=False):
    """Make the closed-loop steps of controller ``c`` (a BatchedController) use the Philox seeds ``seeds`` = (PID lap, LMPC
    steps) instead of the ones they are called with, or, with ``zeros``, host-given draws of zeros.  For closed_loop.run's hook."""
    pid_step, step = c.rollout_pid_step, c.rollout_step
    zp, zs = (np.zeros((c.B, 2)), np.zeros((c.B, 3))) if zeros else (None, None)

    def rollout_pid_step(vt, z_pid=None, z_sim=None, seed=0):
        pid_step(vt, z_pid=zp, z_sim=zs, seed=seeds[0] if seeds else seed)

    def rollout_step(z=None, seed=0, mode=None):
        step(z=zs, seed=seeds[1] if seeds else seed, mode=mode)

    c.rollout_pid_step, c.rollout_step = rollout_pid_step, rollout_step
