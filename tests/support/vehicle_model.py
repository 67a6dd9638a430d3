"""Test-side restatement of Simulator.dynModel / Simulator.sim (SysModel.py:22-147) for any vehicle.

oracle/vehicle.py restates the reference with its one car folded in as constants; this module takes the ten vehicle constants
(SysModel.py:61-70) as an argument instead, so that the device simulator's per-controller vehicles (lmpc_rollout_set_vehicles)
can be checked.  It is itself checked bit for bit against the reference's own dynModel with its constants replaced
(tests/golden/vehicle_golden.npz) and, on the reference car, against oracle.vehicle.dyn_model.  Same arithmetic, same order of
operations and the same draws (three per call: vx, vy, wz) as the oracle.
"""
import numpy as np

VEHICLE_FIELDS = ("m", "lf", "lr", "Iz", "Df", "Cf", "Bf", "Dr", "Cr", "Br")


def dyn_model(track, x, x_glob, u, vehicle, dt=0.1, rng=None):
    """One control period of SysModel.py:56-147 with ``vehicle`` (an object with the ten field names above) in place of the
    reference's constants: 100 explicit-Euler sub-steps of 1 ms + clipped noise.  ``rng`` None => global np.random."""
    randn = np.random.randn if rng is None else rng.standard_normal
    m, lf, lr, Iz, Df, Cf, Bf, Dr, Cr, Br = (getattr(vehicle, f) for f in VEHICLE_FIELDS)
    h = 0.001
    delta, a = u[0], u[1]
    psi, X, Y = x_glob[3], x_glob[4], x_glob[5]
    vx, vy, wz, epsi, s, ey = x[0], x[1], x[2], x[3], x[4], x[5]
    glob = np.zeros(6)
    cur_next = np.zeros(6)
    i = 0
    while (i + 1) * h <= dt:
        af = delta - np.arctan2(vy + lf * wz, vx)
        ar = -np.arctan2(vy - lf * wz, vx)              # lf, as SysModel.py:97 has it
        Fyf = Df * np.sin(Cf * np.arctan(Bf * af))
        Fyr = Dr * np.sin(Cr * np.arctan(Br * ar))
        nvx = vx + h * (a - 1 / m * Fyf * np.sin(delta) + wz * vy)
        nvy = vy + h * (1 / m * (Fyf * np.cos(delta) + Fyr) - wz * vx)
        nwz = wz + h * (1 / Iz * (lf * Fyf * np.cos(delta) - lr * Fyr))
        glob[0], glob[1], glob[2] = nvx, nvy, nwz
        glob[3] = psi + h * wz
        glob[4] = X + h * (vx * np.cos(psi) - vy * np.sin(psi))
        glob[5] = Y + h * (vx * np.sin(psi) + vy * np.cos(psi))
        cur = track.curvature(s)
        cur_next[0], cur_next[1], cur_next[2] = nvx, nvy, nwz
        cur_next[3] = epsi + h * (wz - (vx * np.cos(epsi) - vy * np.sin(epsi)) / (1 - cur * ey) * cur)
        cur_next[4] = s + h * ((vx * np.cos(epsi) - vy * np.sin(epsi)) / (1 - cur * ey))
        cur_next[5] = ey + h * (vx * np.sin(epsi) + vy * np.cos(epsi))
        psi, X, Y = glob[3], glob[4], glob[5]
        vx, vy, wz, epsi, s, ey = cur_next
        i += 1
    n_vx = np.max([-0.05, np.min([randn() * 0.01, 0.05])])
    n_vy = np.max([-0.05, np.min([randn() * 0.01, 0.05])])
    n_wz = np.max([-0.05, np.min([randn() * 0.005, 0.05])])
    cur_next[0] += 0.01 * n_vx
    cur_next[1] += 0.01 * n_vy
    cur_next[2] += 0.01 * n_wz
    return cur_next.copy(), glob.copy()


def closed_loop(track, x_start, controller, vehicle, *, max_steps, dt=0.1, rng=None):
    """SysModel.py:22-54 in multi-lap mode for ``max_steps`` steps with ``vehicle``.  Returns x_cl[T,6], u_cl[T,2], x_glob[T,6]
    and the state after the last step (both frames, s not wrapped)."""
    xs = [np.asarray(x_start[0], dtype=float)]
    gs = [np.asarray(x_start[1], dtype=float)]
    us = []
    for _ in range(max_steps):
        controller.solve(xs[-1])
        us.append(controller.uPred[0, :].copy())
        xt, gt = dyn_model(track, xs[-1], gs[-1], us[-1], vehicle, dt=dt, rng=rng)
        xs.append(xt)
        gs.append(gt)
    last = (xs.pop(), gs.pop())
    return np.array(xs), np.array(us), np.array(gs), last
