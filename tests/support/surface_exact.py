"""Exact restatement of the track surfaces (lmpc_rollout_set_surfaces), for tests: the plant of plant_exact.dyn_model and the
nominal model of nominal_model.rows with each simulator sub-step's peak tyre forces taken from the zone its s lies in.

  ExactSurface  one surface row: the zone of an exact s against the fp64 bounds, wrapped as ExactTrack.lookup wraps it
  dyn_model     plant_exact.dyn_model with ``surface=``; without a surface it is that function, operation for operation
  phi_sens      nominal_model.phi_sens with ``surface=`` on a track: (epsi, s, ey) carried through the sub-steps
  rows          nominal_model.rows on top of phi_sens
  numdiff       nominal_model.numdiff of this dyn_model

Zones are piecewise constant in s, so they add nothing to the derivatives.  Every function reports the smallest distance of the
s of sub-steps 1.. to a zone bound (``zone_margin``), as plant_exact reports its segment margin, so a case can check its own.
The variants of ``dyn_model`` (keyword ``variant``) are the known-wrong implementations the tests' bounds must reject.
"""
import math

import mpmath as mp
import numpy as np

from plant_exact import DPS, LookupFailed, VEHICLE_FIELDS, _f, _substeps
from nominal_model import _FLAT, _rates


class ExactSurface:
    """A track-surface row (lmpc_rollout_set_surfaces): zones (s_start, s_end, mu_f, mu_r) as fp64 values.  ``at`` places the
    exact s of a sub-step against the fp64 bounds, wrapped as ExactTrack.lookup wraps it, and returns the sub-step's peak forces
    fl(mu_f Df), fl(mu_r Dr) (each product rounded once to fp64, as the device forms it) or Df, Dr exactly off every zone, with the
    distance of the wrapped s to the nearest zone bound.  ``variant``: "closed_end" (s <= s_end matches), "unwrapped" (the zone
    tested on the unwrapped s), "front_only" (mu_r ignored)."""

    def __init__(self, zones):
        self.zones = [tuple(float(v) for v in z) for z in zones]
        self.bounds = sorted(set(_f(z[0]) for z in self.zones) | set(_f(z[1]) for z in self.zones))

    def at(self, s, L, Df, Dr, variant=""):
        dist = min((abs(s - b) for b in self.bounds), default=mp.inf) if mp.isfinite(s) else mp.inf
        if not mp.isfinite(s) or s > 64 * L:
            return _f(Df), _f(Dr), dist
        if variant != "unwrapped":
            while s > L:
                s = s - L
            dist = min((abs(s - b) for b in self.bounds), default=mp.inf)
        for s0, s1, muf, mur in self.zones:
            if _f(s0) <= s and (s <= _f(s1) if variant == "closed_end" else s < _f(s1)):
                dr = _f(Dr) if variant == "front_only" else _f(np.float64(mur) * np.float64(Dr))
                return _f(np.float64(muf) * np.float64(Df)), dr, dist
        return _f(Df), _f(Dr), dist


def dyn_model(vehicle, track, x, x_glob, u, z=(0.0, 0.0, 0.0), noise=None, dt=0.1, on_fail="raise", variant=None, surface=None):
    """plant_exact.dyn_model with a track surface: one control period of SysModel.py:56-147, exactly.  ``vehicle``: an object with the ten fields above; ``track``: an
    ExactTrack; ``z``: the three standard-normal draws (vx, vy, wz); ``noise``: an object with sim_sigma, sim_clip, sim_gain
    (None: the reference's constants).  ``on_fail``: "raise" (the reference) or "zero" (go on with curvature 0, as the device
    does, and report it).  Returns dict(x, x_glob: lists of 6 mpf, margin: smallest distance of the s of sub-steps 1.. to a
    segment boundary (sub-step 0's s is an fp64 input and is placed exactly by every implementation), failed: bool,
    done: s_next > TrackLength).
    ``variant`` (known-wrong implementations): "alpha_r_lr" (lr in place of lf in alpha_r), "curvature_at_next_s" (the epsi
    update reads the curvature at the updated s), "noise_global" (noise added to the global copy), "substeps_99",
    "substeps_101"; with a ``surface`` (an ExactSurface) also "mu_at_start" (the zone of sub-step 0 for the whole period),
    "mu_front_only", "zone_closed_end" and "zone_unwrapped" (ExactSurface's variants).  With a surface the result also holds
    zone_margin: the smallest distance of the s of sub-steps 1.. to a zone bound."""
    variant = variant or ""
    with mp.workdps(DPS):
        m, lf, lr, Iz, Df, Cf, Bf, Dr, Cr, Br = (_f(getattr(vehicle, k)) for k in VEHICLE_FIELDS)
        h = _f(0.001)
        delta, acc = _f(u[0]), _f(u[1])
        vx, vy, wz, epsi, s, ey = (_f(v) for v in x)
        psi, X, Y = _f(x_glob[3]), _f(x_glob[4]), _f(x_glob[5])
        n = _substeps(dt) + {"substeps_99": -1, "substeps_101": 1}.get(variant, 0)
        sd, cd = mp.sin(delta), mp.cos(delta)
        arm_r = lr if variant == "alpha_r_lr" else lf
        margin, failed = mp.inf, False
        zone_margin = mp.inf
        zvar = {"mu_front_only": "front_only", "zone_closed_end": "closed_end", "zone_unwrapped": "unwrapped"}.get(variant, "")
        D0 = None

        # IEEE sign of an exactly zero atan2 argument (vy +- lf wz == 0 with vx <= 0: the branch cut at +-pi): taken from the
        # fp64 inputs at sub-step 0, where they can be signed zeros; later sub-steps produce +0
        y_f = (float(x[1]) + float(vehicle.lf) * float(x[2]), float(x[1]) - float(vehicle.lf) * float(x[2]))

        def atan2(y, xv, i, k):
            if y == 0 and xv <= 0:
                r = math.atan2(y_f[k] if i == 0 else 0.0, float(x[0]) if i == 0 else float(xv))
                return mp.mpf(0) if r == 0 else math.copysign(1.0, r) * mp.pi
            return mp.atan2(y, xv)

        def curvature(sv, i):
            nonlocal margin, failed
            try:
                c, d = track.lookup(sv)
            except LookupFailed:
                if on_fail != "zero":
                    raise
                failed = True
                return mp.mpf(0)
            if i > 0:
                margin = min(margin, d)
            return c

        for i in range(n):
            Dfi, Dri = Df, Dr
            if surface is not None:
                if variant == "mu_at_start" and D0 is not None:
                    Dfi, Dri = D0
                else:
                    Dfi, Dri, d = surface.at(s, track.L, vehicle.Df, vehicle.Dr, zvar)
                    D0 = (Dfi, Dri)
                    if i > 0:
                        zone_margin = min(zone_margin, d)
            af = delta - atan2(vy + lf * wz, vx, i, 0)
            ar = -atan2(vy - arm_r * wz, vx, i, 1)
            Fyf = Dfi * mp.sin(Cf * mp.atan(Bf * af))
            Fyr = Dri * mp.sin(Cr * mp.atan(Br * ar))
            nvx = vx + h * (acc - 1 / m * Fyf * sd + wz * vy)
            nvy = vy + h * (1 / m * (Fyf * cd + Fyr) - wz * vx)
            nwz = wz + h * (1 / Iz * (lf * Fyf * cd - lr * Fyr))
            npsi = psi + h * wz
            nX = X + h * (vx * mp.cos(psi) - vy * mp.sin(psi))
            nY = Y + h * (vx * mp.sin(psi) + vy * mp.cos(psi))
            cur = curvature(s, i)
            ce, se = mp.cos(epsi), mp.sin(epsi)
            vl = vx * ce - vy * se
            ns = s + h * (vl / (1 - cur * ey))
            cur_e = curvature(ns, i + 1) if variant == "curvature_at_next_s" else cur
            nepsi = epsi + h * (wz - vl / (1 - cur_e * ey) * cur_e)
            ney = ey + h * (vx * se + vy * ce)
            psi, X, Y = npsi, nX, nY
            vx, vy, wz, epsi, s, ey = nvx, nvy, nwz, nepsi, ns, ney
        nz = noise
        sig = [_f(v) for v in (nz.sim_sigma if nz else (0.01, 0.01, 0.005))]
        clip = [_f(v) for v in (nz.sim_clip if nz else (0.05, 0.05, 0.05))]
        gain = _f(nz.sim_gain if nz else 0.01)
        draw = [max(-clip[j], min(_f(z[j]) * sig[j], clip[j])) for j in range(3)]
        xs = [vx, vy, wz, epsi, s, ey]
        gs = [vx, vy, wz, psi, X, Y]
        tgt = gs if variant == "noise_global" else xs
        for j in range(3):
            tgt[j] = tgt[j] + gain * draw[j]
        return dict(x=xs, x_glob=gs, margin=margin, failed=failed, done=bool(s > track.L), draw=[gain * d for d in draw],
                    zone_margin=zone_margin)


def phi_sens(vehicle, x, u, dt=0.1, variant=None, surface=None, track=None):
    """(Phi: 3 mpf, S: 3 x 5 mpf) at the fp64 state x (its first three entries) and input u, exactly.  With a ``surface`` (an
    ExactSurface) on ``track`` (an ExactTrack), (epsi, s, ey) of x are carried through the sub-steps with the
    plant's curvature lookup (curvature 0 where it fails, as the device goes on) and each sub-step's peak forces follow the zone
    of its s; the zones add nothing to the derivatives.  ``phi_sens.zone_margin`` is then the smallest distance of the s of
    sub-steps 1.. to a zone bound."""
    variant = variant or ""
    phi_sens.zone_margin = mp.inf
    with mp.workdps(DPS):
        m, lf, lr, Iz, Df, Cf, Bf, Dr, Cr, Br = (_f(getattr(vehicle, k)) for k in VEHICLE_FIELDS)
        arm_r = lr if variant == "alpha_r_lr" else lf
        delta, acc = _f(u[0]), _f(u[1])
        z = [_f(x[0]), _f(x[1]), _f(x[2])]
        S = [[mp.mpf(1 if c == r else 0) for c in range(5)] for r in range(3)]
        if variant == "euler_dt":
            steps, h = 1, _f(dt)
        else:
            steps, h = _substeps(dt) - (1 if variant == "substeps_99" else 0), _f(0.001)
        epsi, s, ey = (_f(x[j]) for j in (3, 4, 5)) if surface is not None else (None, None, None)
        for k in range(steps):
            Dfi, Dri = Df, Dr
            if surface is not None:
                Dfi, Dri, d = surface.at(s, track.L, vehicle.Df, vehicle.Dr)
                if k > 0:
                    phi_sens.zone_margin = min(phi_sens.zone_margin, d)
                try:
                    cur = track.lookup(s)[0]
                except LookupFailed:
                    cur = mp.mpf(0)
                ce, se = mp.cos(epsi), mp.sin(epsi)
                vl = z[0] * ce - z[1] * se
                epsi, s, ey = (epsi + h * (z[2] - vl / (1 - cur * ey) * cur), s + h * (vl / (1 - cur * ey)),
                               ey + h * (z[0] * se + z[1] * ce))
            f, fz, fu = _rates(m, lf, lr, Iz, Dfi, Cf, Bf, Dri, Cr, Br, z[0], z[1], z[2], delta, acc, arm_r, variant == "no_sin_delta")
            S = [[S[r][c] + h * (sum(fz[r][j] * S[j][c] for j in range(3)) + (fu[r][c - 3] if c >= 3 else 0)) for c in range(5)]
                 for r in range(3)]
            z = [z[r] + h * f[r] for r in range(3)]
        return z, S


def rows(vehicle, x, u, dt=0.1, variant=None, surface=None, track=None):
    """Rows 0..2 of the stage model at (x, u) as the device lays them out: A [3][6], B [3][2], C [3] (mpf), exactly (with a
    surface on a track as in ``phi_sens``)."""
    phi, S = phi_sens(vehicle, x, u, dt, variant, surface, track)
    with mp.workdps(DPS):
        A = [[S[r][0], S[r][1], S[r][2], mp.mpf(0), mp.mpf(0), mp.mpf(0)] for r in range(3)]
        B = [[S[r][3], S[r][4]] for r in range(3)]
        C = [phi[r] - (sum(A[r][j] * _f(x[j]) for j in range(6)) + B[r][0] * _f(u[0]) + B[r][1] * _f(u[1])) for r in range(3)]
    return A, B, C


def _phi_plant(vehicle, xv, uv, dt, kin=None, surface=None, track=None):
    """Phi from dyn_model with zero noise, on a straight track (the velocity subsystem does not read the track), or
    with a surface from the kinematic state kin = (epsi, s, ey) on ``track``."""
    if surface is None:
        out = dyn_model(vehicle, _FLAT, [xv[0], xv[1], xv[2], 0.0, 1.0, 0.0], [0.0] * 6, uv, z=(0.0, 0.0, 0.0), dt=dt)
    else:
        out = dyn_model(vehicle, track, [xv[0], xv[1], xv[2]] + list(kin), [0.0] * 6, uv, z=(0.0, 0.0, 0.0), dt=dt, on_fail="zero",
                        surface=surface)
    return out["x"][:3]


def numdiff(vehicle, x, u, dt=0.1, k=2.0 ** -24, surface=None, track=None):
    """(Phi, S) of dyn_model (with the surface) by central differences at steps k and k / 2 extrapolated to O(k^4) (Richardson; the
    evaluations are exact to DPS digits, so a small k costs no accuracy).  The
    steps are powers of two applied in fp64 (exact for the magnitudes of the test states; the actual step is used either way),
    so every evaluation is exact at its input.  With a ``surface`` on ``track``, x[3:6] is the kinematic state the plant
    starts from (the differences move no zone bound into the period when the case's zone margin exceeds the steps' effect)."""
    base = [float(x[0]), float(x[1]), float(x[2]), float(u[0]), float(u[1])]
    kin = [float(v) for v in x[3:6]] if surface is not None else None
    with mp.workdps(DPS):
        phi = _phi_plant(vehicle, base[:3], base[3:], dt, kin, surface, track)
        S = [[None] * 5 for _ in range(3)]
        for c in range(5):
            est = []
            for step in (k, k / 2):
                p, q = list(base), list(base)
                p[c] = base[c] + step
                q[c] = base[c] - step
                fp = _phi_plant(vehicle, p[:3], p[3:], dt, kin, surface, track)
                fq = _phi_plant(vehicle, q[:3], q[3:], dt, kin, surface, track)
                hs = _f(p[c]) - _f(q[c])
                est.append([(fp[r] - fq[r]) / hs for r in range(3)])
            for r in range(3):
                S[r][c] = (4 * est[1][r] - est[0][r]) / 3
        return phi, S
