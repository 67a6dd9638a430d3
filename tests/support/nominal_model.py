"""Exact restatement of the nominal prediction model (lmpc_set_prediction_models, nominal_model_kernel), for tests.

Phi is the noise-free map of the velocity subsystem (vx, vy, wz, delta, a) -> (vx, vy, wz) over one control period: the
simulator's sub-steps (SysModel.py:94-106, plant_exact.dyn_model) with h = 0.001 while (i + 1) h <= dt.  ``rows`` evaluates Phi
and its forward sensitivities S = dPhi/d(vx, vy, wz, delta, a) in mpmath at DPS digits from the fp64 inputs, with no rounding in
between, and forms rows 0..2 of the stage model (A, B, C) the device writes.  ``numdiff`` checks those formulas independently:
central differences of plant_exact.dyn_model (zero noise), extrapolated (Richardson), in the same exact arithmetic.  With a
track surface (``surface=``, a plant_exact.ExactSurface, on ``track=``) every function carries (epsi, s, ey) through the
sub-steps so that each sub-step's peak forces follow the zone of its s; the zones add nothing to the derivatives.

The variants of ``rows`` (keyword ``variant``) are the known-wrong implementations the device bound must reject:
  alpha_r_lr     lr in place of lf in alpha_r (the same as the correct model for a car with lf == lr)
  substeps_99    one sub-step short
  no_sin_delta   the front force's -Fyf sin(delta) / m term of the vx rate dropped
  euler_dt       a single explicit-Euler step of dt: Phi = z + dt f, A = I + dt f_z, B = dt f_u
"""
import mpmath as mp
import numpy as np

from plant_exact import DPS, ExactTrack, LookupFailed, VEHICLE_FIELDS, _f, _substeps, dyn_model

# |dev - exact| <= NOMINAL_BOUND (1 + |exact|) per entry of rows 0..2 of A, B and C (the measured H100 deviation and its margin:
# profiles/h100_prediction_models.txt)
NOMINAL_BOUND = 2.0 ** -40

VARIANTS = ("alpha_r_lr", "substeps_99", "no_sin_delta", "euler_dt")


def _rates(m, lf, lr, Iz, Df, Cf, Bf, Dr, Cr, Br, vx, vy, wz, delta, acc, arm_r, no_sin):
    """(f, f_z, f_u) of the velocity subsystem at one state: the rates of SysModel.py:98-100 and their derivatives."""
    sd, cd = mp.sin(delta), mp.cos(delta)
    pf, pq = vy + lf * wz, vy - arm_r * wz
    af = delta - mp.atan2(pf, vx)
    ar = -mp.atan2(pq, vx)
    tf, tr = mp.atan(Bf * af), mp.atan(Br * ar)
    Fyf, Fyr = Df * mp.sin(Cf * tf), Dr * mp.sin(Cr * tr)
    gf = Df * mp.cos(Cf * tf) * Cf * Bf / (1 + (Bf * af) ** 2)
    gr = Dr * mp.cos(Cr * tr) * Cr * Br / (1 + (Br * ar) ** 2)
    rf, rr = 1 / (vx ** 2 + pf ** 2), 1 / (vx ** 2 + pq ** 2)
    daf = [pf * rf, -vx * rf, -lf * vx * rf]
    dar = [pq * rr, -vx * rr, arm_r * vx * rr]
    s = 0 if no_sin else 1
    f = [acc - s * Fyf * sd / m + wz * vy, (Fyf * cd + Fyr) / m - wz * vx, (lf * Fyf * cd - lr * Fyr) / Iz]
    fz = [[-s * sd / m * gf * daf[j] for j in range(3)],
          [(cd * gf * daf[j] + gr * dar[j]) / m for j in range(3)],
          [(lf * cd * gf * daf[j] - lr * gr * dar[j]) / Iz for j in range(3)]]
    fz[0][1] += wz; fz[0][2] += vy
    fz[1][0] -= wz; fz[1][2] -= vx
    fu = [[-s * (gf * sd + Fyf * cd) / m, mp.mpf(1)],
          [(gf * cd - Fyf * sd) / m, mp.mpf(0)],
          [lf * (gf * cd - Fyf * sd) / Iz, mp.mpf(0)]]
    return f, fz, fu


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


def from_abc(abc):
    """Rows 0..2 of one stage's 54 entries (A [6][6] | B [6][2] | C [6]) as (A [3][6], B [3][2], C [3]) fp64 arrays."""
    abc = np.asarray(abc, float)
    return abc[:36].reshape(6, 6)[:3], abc[36:48].reshape(6, 2)[:3], abc[48:54][:3]


def deviation(dev, exact):
    """max over the entries of rows 0..2 of |dev - exact| / (1 + |exact|), the measure NOMINAL_BOUND bounds: ``dev`` the
    device's (A, B, C) (from_abc), ``exact`` the mpf (A, B, C) of ``rows``."""
    worst = 0.0
    with mp.workdps(DPS):
        for d, e in zip(dev, exact):
            for dv, ev in zip(np.asarray(d, float).ravel(), np.asarray(e, dtype=object).ravel()):
                if not np.isfinite(dv):
                    return float("inf")
                worst = max(worst, float(abs(_f(dv) - ev) / (1 + abs(ev))))
    return worst


_FLAT = ExactTrack([[0.0, 1000.0, 0.0]], 1000.0)


def _phi_plant(vehicle, xv, uv, dt, kin=None, surface=None, track=None):
    """Phi from plant_exact.dyn_model with zero noise, on a straight track (the velocity subsystem does not read the track), or
    with a surface from the kinematic state kin = (epsi, s, ey) on ``track``."""
    if surface is None:
        out = dyn_model(vehicle, _FLAT, [xv[0], xv[1], xv[2], 0.0, 1.0, 0.0], [0.0] * 6, uv, z=(0.0, 0.0, 0.0), dt=dt)
    else:
        out = dyn_model(vehicle, track, [xv[0], xv[1], xv[2]] + list(kin), [0.0] * 6, uv, z=(0.0, 0.0, 0.0), dt=dt, on_fail="zero",
                        surface=surface)
    return out["x"][:3]


def numdiff(vehicle, x, u, dt=0.1, k=2.0 ** -24, surface=None, track=None):
    """(Phi, S) of plant_exact.dyn_model (with the surface) by central differences at steps k and k / 2 extrapolated to O(k^4) (Richardson; the
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
