"""Exact restatement of the plant kernels, for tests: the operations of the reference evaluated in multi-precision arithmetic
(mpmath, DPS digits) from the fp64 inputs and constants the device actually used, with no rounding in between.

  dyn_model     Simulator.dynModel (SysModel.py:56-147)        sim_step_kernel, with or without a track surface (ExactSurface)
  pid_input     PID.solve (Utilities.py:42-68)                 pid_input_kernel
  regression    Regression (Utilities.py:5-28)                 ridge_sysid_kernel
  compute_cost  LMPC.computeCost (PC.py:447-464)               lap_cost_block (rollout_cost_kernel, lap hand-over, seeding)

Every fp64 value converts to an mpf exactly, so the results are the real-number values of the reference's formulas at those
inputs; the fp64 implementations (NumPy's and the device's) are judged by their distance to them.  The curvature lookup of
each sub-step (Track.py:292-310) compares the exact s with the track table's fp64 boundaries s0 and s0 + length (that sum
rounded to fp64, as both the reference and the device form it) and wraps by repeated exact subtraction of the fp64
TrackLength.  A state a fp64 implementation could place on the other side of a boundary is one whose exact s lies within its
rounding error of that boundary: ``dyn_model`` reports the smallest distance of any computed sub-step's s to a boundary, so a
case can check its own margin.  A track surface (lmpc_rollout_set_surfaces, ExactSurface) sets each sub-step's peak tyre forces
from the zone its s lies in; ``dyn_model`` reports the distance to a zone bound the same way.

The variants of ``dyn_model`` and ``regression`` (keyword ``variant``) are the known-wrong implementations the tests' bounds
must reject.
"""
import math

import mpmath as mp
import numpy as np

DPS = 60
EPS = 2.0 ** -52
SIM_BOUND = 2.0 ** -44          # |fp64 - exact| <= SIM_BOUND (1 + |exact|) per component and control period

VEHICLE_FIELDS = ("m", "lf", "lr", "Iz", "Df", "Cf", "Bf", "Dr", "Cr", "Br")


class LookupFailed(ValueError):
    """Map.curvature has no segment for s: the reference raises (Track.py:292-310)."""


def _f(v):
    return mp.mpf(float(v))


class ExactTrack:
    """A track table ([nseg, 3] = s_start, length, curvature, as the device reads it) and its fp64 TrackLength."""

    def __init__(self, seg_table, track_length):
        seg = np.asarray(seg_table, float).reshape(-1, 3)
        self.s0 = [_f(r[0]) for r in seg]
        self.end = [_f(np.float64(r[0]) + np.float64(r[1])) for r in seg]
        self.cur = [_f(r[2]) for r in seg]
        self.L = _f(track_length)
        self.bounds = sorted(set(self.s0 + self.end))

    def lookup(self, s):
        """(curvature, distance of the wrapped s to the nearest boundary).  Raises LookupFailed where the device's lookup
        fails: s not finite, s beyond 64 laps (the device's guard against a runaway state), or no segment after the wrap
        (s < 0, s exactly at the finish line)."""
        if not mp.isfinite(s) or s > 64 * self.L:
            raise LookupFailed("s = %s" % mp.nstr(s, 20))
        while s > self.L:
            s = s - self.L
        for s0, e, c in zip(self.s0, self.end, self.cur):
            if s >= s0 and s < e:
                return c, min(abs(s - b) for b in self.bounds)
        raise LookupFailed("s = %s has no segment" % mp.nstr(s, 20))


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


def _substeps(dt, h=0.001):
    """SysModel.py:83's loop count, in fp64 as the reference and the device evaluate it."""
    i = 0
    while (i + 1) * h <= dt:
        i += 1
    return i


def dyn_model(vehicle, track, x, x_glob, u, z=(0.0, 0.0, 0.0), noise=None, dt=0.1, on_fail="raise", variant=None, surface=None):
    """One control period of SysModel.py:56-147, exactly.  ``vehicle``: an object with the ten fields above; ``track``: an
    ExactTrack; ``surface``: an ExactSurface, whose zone each sub-step's peak tyre forces follow, or None; ``z``: the three
    standard-normal draws (vx, vy, wz); ``noise``: an object with sim_sigma, sim_clip, sim_gain
    (None: the reference's constants).  ``on_fail``: "raise" (the reference) or "zero" (go on with curvature 0, as the device
    does, and report it).  Returns dict(x, x_glob: lists of 6 mpf, margin: smallest distance of the s of sub-steps 1.. to a
    segment boundary (sub-step 0's s is an fp64 input and is placed exactly by every implementation), failed: bool,
    done: s_next > TrackLength).
    ``variant`` (known-wrong implementations): "alpha_r_lr" (lr in place of lf in alpha_r), "curvature_at_next_s" (the epsi
    update reads the curvature at the updated s), "noise_global" (noise added to the global copy), "substeps_99",
    "substeps_101"; with a ``surface`` (an ExactSurface) also "mu_at_start" (the zone of sub-step 0 for the whole period),
    "mu_front_only", "zone_closed_end" and "zone_unwrapped" (ExactSurface's variants).  The result also holds zone_margin: the
    smallest distance of the s of sub-steps 1.. to a zone bound (inf without a surface)."""
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


def to_f64(v):
    return np.array([float(e) for e in v])


def sim_error(dev, exact):
    """max over components of |dev - exact| / (1 + |exact|), the measure SIM_BOUND bounds."""
    dev = np.asarray(dev, float)
    with mp.workdps(DPS):
        return max(float(abs(_f(d) - e) / (1 + abs(e))) for d, e in zip(dev, exact))


def pid_input(x, vt, z, pid_sigma=(0.25, 0.10), pid_clip=(0.9, 0.2)):
    """Utilities.py:42-68 exactly: [-0.6 ey - 0.9 epsi + clip(z0 sigma0), 1.5 (vt - vx) + clip(z1 sigma1)] (mpf pair)."""
    with mp.workdps(DPS):
        c0 = max(-_f(pid_clip[0]), min(_f(z[0]) * _f(pid_sigma[0]), _f(pid_clip[0])))
        c1 = max(-_f(pid_clip[1]), min(_f(z[1]) * _f(pid_sigma[1]), _f(pid_clip[1])))
        return (_f(-0.6) * _f(x[5]) - _f(0.9) * _f(x[3]) + c0, _f(1.5) * (_f(vt) - _f(x[0])) + c1)


def regression(x, u, lamb, variant=None):
    """Utilities.py:5-28 exactly: W = (Z'Z + lamb I)^-1 Z'Y with z_t = [x_t u_t], y_t = x_{t+1}, t = 1 .. T-2.  Returns
    dict(A [6,6], B [6,2] as fp64 arrays of the exactly rounded values, W (mp matrix), maxW, cond = the 1-norm condition
    number of Z'Z + lamb I).  ``variant``: "rows_0" (t = 0 .. T-3), "no_lambda"."""
    x = np.asarray(x, float)
    u = np.asarray(u, float)
    T = x.shape[0]
    t0 = 0 if variant == "rows_0" else 1
    lam = 0.0 if variant == "no_lambda" else lamb
    with mp.workdps(DPS):
        rows = range(t0, t0 + T - 2)
        Z = [[_f(v) for v in np.concatenate([x[t], u[t]])] for t in rows]
        Y = [[_f(v) for v in x[t + 1]] for t in rows]
        M = mp.matrix(8, 8)
        R = mp.matrix(8, 6)
        for zr, yr in zip(Z, Y):
            for i in range(8):
                zi = zr[i]
                if zi == 0:
                    continue
                for j in range(8):
                    M[i, j] += zi * zr[j]
                for j in range(6):
                    R[i, j] += zi * yr[j]
        for i in range(8):
            M[i, i] += _f(lam)
        Minv = mp.inverse(M)
        W = Minv * R
        cond = mp.mnorm(M, 1) * mp.mnorm(Minv, 1)
        Wf = np.array([[float(W[i, j]) for j in range(6)] for i in range(8)])
        return dict(A=Wf.T[:, 0:6].copy(), B=Wf.T[:, 6:8].copy(), W=W, maxW=float(np.max(np.abs(Wf))), cond=float(cond),
                    T=T)


def regression_gauss_jordan(x, u, lamb):
    """NumPy emulation of ridge_sysid_kernel's arithmetic: the same sums over t = 1 .. T-2, the same Gauss-Jordan elimination
    with partial pivoting on [Z'Z + lamb I | Z'Y] and the same final divisions (fp64, no fused operations).  Returns A, B and
    whether the kernel would flag the solve (bit 1: T < 12 or a zero pivot column)."""
    x = np.asarray(x, float)
    u = np.asarray(u, float)
    T = x.shape[0]
    Z = np.hstack([x, u])
    S = np.zeros((8, 14))
    for r in range(8):
        for c in range(14):
            acc = 0.0
            for t in range(1, T - 1):
                acc += Z[t, r] * (Z[t, c] if c < 8 else x[t + 1, c - 8])
            S[r, c] = acc + (lamb if r == c else 0.0)
    ok = T >= 12
    for p in range(8):
        piv, best = p, abs(S[p, p])
        for r in range(p + 1, 8):
            if abs(S[r, p]) > best:
                best, piv = abs(S[r, p]), r
        if not best > 0.0:
            ok = False
        S[[p, piv]] = S[[piv, p]]
        inv = 1.0 / S[p, p] if S[p, p] != 0.0 else 0.0
        f = S[:, p] * inv
        prow = S[p].copy()
        for r in range(8):
            if r != p:
                S[r, p + 1:] -= f[r] * prow[p + 1:]
    with np.errstate(divide="ignore", invalid="ignore"):
        W = S[:, 8:] / np.diag(S)[:, None]
    return W.T[:, 0:6].copy(), W.T[:, 6:8].copy(), not ok


def sysid_error(A, B, ref):
    """max |(A | B) - exact| / (max(cond, T) eps max|W|): the measure SYSID_C bounds (the T covers the rounding of the T-term
    sums of the normal equations, which dominates when the ridge makes them well conditioned)."""
    with mp.workdps(DPS):
        W = ref["W"]
        e = 0.0
        for i in range(6):
            for j in range(6):
                e = max(e, float(abs(_f(A[i, j]) - W[j, i])))
            for k in range(2):
                e = max(e, float(abs(_f(B[i, k]) - W[6 + k, i])))
    return e / (max(ref["cond"], ref["T"]) * EPS * ref["maxW"])


# The sysid bound |W_dev - W_exact| <= SYSID_C max(cond, T) eps max|W|: at least four times the largest ratio the NumPy
# emulation of the kernel's elimination (regression_gauss_jordan) reaches on the calibration records of
# tests/test_plant_reference.py (0.120, the golden PID lap with lambda = 1e3; 1.1e-3 with lambda = 1e-7 at cond 5.5e7).
SYSID_C = 0.5


def compute_cost(s, track_length):
    """PC.py:447-464: Qfun[T-1] = 0, Qfun[j] = Qfun[j+1] + 1 if s_j < TrackLength else 0 (integers, so exact in fp64).
    ``s``: the lap's s column."""
    s = np.asarray(s, float)
    T = s.shape[0]
    q = np.zeros(T)
    for i in range(T):
        j = T - 1 - i
        if i == 0:
            q[j] = 0
        elif s[j] < track_length:
            q[j] = q[j + 1] + 1
        else:
            q[j] = 0
    return q


def compute_cost_le(s, track_length):
    """A known-wrong computeCost: s_j <= TrackLength keeps counting."""
    s = np.asarray(s, float)
    q = np.zeros(s.shape[0])
    for j in range(s.shape[0] - 2, -1, -1):
        q[j] = q[j + 1] + 1 if s[j] <= track_length else 0
    return q


def ulp(v):
    return math.ulp(float(v))
