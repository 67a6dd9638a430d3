"""Numpy restatement of the observer's model gains (lmpc_rollout_set_observer_gains; observer_gain_kernel and
observe_kernel<true, true> in csrc/observer.cuh; DESIGN.md, "Observer gains"), for tests.

  curvature       the device's curvature lookup in fp64 (wrap by subtraction, first segment with s0 <= s < s0 + len)
  zone_forces     a surface row's peak tyre forces at s: fl(mu_f Df), fl(mu_r Dr) in a zone, else Df, Dr
  tangent_period  Phi_car(x, u) and A = dPhi_car/dx by forward mode through the simulator's sub-steps, with the expressions of
                  sim_substep_tangent (curvature and zone forces held constant, the input not differentiated)
  sda             the filter DARE P = A P A' - A P (P + R)^-1 P A' + Q by the structured doubling algorithm of the kernel
  kalman_gain     K = P (P + R)^-1
  blend           x_hat of one controller from the device's K, its prior p (after the lap-wrap fix) and y, rounded as the
                  kernel rounds it: e_j = y_j - p_j, c_i = K_i0 e_0 + ... + K_i5 e_5 left to right, x_hat_i = p_i + c_i
"""
import numpy as np

import observer as ob

FLAG_OBSERVER_GAIN = 4096
DARE_ITERS = 64
DARE_TOL = 1e-13
H = 0.001


def curvature(seg, L, s):
    """(curvature, ok) of the device's lookup: seg [nseg, 3] = (s_start, length, curvature)."""
    seg = np.asarray(seg, np.float64).reshape(-1, 3)
    L = np.float64(L)
    s = np.float64(s)
    if not s <= 64.0 * L:
        return 0.0, False
    while s > L:
        s = s - L
    for s0, ln, c in seg:
        if s0 <= s < s0 + ln:
            return np.float64(c), True
    return 0.0, False


def zone_forces(zones, s, L, Df, Dr):
    """The sub-step's peak forces under a surface row ``zones`` [(s_start, s_end, mu_f, mu_r), ...] (None: no surface)."""
    if zones is None:
        return np.float64(Df), np.float64(Dr)
    s, L = np.float64(s), np.float64(L)
    if not s <= 64.0 * L:
        return np.float64(Df), np.float64(Dr)
    while s > L:
        s = s - L
    for z0, z1, mf, mr in zones:
        if z0 <= s < z1:
            return np.float64(mf) * np.float64(Df), np.float64(mr) * np.float64(Dr)
    return np.float64(Df), np.float64(Dr)


def tangent_period(v, seg, L, x, u, dt=0.1, zones=None, s_trace=None):
    """(p [6], A [6, 6], ok) for car ``v`` (ten vehicle fields) from the curvilinear state x under u = (delta, a).  ``s_trace``
    (a list) collects the s every sub-step starts from."""
    f = np.float64
    m, lf, lr, Iz = f(v.m), f(v.lf), f(v.lr), f(v.Iz)
    Df, Cf, Bf, Dr, Cr, Br = f(v.Df), f(v.Cf), f(v.Bf), f(v.Dr), f(v.Cr), f(v.Br)
    delta, acc = f(u[0]), f(u[1])
    sd, cd = np.sin(delta), np.cos(delta)
    x = np.array(x, np.float64)
    D = np.eye(6)
    ok = True
    i = 0
    while (i + 1) * H <= dt:
        vx, vy, wz, epsi, s, ey = x
        if s_trace is not None:
            s_trace.append(float(s))
        dvx, dvy, dwz, depsi, ds, dey = D
        Dfi, Dri = zone_forces(zones, s, L, Df, Dr)
        yf, yr = vy + lf * wz, vy - lf * wz
        af = delta - np.arctan2(yf, vx)
        ar = -np.arctan2(yr, vx)
        daf = -(vx * (dvy + lf * dwz) - yf * dvx) / (vx * vx + yf * yf)
        dar = -(vx * (dvy - lf * dwz) - yr * dvx) / (vx * vx + yr * yr)
        tf, tr = Cf * np.arctan(Bf * af), Cr * np.arctan(Br * ar)
        Fyf, Fyr = Dfi * np.sin(tf), Dri * np.sin(tr)
        dFyf = Dfi * np.cos(tf) * Cf * Bf / (1 + Bf * af * Bf * af) * daf
        dFyr = Dri * np.cos(tr) * Cr * Br / (1 + Br * ar * Br * ar) * dar
        cur, okc = curvature(seg, L, s)
        ok = ok and okc
        ce, se = np.cos(epsi), np.sin(epsi)
        den = 1 - cur * ey
        q = (vx * ce - vy * se) / den
        dnum = dvx * ce - vx * se * depsi - dvy * se - vy * ce * depsi
        dq = (dnum + q * cur * dey) / den
        nD = np.empty_like(D)
        nD[0] = dvx + H * (-(1 / m) * dFyf * sd + dwz * vy + wz * dvy)
        nD[1] = dvy + H * (1 / m * (dFyf * cd + dFyr) - dwz * vx - wz * dvx)
        nD[2] = dwz + H * (1 / Iz * (lf * dFyf * cd - lr * dFyr))
        nD[3] = depsi + H * (dwz - dq * cur)
        nD[4] = ds + H * dq
        nD[5] = dey + H * (dvx * se + vx * ce * depsi + dvy * ce - vy * se * depsi)
        x = np.array([vx + H * (acc - 1 / m * Fyf * sd + wz * vy),
                      vy + H * (1 / m * (Fyf * cd + Fyr) - wz * vx),
                      wz + H * (1 / Iz * (lf * Fyf * cd - lr * Fyr)),
                      epsi + H * (wz - q * cur),
                      s + H * q,
                      ey + H * (vx * se + vy * ce)])
        D = nD
        i += 1
    return x, D, ok


def sda(A, q, r, iters=DARE_ITERS, tol=DARE_TOL):
    """(P, converged, doublings) of the filter DARE for A [6, 6], Q = diag(q), R = diag(r): A0 = A', G0 = R^-1, H0 = Q;
    W = I + G H, A <- A W^-1 A, G <- G + A W^-1 G A', H <- H + A' H W^-1 A, stopped once max|H' - H| <= tol max|H'|; P is the
    symmetric part of the last H."""
    Ak = np.array(A, np.float64).T.copy()
    G = np.diag(1.0 / np.asarray(r, np.float64))
    Hk = np.diag(np.asarray(q, np.float64))
    I = np.eye(Ak.shape[0])
    for it in range(iters):
        W = I + G @ Hk
        X1 = np.linalg.solve(W, Ak)
        X2 = np.linalg.solve(W, G)
        An = Ak @ X1
        Gn = G + Ak @ X2 @ Ak.T
        Hn = Hk + Ak.T @ (Hk @ X1)
        conv = np.max(np.abs(Hn - Hk)) <= tol * np.max(np.abs(Hn))
        Ak, G, Hk = An, Gn, Hn
        if conv:
            return 0.5 * (Hk + Hk.T), True, it + 1
    return 0.5 * (Hk + Hk.T), False, iters


def kalman_gain(P, r):
    """K = P (P + R)^-1."""
    S = P + np.diag(np.asarray(r, np.float64))
    return np.linalg.solve(S, P).T


def dare_residual(A, P, q, r):
    """max|P - (A P A' - A P (P + R)^-1 P A' + Q)| / max|P|."""
    A, P = np.asarray(A, np.float64), np.asarray(P, np.float64)
    S = P + np.diag(np.asarray(r, np.float64))
    rhs = A @ P @ A.T - A @ P @ np.linalg.solve(S, P @ A.T) + np.diag(np.asarray(q, np.float64))
    return np.max(np.abs(P - rhs)) / np.max(np.abs(P))


def blend(y, p, K, L):
    """x_hat [6] of a mode 1 gain row from y, the prior p (before or after the lap-wrap fix) and the device's K [6, 6]."""
    y = np.asarray(y, np.float64)
    p = np.array(p, np.float64)
    K = np.asarray(K, np.float64).reshape(6, 6)
    p[4] = ob.wrap_guess_s(p[4], y[4], L)
    e = [y[j] - p[j] for j in range(6)]
    x = np.empty(6)
    for i in range(6):
        c = K[i, 0] * e[0]
        for j in range(1, 6):
            c = c + K[i, j] * e[j]
        x[i] = p[i] + c
    return x
