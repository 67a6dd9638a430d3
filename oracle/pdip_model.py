"""NumPy model of the GPU solver's algorithm (Mehrotra primal-dual interior point with a
stage-wise Riccati factorisation).  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

This is NOT a restatement of anything in the reference: it is an executable specification
of racinglmpc_b200/csrc/ftocp_pdip.cuh, written first so that the algorithm could be
validated on the CPU against the OSQP-algorithm oracle (two independent algorithms must
agree on the optimum) before any kernel existed.  Tests use it to localise kernel bugs.

Problem (same data the reference assembles at PredictiveControllers.py:166-257,340-362):
  z = [x_1..x_N | u_0..u_{N-1} | s_0..s_{N-1} | lambda | xi],  x_0 = x(t) fixed
  cost  sum_k (x_k-xRef)'Q(x_k-xRef) + (x_N-xRef)'Qf(x_N-xRef) + u_k'R u_k
        + sum_k (u_k-u_{k-1})' dR (u_k-u_{k-1})  (u_{-1} = OldInput)
        + qs_quad |s|^2 + qs_lin 1's + Qfun'lambda + xi' Qts xi           (constants dropped)
  s.t.  x_{k+1} = A_k x_k + B_k u_k + C_k ;  Fx x_k - s_k <= bx (k<N) ; Fu u_k <= bu ;
        s >= 0 ; lambda >= 0 ; x_N - SS lambda + xi = 0 ; 1'lambda = 1.
"""
import numpy as np

RECENTER = True       # replace the corrector by a pure centring step when its step cannot re-enter the neighbourhood
RECENTER_AFTER = 3    # ... within this many reductions (kernel: RECENTRE_AFTER)
W_REFINE = 1      # refinement steps of the 6x6 covariance-form solve, residual taken through the recovered dlam
ADAPTIVE_FLOOR = False  # experiment (relax the floor on stall): helps some instances, hurts others -> off
EXACT_TERMINAL_RECOVERY = False
TERM_REFINE = 0   # terminal-block iterative refinement (experiment; the kernel does not need it)
DEBUG_HOOK = False
D4_MIN = 1e-6   # floor on the lambda barrier diagonal nu4/lambda (static primal regularisation).
                # Without W_REFINE the 6x6 covariance-form elimination of lambda loses the Newton direction below
                # ~1e-5 (measured: tests/golden snapshots); with one refinement step 1e-4..1e-7 all converge in
                # 9-16 iterations and 1e-6 removes the stall of LP-degenerate instances the 1e-4 floor caused.


class StageQP:
    """Plain container; fields mirror the C-ABI structs (include/lmpc_b200.h)."""

    def __init__(self, N, Q, R, Qf, dR, qs_quad, qs_lin, xRef, Fx, bx, Fu, bu,
                 A, B, C, x0, uOld, SS=None, Qfun=None, Qts=None):
        self.N = N
        self.Q, self.R, self.Qf = np.asarray(Q, float), np.asarray(R, float), np.asarray(Qf, float)
        self.dR = np.asarray(dR, float).ravel()
        self.qs_quad, self.qs_lin = float(qs_quad), float(qs_lin)
        self.xRef = np.asarray(xRef, float).ravel()
        self.Fx, self.bx = np.asarray(Fx, float), np.asarray(bx, float).ravel()
        self.Fu, self.bu = np.asarray(Fu, float), np.asarray(bu, float).ravel()
        self.A, self.B, self.C = np.asarray(A, float), np.asarray(B, float), np.asarray(C, float)
        self.x0, self.uOld = np.asarray(x0, float).ravel(), np.asarray(uOld, float).ravel()
        self.SS = None if SS is None else np.asarray(SS, float)
        self.Qfun = None if Qfun is None else np.asarray(Qfun, float).ravel()
        self.Qts = None if Qts is None else np.asarray(Qts, float)
        self.m = 0 if SS is None else self.SS.shape[1]


def from_params(p, A, B, C, x0, uOld, SS=None, Qfun=None, Qts=None):
    """Build a StageQP from an oracle.ftocp.FTOCPParams (LTI: A,B single matrices)."""
    N, n = p.N, p.n
    A = np.asarray(A, float)
    if A.ndim == 2:
        A = np.tile(A, (N, 1, 1))
        B = np.tile(np.asarray(B, float), (N, 1, 1))
        C = np.zeros((N, n))
    return StageQP(N, p.Q, p.R, p.Qf, p.dR, p.Qslack[0], p.Qslack[1], p.xRef, p.Fx, np.squeeze(p.bx),
                   p.Fu, np.squeeze(p.bu), A, B, C, x0, np.asarray(uOld, float).ravel(), SS, Qfun, Qts)


def kernel_constants(N, lmpc):
    """The LMPC_TUNE_* defaults of racinglmpc_b200/csrc/ftocp_pdip.cuh as keyword arguments of solve(): problems with a safe
    set keep the round-1 values, MPC-type problems use the ones swept through the host emulation (DESIGN.md section 2)."""
    if lmpc:
        return dict(s0=0.3, mu0_scale=1.0, step=0.995, backoff=0.8, gamma=0.01)
    return dict(s0=0.1 if N <= 16 else (0.2 if N <= 24 else 0.5), mu0_scale=0.05, step=0.999, backoff=0.9, gamma=0.003)


def solve(qp, eps=1e-9, max_iter=60, verbose=False, eps_step=1e-7, eps_gap=None, mu0="auto", s0=0.3, gamma=0.01, warm=None, snap_mu=None,
          warm_theta=0.5, mu0_scale=1.0, step=0.995, backoff=0.8):
    """Returns dict(x[N+1,n], u[N,d], s[N,ncx], lam[m], xi[n], iters, r_prim, r_dual, gap, status).
    s0 / mu0_scale / step / backoff / gamma: starting point and step rule (defaults = the round-1 kernel;
    ``solve(qp, **kernel_constants(qp.N, qp.m > 0))`` follows the kernel for either problem type)."""
    N, n, d = qp.N, 6, 2
    Fx, bx, Fu, bu = qp.Fx, qp.bx, qp.Fu, qp.bu
    ncx, ncu, m = Fx.shape[0], Fu.shape[0], qp.m
    Q2, R2, Qf2 = 2 * qp.Q, 2 * qp.R, 2 * qp.Qf
    qx, qxN = -2 * qp.Q @ qp.xRef, -2 * qp.Qf @ qp.xRef
    dR2 = 2 * qp.dR
    A, B, C = qp.A, qp.B, qp.C
    lmpc = m > 0
    if lmpc:
        SS, Qfun, T = qp.SS, qp.Qfun, 2 * qp.Qts
        Tinv = np.linalg.inv(T)

    # ---------------- initial point ------------------------------------------------
    g = Fu @ qp.uOld
    tau = 1.0
    for j in range(ncu):
        if g[j] > 0.9 * bu[j]:
            tau = min(tau, 0.9 * bu[j] / g[j])
    u = np.tile(tau * qp.uOld, (N, 1))
    if warm is not None and warm.get("primal_only"):
        u = warm["u"].copy()
        for k in range(N):            # keep the input rows strictly inside their bounds
            g = Fu @ u[k]
            t = 1.0
            for j in range(ncu):
                if g[j] > 0.9 * bu[j]:
                    t = min(t, 0.9 * bu[j] / g[j])
            u[k] *= t
    x = np.zeros((N + 1, n))
    x[0] = qp.x0
    for k in range(N):
        x[k + 1] = A[k] @ x[k] + B[k] @ u[k] + C[k]
    s = np.zeros((N, ncx))
    w1 = np.zeros((N, ncx))
    for k in range(N):
        viol = Fx @ x[k] - bx
        s[k] = np.maximum(viol, 0.0) + s0
        w1[k] = bx - Fx @ x[k] + s[k]
    w2 = np.array([bu - Fu @ u[k] for k in range(N)])
    if mu0 is None:
        nu1, nu2, nu3 = np.ones((N, ncx)), np.ones((N, ncu)), np.ones((N, ncx))
    elif mu0 == "auto":
        # slack-stationarity holds exactly (nu1 + nu3 = 2 qs s + ql) with w1 nu1 = s nu3 = mu_row;
        # every other family is centred at the mean of those products
        mur = (2 * qp.qs_quad * s + qp.qs_lin) * (w1 * s) / (w1 + s)
        nu1, nu3 = mur / w1, mur / s
        mu0 = max(mu0_scale * float(np.mean(mur)), 1e-3)
        nu2 = mu0 / w2
    else:                                   # centred start: every complementarity product = mu0
        nu1, nu2, nu3 = mu0 / w1, mu0 / w2, mu0 / s
    if lmpc:
        lam = np.ones(m) / m
        xi = SS @ lam - x[N]
        yT = -T @ xi
        red = Qfun - SS.T @ yT
        y1 = -np.min(red) + (1.0 if mu0 is None else mu0 * m)
        nu4 = red + y1
    n_ineq = N * (2 * ncx + ncu) + m
    if warm is not None and not warm.get("primal_only"):
        # warm start from an intermediate iterate of the previous (shifted) problem: inputs, lane slacks and all
        # multipliers are taken over, states are rolled out from the new x0, derived slacks kept >= theta * old
        u = warm["u"].copy()
        for k in range(N):
            x[k + 1] = A[k] @ x[k] + B[k] @ u[k] + C[k]
        s = warm["s"].copy()
        w1 = np.array([bx - Fx @ x[k] + s[k] for k in range(N)])
        low = w1 < warm_theta * warm["w1"]
        s = np.where(low, s + warm_theta * warm["w1"] - w1, s)
        w1 = np.array([bx - Fx @ x[k] + s[k] for k in range(N)])
        w2 = np.array([bu - Fu @ u[k] for k in range(N)])
        nu1, nu2, nu3 = warm["nu1"].copy(), warm["nu2"].copy(), warm["nu3"].copy()
        if lmpc:
            lam, nu4, y1 = warm["lam"].copy(), warm["nu4"].copy(), float(warm["y1"])
    snap = None

    def u_rate_grad(u):
        gr = np.zeros((N, d))
        for k in range(N):
            prev = qp.uOld if k == 0 else u[k - 1]
            gr[k] += dR2 * (u[k] - prev)
            if k < N - 1:
                gr[k] += dR2 * (u[k] - u[k + 1])
        return gr

    status, it = 2, 0
    d4_floor, rdual_prev, al_prev = D4_MIN, 1e300, 0.0
    step_prev = np.inf       # |alpha (dx, du)|_inf of the step just taken: residuals alone do not bound the distance to the optimum
    for it in range(max_iter + 1):
        # ---- residuals -----------------------------------------------------------
        r1 = np.array([Fx @ x[k] - s[k] + w1[k] - bx for k in range(N)])
        r2 = np.array([Fu @ u[k] + w2[k] - bu for k in range(N)])
        rdyn = np.array([x[k + 1] - A[k] @ x[k] - B[k] @ u[k] - C[k] for k in range(N)])
        rs = 2 * qp.qs_quad * s + qp.qs_lin - nu1 - nu3
        if lmpc:
            xi = SS @ lam - x[N]            # derived: terminal equality holds by construction
            yT = -T @ xi                    # derived: xi-stationarity holds by construction
            rT = np.zeros(n)
            rone = np.sum(lam) - 1.0
            rxi = np.zeros(n)
            rlam = Qfun - SS.T @ yT + y1 - nu4
        # costates defined so that the x-stationarity rows hold exactly
        pi = np.zeros((N + 1, n))
        pi[N] = -(Qf2 @ x[N] + qxN + (yT if lmpc else 0.0))
        for k in range(N - 1, 0, -1):
            pi[k] = -(Q2 @ x[k] + qx + Fx.T @ nu1[k]) + A[k].T @ pi[k + 1]
        ru = np.array([R2 @ u[k] + Fu.T @ nu2[k] - B[k].T @ pi[k + 1] for k in range(N)]) + u_rate_grad(u)
        comp = np.sum(w1 * nu1) + np.sum(w2 * nu2) + np.sum(s * nu3) + (np.sum(lam * nu4) if lmpc else 0.0)
        mu = comp / n_ineq
        r_prim = max(np.abs(r1).max(), np.abs(r2).max(), np.abs(rdyn).max(),
                     (max(np.abs(rT).max(), abs(rone)) if lmpc else 0.0))
        r_dual = max(np.abs(ru).max(), np.abs(rs).max(),
                     (max(np.abs(rxi).max(), np.abs(rlam).max()) if lmpc else 0.0))
        if verbose:
            print("it %2d  rp %.2e rd %.2e mu %.2e" % (it, r_prim, r_dual, mu))
        if snap_mu is not None and snap is None and (mu <= snap_mu):
            snap = dict(u=u.copy(), s=s.copy(), w1=w1.copy(), nu1=nu1.copy(), nu2=nu2.copy(), nu3=nu3.copy(), mu=mu, it=it)
            if lmpc:
                snap.update(lam=lam.copy(), nu4=nu4.copy(), y1=y1)
        if r_prim <= eps and r_dual <= eps and mu <= (eps if eps_gap is None else eps_gap) and step_prev <= eps_step:
            status = 1
            break
        if ADAPTIVE_FLOOR and lmpc and it > 0 and al_prev >= 0.9 and r_dual > 0.25 * rdual_prev:
            d4_floor = min(d4_floor, 0.1 * D4_MIN)
            if verbose:
                print("      floor ->", d4_floor)
        rdual_prev = r_dual
        if it == max_iter:
            break

        # ---- barrier diagonals, condensed stage Hessians ---------------------------
        d1, d2, d3 = nu1 / w1, nu2 / w2, nu3 / s
        hs = 2 * qp.qs_quad + d1 + d3
        Dt = d1 * (2 * qp.qs_quad + d3) / hs          # = d1 - d1^2/hs without cancellation
        Hxx = [Q2 + Fx.T @ (Dt[k][:, None] * Fx) for k in range(N)]
        Huu = []
        for k in range(N):
            c = 2.0 if k < N - 1 else 1.0
            Huu.append(R2 + np.diag(c * dR2) + Fu.T @ (d2[k][:, None] * Fu))
        if lmpc:
            d4 = np.maximum(nu4 / lam, d4_floor)
            delta = np.sum(1.0 / d4)
            sbar = (SS / d4[None, :]) @ np.ones(m) / delta   # D^-1-weighted centroid
            Sc = SS - sbar[:, None]
            SD = Sc / d4[None, :]
            W = SD @ Sc.T + Tinv
            Lw = np.linalg.cholesky(W)
            Lwi = np.linalg.inv(Lw)              # triangular inverse (kernel: forward substitution)
            Wi = Lwi.T @ Lwi                     # PSD by construction, benign error structure
            PN = Qf2 + Wi
        else:
            PN = Qf2.copy()

        # ---- Riccati factorisation (matrices) -----------------------------------
        Pxx, Pxv, Pvv = PN, np.zeros((n, d)), np.zeros((d, d))
        Ls, Zs, Zvs = [None] * N, [None] * N, [None] * N
        for k in range(N - 1, -1, -1):
            M = B[k].T @ Pxx + Pxv.T
            Lam = Huu[k] + M @ B[k] + B[k].T @ Pxv + Pvv
            L = np.linalg.cholesky(Lam)
            Y = M @ A[k]
            Z = np.linalg.solve(L, Y)
            Zv = np.linalg.solve(L, np.diag(dR2))
            Ls[k], Zs[k], Zvs[k] = L, Z, Zv
            Pxx_new = Hxx[k] + A[k].T @ Pxx @ A[k] - Z.T @ Z
            Pxv = Z.T @ Zv
            Pvv = -Zv.T @ Zv
            Pxx = 0.5 * (Pxx_new + Pxx_new.T)

        def solve_rhs(rc1, rc2, rc3, rc4):
            """One back/forward sweep for given complementarity right-hand sides."""
            e1 = -rc1 / w1 + d1 * r1
            gs = -rs + e1 - rc3 / s
            ex = (e1 * (2 * qp.qs_quad + d3) + d1 * (rs + rc3 / s)) / hs   # = e1 - d1*gs/hs, cancellation-free
            eu = -rc2 / w2 + d2 * r2
            rtx = [Fx.T @ ex[k] for k in range(N)]             # r_x == 0 by construction
            rtu = [ru[k] + Fu.T @ eu[k] for k in range(N)]
            if lmpc:
                rho_l = -rlam - rc4 / lam
                c1 = -SD @ rho_l + sbar * rone
                beta = -rone - np.sum(rho_l / d4)
                pN = Wi @ c1
            else:
                pN = np.zeros(n)
            px, pv = pN, np.zeros(d)
            z0s = [None] * N
            for k in range(N - 1, -1, -1):
                g0 = rtu[k] + B[k].T @ px + pv
                z0 = np.linalg.solve(Ls[k], g0)
                z0s[k] = z0
                px = rtx[k] + A[k].T @ px - Zs[k].T @ z0
                pv = Zvs[k].T @ z0
            dx = np.zeros((N + 1, n))
            du = np.zeros((N, d))
            dv = np.zeros(d)
            for k in range(N):
                du[k] = -np.linalg.solve(Ls[k].T, Zs[k] @ dx[k] - Zvs[k] @ dv + z0s[k])
                dx[k + 1] = A[k] @ dx[k] + B[k] @ du[k]
                dv = du[k]
            ds = np.array([(gs[k] + d1[k] * (Fx @ dx[k])) / hs[k] for k in range(N)])
            dw1 = np.array([-r1[k] - Fx @ dx[k] + ds[k] for k in range(N)])
            dw2 = np.array([-r2[k] - Fu @ du[k] for k in range(N)])
            dnu1 = (-rc1 - nu1 * dw1) / w1
            dnu2 = (-rc2 - nu2 * dw2) / w2
            dnu3 = (-rc3 - nu3 * ds) / s
            out = dict(dx=dx, du=du, ds=ds, dw1=dw1, dw2=dw2, dnu1=dnu1, dnu2=dnu2, dnu3=dnu3)
            if lmpc:
                dyT = Wi @ (dx[N] + c1)
                dy1t = -beta / delta                        # multiplier of the centred simplex row
                dlam = (rho_l + Sc.T @ dyT - dy1t) / d4
                for _ in range(W_REFINE):
                    # iterative refinement of the 6x6 covariance-form solve, residual evaluated THROUGH the recovered dlam:
                    #   T^-1 dyT + S~ dlam = dx_N - sbar*b1   (b1 = -rone)
                    e_T = dx[N] + sbar * rone - Tinv @ dyT - Sc @ dlam
                    ddy = Wi @ e_T
                    dyT = dyT + ddy
                    dlam = dlam + (Sc.T @ ddy) / d4
                d4_true = nu4 / lam
                for _ in range(TERM_REFINE if np.min(d4_true) < d4_floor else 0):
                    # iterative refinement of (dlam, dy1) for the given dx_N: residual of the terminal block in
                    # INFORMATION form with the TRUE barrier diagonal, correction by the floored covariance-form solve
                    yTi = T @ (dx[N] - Sc @ dlam - sbar * np.sum(dlam))
                    e_l = rho_l - (d4_true * dlam - Sc.T @ yTi + dy1t)
                    e_1 = -rone - np.sum(dlam)
                    cc1 = -SD @ e_l - sbar * e_1
                    cyT = Wi @ cc1
                    cy1 = -(e_1 - np.sum(e_l / d4)) / delta
                    dlam = dlam + (e_l + Sc.T @ cyT - cy1) / d4
                    dy1t = dy1t + cy1
                if EXACT_TERMINAL_RECOVERY:
                    # experiment: information-form recovery of (dlam, dy1) given dx_N (dense bordered solve)
                    Kb = np.zeros((m + 1, m + 1))
                    Kb[:m, :m] = np.diag(nu4 / lam) + SS.T @ T @ SS
                    Kb[:m, m] = 1.0
                    Kb[m, :m] = 1.0
                    sol_ = np.linalg.solve(Kb, np.concatenate([rho_l + SS.T @ (T @ dx[N]), [-rone]]))
                    dlam = sol_[:m]
                dyT = T @ (dx[N] - SS @ dlam)
                dy1 = dy1t + sbar @ dyT
                if EXACT_TERMINAL_RECOVERY:
                    dy1 = sol_[m]
                dxi = np.zeros(n)
                dnu4 = (-rc4 - nu4 * dlam) / lam
                out.update(dy1=dy1, dyT=dyT, dlam=dlam, dxi=dxi, dnu4=dnu4)
            return out

        def max_step(st, cap=1.0):
            al = cap
            pairs = [(w1, st["dw1"]), (w2, st["dw2"]), (s, st["ds"]), (nu1, st["dnu1"]),
                     (nu2, st["dnu2"]), (nu3, st["dnu3"])]
            if lmpc:
                pairs += [(lam, st["dlam"]), (nu4, st["dnu4"])]
            for v, dv_ in pairs:
                neg = dv_ < 0
                if np.any(neg):
                    al = min(al, np.min(-v[neg] / dv_[neg]))
            return al

        # ---- predictor ---------------------------------------------------------------
        aff = solve_rhs(w1 * nu1, w2 * nu2, s * nu3, (lam * nu4) if lmpc else None)
        a_aff = max_step(aff)
        comp_aff = (np.sum((w1 + a_aff * aff["dw1"]) * (nu1 + a_aff * aff["dnu1"]))
                    + np.sum((w2 + a_aff * aff["dw2"]) * (nu2 + a_aff * aff["dnu2"]))
                    + np.sum((s + a_aff * aff["ds"]) * (nu3 + a_aff * aff["dnu3"])))
        if lmpc:
            comp_aff += np.sum((lam + a_aff * aff["dlam"]) * (nu4 + a_aff * aff["dnu4"]))
        sigma = (comp_aff / comp) ** 3
        # ---- corrector ---------------------------------------------------------------
        sm = sigma * mu
        cc = solve_rhs(w1 * nu1 + aff["dw1"] * aff["dnu1"] - sm, w2 * nu2 + aff["dw2"] * aff["dnu2"] - sm,
                       s * nu3 + aff["ds"] * aff["dnu3"] - sm,
                       (lam * nu4 + aff["dlam"] * aff["dnu4"] - sm) if lmpc else None)
        al = min(1.0, step * max_step(cc, 1e300))         # as the kernel: full step when the boundary is > 1/step away
        if gamma > 0.0:
            # stay in a wide neighbourhood of the central path: min_i w_i nu_i >= gamma * mu
            def prods(a):
                pr = [((w1 + a * cc["dw1"]) * (nu1 + a * cc["dnu1"])).ravel(), ((w2 + a * cc["dw2"]) * (nu2 + a * cc["dnu2"])).ravel(),
                      ((s + a * cc["ds"]) * (nu3 + a * cc["dnu3"])).ravel()]
                if lmpc:
                    pr.append((lam + a * cc["dlam"]) * (nu4 + a * cc["dnu4"]))
                return np.concatenate(pr)
            ok_nb = False
            for tr in range(12):
                pr = prods(al)
                if pr.min() >= gamma * pr.mean():
                    ok_nb = True
                    break
                if RECENTER and tr >= RECENTER_AFTER:
                    break
                al *= backoff
            if verbose and not ok_nb:
                p0 = prods(0.0)
                print("      neighbourhood backtracking failed: current min/mean %.3e, tries %d" % (p0.min() / p0.mean(), tr))
            if RECENTER and not ok_nb:
                # pure centring step from the same factorisation: sigma = 1, no second-order term
                cc = solve_rhs(w1 * nu1 - mu, w2 * nu2 - mu, s * nu3 - mu, (lam * nu4 - mu) if lmpc else None)
                al = min(1.0, step * max_step(cc, 1e300))
                for tr in range(12):
                    pr = prods(al)
                    if pr.min() >= gamma * pr.mean():
                        break
                    al *= backoff
                if verbose:
                    print("      recentring step alpha %.3f  -> min/mean %.3e" % (al, pr.min() / pr.mean()))
        if DEBUG_HOOK:
            # residual of the u-rows and lambda-rows of the Newton system for the corrector step
            dx_, du_ = cc["dx"], cc["du"]
            mu_c = np.zeros((N + 1, n))
            mu_c[N] = Qf2 @ dx_[N] + (cc["dyT"] if lmpc else 0.0)
            rc1 = w1 * nu1 + aff["dw1"] * aff["dnu1"] - sm
            rc3 = s * nu3 + aff["ds"] * aff["dnu3"] - sm
            rc2 = w2 * nu2 + aff["dw2"] * aff["dnu2"] - sm
            e1 = -rc1 / w1 + d1 * r1
            ex = (e1 * (2 * qp.qs_quad + d3) + d1 * (rs + rc3 / s)) / hs
            eu = -rc2 / w2 + d2 * r2
            for k in range(N - 1, 0, -1):
                mu_c[k] = Hxx[k] @ dx_[k] + Fx.T @ ex[k] + A[k].T @ mu_c[k + 1]
            worst_u = 0.0
            for k in range(N):
                e = ru[k] + Fu.T @ eu[k] + Huu[k] @ du_[k] + B[k].T @ mu_c[k + 1]
                if k > 0: e -= dR2 * du_[k - 1]
                if k < N - 1: e -= dR2 * du_[k + 1]
                worst_u = max(worst_u, np.abs(e).max())
            prods = np.concatenate([(w1 * nu1).ravel(), (w2 * nu2).ravel(), (s * nu3).ravel()] + ([lam * nu4] if lmpc else []))
            msg = "   newton-resid u %.2e  a_aff %.3f sigma %.2e alpha %.4f  min(prod)/mu %.2e max %.2e" % (worst_u, a_aff, sigma, al, prods.min() / mu, prods.max() / mu)
            if lmpc:
                rc4 = lam * nu4 + aff["dlam"] * aff["dnu4"] - sm
                e_l = (nu4 / lam) * cc["dlam"] - SS.T @ cc["dyT"] + cc["dy1"] - (-rlam - rc4 / lam)
                msg += " lam %.2e  |dlam| %.2e |dyT| %.2e |dxN| %.2e alpha %.3f sigma %.2e minD4 %.1e" % (np.abs(e_l).max(), np.abs(cc["dlam"]).max(), np.abs(cc["dyT"]).max(), np.abs(dx_[N]).max(), al, sigma, (nu4/lam).min())
            print(msg)
        al_prev = al
        step_prev = al * max(np.abs(cc["dx"]).max(), np.abs(cc["du"]).max())
        x = x + al * cc["dx"]
        u = u + al * cc["du"]
        s = s + al * cc["ds"]
        w1 = w1 + al * cc["dw1"]
        w2 = w2 + al * cc["dw2"]
        nu1, nu2, nu3 = nu1 + al * cc["dnu1"], nu2 + al * cc["dnu2"], nu3 + al * cc["dnu3"]
        if lmpc:
            lam, xi = lam + al * cc["dlam"], xi + al * cc["dxi"]
            yT, y1, nu4 = yT + al * cc["dyT"], y1 + al * cc["dy1"], nu4 + al * cc["dnu4"]

    out = dict(x=x, u=u, s=s, iters=it, r_prim=r_prim, r_dual=r_dual, gap=mu, status=status, snap=snap)
    if lmpc:
        out.update(lam=lam, xi=xi)
    return out


def pack(qp, sol):
    """Decision vector in the reference's order (PC.py:251,361,365-375)."""
    parts = [sol["x"].ravel(), sol["u"].ravel(), sol["s"].ravel()]
    if qp.m:
        parts += [sol["lam"], sol["xi"]]
    return np.concatenate(parts)
