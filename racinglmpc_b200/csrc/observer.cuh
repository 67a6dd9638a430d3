// racinglmpc_b200/csrc/observer.cuh — the per-controller state observers (DESIGN.md, "Per-controller state observers",
// "Observer priors", "Observer gains"): the model prior, the model-based gain and the blend.
#pragma once
#include "safeset.cuh"
#include "lap_schedule.cuh"
#include "car.cuh"

namespace lmpc {

// ------------------------------------------------------------------------------------------------
// State observers (DESIGN.md, "Per-controller state observers"): the state x_hat a controller reads, blended from the state it
// is given, y, and its own one-step prediction p = xPred[1] of its previous QP (row 1 of xPredPrev), with the fixed gains of its
// row: x_hat_j = p_j + l_j (y_j - p_j), each operation rounded on its own (no contraction), l_j == 1 copying y_j and l_j == 0
// taking p_j.  p_s gets K2's lap-wrap fix first.  No prior (has_pred == 0), a mode 0 row or a step that is not an LMPC / LTV step
// gives x_hat = y exactly; a non-finite prior on a channel with l_j < 1 gives x_hat = y and LMPC_FLAG_OBSERVER_RESET.  In a PID
// or LTI step (blend == 0) a mode 1 row also clears has_pred: xPredPrev is not shifted there and would be stale next step.  One
// thread per controller; a retired controller reads, writes and flags nothing.  The observer has no state of its own.
// MODEL (a prior table is installed, DESIGN.md, "Observer priors"): a row of source 1 or 2 takes the model prior
// p = Phi_car(xPredPrev[0], OldInput) (sim_period) in place of the plan, and the kernel writes the prior it formed to x_prior.
struct ObserveArgs {
    int batch, N;
    int blend;                     // 1: a step of mode 0 or 1; 0: a PID step or a step of mode 2
    const double* y;               // [B][6] the state the controllers are given (x_meas, or the plant state)
    const double* xPredPrev;       // [B][N+1][6] the previous QP's prediction
    int* has_pred;                 // [B]
    double* x_est;                 // [B][6] x_hat
    int* flags;                    // [B] step flags, cleared before this launch (blend == 1)
    Table<lmpc_observer_params> obs;
    Tracks trk;
    LapBudget retire;
};
// What the MODEL instantiation reads besides (a second kernel parameter: the instantiation without a prior table keeps the code
// it had before this feature)
struct ObservePrior {
    Table<lmpc_observer_prior_params> pri;   // the prior source of every controller
    double dt;                               // the control period (ModelConst::dt)
    const double* OldInput;                  // [B][2] the input applied in the previous step
    double* x_prior;                         // [B][6] the prior formed (NaN: none)
    Table<lmpc_vehicle_params> veh;          // the simulator's vehicle table and lap schedule (source 2)
    LapSchedule veh_s;
    Table<lmpc_surface_params> surf;         // the simulator's surface table (tab null: none) and lap schedule (source 2)
    LapSchedule surf_s;
};

// The model prior of controller b (source 1: the row's car, no surface; source 2: the car and surface the plant drove the
// previous step with -- the lap before lap_n when a hand-over came in between, seen as x_hat_{k-1}.s - y.s > TrackLength / 2).
// false when an input is not finite or a curvature lookup failed.  observer_gain_kernel picks the same point and rows with its
// own copy of these lines: a helper shared by both (a struct or out-parameters) changed the SASS of observe_kernel<true, *>.
__device__ __forceinline__ bool model_prior(const ObserveArgs& a, const ObservePrior& m, int b, const lmpc_observer_prior_params& r,
                                            const double (&yv)[6], double (&p)[6]) {
    const double* xp = a.xPredPrev + (size_t)b * (a.N + 1) * 6;
    const double delta = m.OldInput[(size_t)b * 2], acc = m.OldInput[(size_t)b * 2 + 1];
    bool finite = isfinite(delta) && isfinite(acc);
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        p[j] = xp[j];
        finite = finite && isfinite(p[j]);
    }
    const TrackRec& trk = a.trk.of(b);
    const int back = p[4] - yv[4] > trk.TrackLength / 2 ? 1 : 0;
    const bool plant = r.source == 2;
    const lmpc_vehicle_params& v = plant ? m.veh_s.of_before(m.veh, b, back) : r.vehicle;
    const lmpc_surface_params* zones = plant && m.surf.tab ? &m.surf_s.of_before(m.surf, b, back) : nullptr;
    return sim_period(v, trk, zones, m.dt, delta, acc, p) && finite;
}

// ------------------------------------------------------------------------------------------------
// Model-based observer gains (DESIGN.md, "Observer gains"): the frozen-time Kalman gain of every mode 1 row of the gain table.
// observer_gain_kernel linearises the controller's one-period map at the prior's point, A = dPhi_car/dx (sim_period_tangent),
// solves the filter DARE P = A P A' - A P (P + R)^-1 P A' + Q for that A (observer_dare), and writes A, P and K = P (P + R)^-1;
// observe_kernel<true, true> then blends with K.  Nothing is carried from step to step: the gain is a function of the step's own
// inputs (xPredPrev[0], OldInput, y and the rows), so it adds no state and no snapshot section.
struct ObserveGain {
    Table<lmpc_observer_gain_params> gains;   // the gain row of every controller
    double* jac;                              // [B][6][6] A (NaN: no model gain formed)
    double* cov;                              // [B][6][6] P
    double* gain;                             // [B][6][6] K (NaN: none formed, or A, P or K not finite, or no convergence)
};
constexpr int OBS_DARE_ITERS = 64;            // the doubling's iteration cap
constexpr double OBS_DARE_TOL = 1e-13;        // stop once max|H' - H| <= tol max|H'|

// One sub-step of sim_substep<false> with the tangent (dvx .. dey) of one direction carried alongside: the primal is computed by
// the same expressions, and the tangent differentiates them.  The curvature (piecewise constant in s) and the sub-step's peak
// tyre forces Dfi, Dri (piecewise constant in s through the surface zones) are taken as constants.  The inputs are not
// differentiated.  It restates the primal of car.cuh's sub-step rather than calling its pieces: built on them, observer_gain_kernel
// went from 168 registers without spills to 128 registers with 52 bytes of spill stores.
__device__ __forceinline__ void sim_substep_tangent(double mass, double lf, double lr, double Iz, double Dfi, double Cf, double Bf,
                                                    double Dri, double Cr, double Br, double delta, double acc, double sd,
                                                    double cd, double h, const TrackRec& trk, int* okc, double (&x)[6],
                                                    double (&d)[6]) {
    const double vx = x[0], vy = x[1], wz = x[2], epsi = x[3], s = x[4], ey = x[5];
    const double dvx = d[0], dvy = d[1], dwz = d[2], depsi = d[3], ds = d[4], dey = d[5];
    const double yf = vy + lf * wz, yr = vy - lf * wz;
    const double af = delta - atan2(yf, vx);
    const double ar = -atan2(yr, vx);
    const double daf = -(vx * (dvy + lf * dwz) - yf * dvx) / (vx * vx + yf * yf);
    const double dar = -(vx * (dvy - lf * dwz) - yr * dvx) / (vx * vx + yr * yr);
    const double tf = Cf * atan(Bf * af), tr = Cr * atan(Br * ar);
    const double Fyf = Dfi * sin(tf);
    const double Fyr = Dri * sin(tr);
    const double dFyf = Dfi * cos(tf) * Cf * Bf / (1 + Bf * af * Bf * af) * daf;
    const double dFyr = Dri * cos(tr) * Cr * Br / (1 + Br * ar * Br * ar) * dar;
    const double nvx = vx + h * (acc - 1 / mass * Fyf * sd + wz * vy);
    const double nvy = vy + h * (1 / mass * (Fyf * cd + Fyr) - wz * vx);
    const double nwz = wz + h * (1 / Iz * (lf * Fyf * cd - lr * Fyr));
    d[0] = dvx + h * (-(1 / mass) * dFyf * sd + dwz * vy + wz * dvy);
    d[1] = dvy + h * (1 / mass * (dFyf * cd + dFyr) - dwz * vx - wz * dvx);
    d[2] = dwz + h * (1 / Iz * (lf * dFyf * cd - lr * dFyr));
    const double cur = curvature_lookup(trk, s, okc);
    const double ce = cos(epsi), se = sin(epsi);
    const double den = 1 - cur * ey;
    const double q = (vx * ce - vy * se) / den;
    const double dnum = dvx * ce - vx * se * depsi - dvy * se - vy * ce * depsi;
    const double dq = (dnum + q * cur * dey) / den;
    const double nepsi = epsi + h * (wz - (vx * ce - vy * se) / (1 - cur * ey) * cur);
    const double ns = s + h * ((vx * ce - vy * se) / (1 - cur * ey));
    const double ney = ey + h * (vx * se + vy * ce);
    d[3] = depsi + h * (dwz - dq * cur);
    d[4] = ds + h * dq;
    d[5] = dey + h * (dvx * se + vx * ce * depsi + dvy * ce - vy * se * depsi);
    x[0] = nvx; x[1] = nvy; x[2] = nwz; x[3] = nepsi; x[4] = ns; x[5] = ney;
}

// sim_period with the tangent d of one direction: x and d in, Phi_car(x) and A d out.  false when a curvature lookup failed.
__device__ __forceinline__ bool sim_period_tangent(const lmpc_vehicle_params& v, const TrackRec& trk, const lmpc_surface_params* zones,
                                                   double dt, double delta, double acc, double (&x)[6], double (&d)[6]) {
    const double h = CAR_H;
    const double sd = sin(delta), cd = cos(delta);
    int i = 0;
    int okc = 1;
    SurfaceCursor zc{zones, 0};
    while ((i + 1) * h <= dt) {
        double Dfi = v.Df, Dri = v.Dr;
        if (zones) surface_forces(zc, x[4], trk.TrackLength, v.Df, v.Dr, &Dfi, &Dri);
        sim_substep_tangent(v.m, v.lf, v.lr, v.Iz, Dfi, v.Cf, v.Bf, Dri, v.Cr, v.Br, delta, acc, sd, cd, h, trk, &okc, x, d);
        ++i;
    }
    return okc != 0;
}

// Gauss-Jordan elimination with partial pivoting of one controller's 6 x NC system in shared memory, M[6][NC] = [S | RHS]: lane r
// of the controller's six owns row r and every lane picks the same pivots.  On return the solution row k, S^-1 RHS, is row
// piv[k] of M (columns 6 .. NC - 1).  Every lane of the warp calls it (active or not): it synchronises the warp.
template <int NC>
__device__ __forceinline__ void gj_solve(double* M, int r, bool active, int (&piv)[6]) {
    unsigned used = 0;
#pragma unroll 1
    for (int k = 0; k < 6; ++k) {
        int pk = 0;
        double best = -1.0;
        for (int i = 0; i < 6; ++i) {
            const double v = fabs(M[i * NC + k]);
            if (!(used & (1u << i)) && v > best) { best = v; pk = i; }
        }
        piv[k] = pk;
        used |= 1u << pk;
        __syncwarp();
        if (active && r == pk) {
            const double inv = 1.0 / M[pk * NC + k];
            for (int c = 0; c < NC; ++c) M[pk * NC + c] *= inv;
        }
        __syncwarp();
        double f = 0.0;
        if (active && r != pk) f = M[r * NC + k];
        __syncwarp();
        if (active && r != pk)
            for (int c = 0; c < NC; ++c) M[r * NC + c] -= f * M[pk * NC + c];
        __syncwarp();
    }
}

// The filter DARE of one controller by the structured doubling algorithm on the dual (control) problem: A0 = A', G0 = R^-1,
// H0 = Q; W = I + G H; A <- A W^-1 A, G <- G + A W^-1 G A', H <- H + A' H W^-1 A; H converges to P.  Lane r owns row r of the
// controller's matrices in shared memory: At (A0, then the iterates), G, H, the 6 x 18 system [W | A | G] and U = H W^-1 A.  The
// iteration stops once max|H' - H| <= OBS_DARE_TOL max|H'| (true), or after OBS_DARE_ITERS (false).  Every lane of the warp takes
// the same number of iterations (a controller that has converged, or is not active, idles through them): the warp synchronises.
struct DareSmem {
    double At[36], G[36], H[36], M[6 * 18], U[36], red[6];
};
__device__ __forceinline__ bool observer_dare(DareSmem& S, int r, bool active) {
    bool done = !active, conv = false;
#pragma unroll 1
    for (int it = 0; it < OBS_DARE_ITERS; ++it) {
        if (!__any_sync(0xffffffffu, !done)) break;
        const bool go = !done;
        if (go) {   // [W | A | G], row r
            for (int c = 0; c < 6; ++c) {
                double w = r == c ? 1.0 : 0.0;
                for (int k = 0; k < 6; ++k) w += S.G[r * 6 + k] * S.H[k * 6 + c];
                S.M[r * 18 + c] = w;
                S.M[r * 18 + 6 + c] = S.At[r * 6 + c];
                S.M[r * 18 + 12 + c] = S.G[r * 6 + c];
            }
        }
        __syncwarp();
        int piv[6];
        gj_solve<18>(S.M, r, go, piv);
        // X1 = W^-1 A (row k: M[piv[k]][6..11]), X2 = W^-1 G (M[piv[k]][12..17])
        double An[6], T[6], Gn[6];
        if (go) {
            for (int c = 0; c < 6; ++c) {
                double a = 0.0, t = 0.0, u = 0.0;
                for (int k = 0; k < 6; ++k) {
                    a += S.At[r * 6 + k] * S.M[piv[k] * 18 + 6 + c];
                    t += S.At[r * 6 + k] * S.M[piv[k] * 18 + 12 + c];
                    u += S.H[r * 6 + k] * S.M[piv[k] * 18 + 6 + c];
                }
                An[c] = a; T[c] = t;
                S.U[r * 6 + c] = u;
            }
            for (int c = 0; c < 6; ++c) {
                double g = S.G[r * 6 + c];
                for (int k = 0; k < 6; ++k) g += T[k] * S.At[c * 6 + k];
                Gn[c] = g;
            }
        }
        __syncwarp();
        double Hn[6], dmax = 0.0, hmax = 0.0;
        if (go) {
            for (int c = 0; c < 6; ++c) {
                double v = S.H[r * 6 + c];
                for (int k = 0; k < 6; ++k) v += S.At[k * 6 + r] * S.U[k * 6 + c];
                Hn[c] = v;
                dmax = fmax(dmax, fabs(v - S.H[r * 6 + c]));
                hmax = fmax(hmax, fabs(v));
            }
        }
        __syncwarp();
        if (go) {
            for (int c = 0; c < 6; ++c) { S.At[r * 6 + c] = An[c]; S.G[r * 6 + c] = Gn[c]; S.H[r * 6 + c] = Hn[c]; }
            S.red[r] = dmax <= OBS_DARE_TOL * hmax ? 1.0 : 0.0;   // NaN or inf anywhere: not converged
        }
        __syncwarp();
        if (go) {
            bool all = true;
            for (int k = 0; k < 6; ++k) all = all && S.red[k] == 1.0;
            if (all) { done = true; conv = true; }
        }
        __syncwarp();
    }
    return conv;
}

// Five controllers per warp, six lanes each (lanes 30, 31 idle); lane r of a controller carries the prior's primal and the tangent
// of direction e_r through the period (column r of A), then owns row r in the DARE and the gain.  A controller forms a model gain
// when it is not retired, its observer row is mode 1 with has_pred == 1, its gain row is mode 1 and its prior row is source 1 or
// 2, and the prior's inputs are finite and its curvature lookups succeed (else observe_kernel sets LMPC_FLAG_OBSERVER_RESET).
// Every controller that is not retired gets all three [6][6] outputs: NaN where no gain was formed.  Launched only in rollout
// steps of mode 0 and 1, between the measurement and the observer kernels.
constexpr int OBS_GAIN_WARPS = 2;                 // warps per block
constexpr int OBS_GAIN_PER_WARP = 5;
__global__ void __launch_bounds__(32 * OBS_GAIN_WARPS) observer_gain_kernel(const ObserveArgs a, const ObservePrior m,
                                                                           const ObserveGain g) {
    __shared__ DareSmem sm[OBS_GAIN_WARPS * OBS_GAIN_PER_WARP];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int grp = lane / 6, r = lane - grp * 6;
    const int slot = warp * OBS_GAIN_PER_WARP + min(grp, OBS_GAIN_PER_WARP - 1);
    const int b = (blockIdx.x * OBS_GAIN_WARPS + warp) * OBS_GAIN_PER_WARP + grp;
    const bool mine = grp < OBS_GAIN_PER_WARP && b < a.batch && !a.retire.retired(b);
    DareSmem& S = sm[slot];
    bool form = mine && a.obs.of(b).mode == 1 && a.has_pred[b] && m.pri.tab && g.gains.of(b).mode == 1 && m.pri.of(b).source != 0;
    double x[6], d[6];
    if (form) {                                  // the prior's point and car, as model_prior picks them
        const lmpc_observer_prior_params& pr = m.pri.of(b);
        const double* xp = a.xPredPrev + (size_t)b * (a.N + 1) * 6;
        const double delta = m.OldInput[(size_t)b * 2], acc = m.OldInput[(size_t)b * 2 + 1];
        bool finite = isfinite(delta) && isfinite(acc);
        for (int j = 0; j < 6; ++j) {
            x[j] = xp[j];
            d[j] = j == r ? 1.0 : 0.0;
            finite = finite && isfinite(x[j]);
        }
        const TrackRec& trk = a.trk.of(b);
        const int back = x[4] - a.y[(size_t)b * 6 + 4] > trk.TrackLength / 2 ? 1 : 0;
        const bool plant = pr.source == 2;
        const lmpc_vehicle_params& v = plant ? m.veh_s.of_before(m.veh, b, back) : pr.vehicle;
        const lmpc_surface_params* zones = plant && m.surf.tab ? &m.surf_s.of_before(m.surf, b, back) : nullptr;
        form = finite && sim_period_tangent(v, trk, zones, m.dt, delta, acc, x, d);
        for (int j = 0; j < 6; ++j) form = form && isfinite(x[j]);
    }
    // every lane of a controller takes the same decision
    const unsigned ok = __ballot_sync(0xffffffffu, form);
    form = mine && ((ok >> (grp * 6)) & 0x3fu) == 0x3fu;
    bool fin = true;
    if (form) {
        const lmpc_observer_gain_params& gp = g.gains.of(b);
        for (int c = 0; c < 6; ++c) {
            S.At[r * 6 + c] = d[c];              // A0 = A': row r is the tangent of direction r
            S.G[r * 6 + c] = r == c ? 1.0 / gp.r[r] : 0.0;
            S.H[r * 6 + c] = r == c ? gp.q[r] : 0.0;
            fin = fin && isfinite(d[c]);
        }
    }
    const unsigned fa = __ballot_sync(0xffffffffu, fin);
    const bool jac_ok = ((fa >> (grp * 6)) & 0x3fu) == 0x3fu;
    __syncwarp();
    const bool conv = observer_dare(S, r, form && jac_ok);
    // P = (H + H') / 2, then K = P (P + R)^-1 = (S^-1 P)' with S = P + R: the system [S | P]
    double P[6];
    if (form && jac_ok) {
        const lmpc_observer_gain_params& gp = g.gains.of(b);
        for (int c = 0; c < 6; ++c) P[c] = 0.5 * (S.H[r * 6 + c] + S.H[c * 6 + r]);
        for (int c = 0; c < 6; ++c) {
            S.M[r * 12 + c] = r == c ? P[c] + gp.r[r] : P[c];
            S.M[r * 12 + 6 + c] = P[c];
        }
    }
    __syncwarp();
    int piv[6];
    gj_solve<12>(S.M, r, form && jac_ok && conv, piv);
    if (!mine) return;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    double* J = g.jac + (size_t)b * 36;
    double* C = g.cov + (size_t)b * 36;
    double* K = g.gain + (size_t)b * 36;
    double Kr[6];
    bool good = form && jac_ok && conv;
    for (int c = 0; c < 6; ++c) {
        Kr[c] = good ? S.M[piv[c] * 12 + 6 + r] : nan;
        good = good && isfinite(Kr[c]) && isfinite(P[c]);
    }
    const unsigned gb = __ballot_sync(__activemask(), good);
    good = ((gb >> (grp * 6)) & 0x3fu) == 0x3fu;
    for (int c = 0; c < 6; ++c) {
        J[c * 6 + r] = form ? d[c] : nan;        // column r of A
        C[r * 6 + c] = form && jac_ok ? P[c] : nan;
        K[r * 6 + c] = good ? Kr[c] : nan;
    }
}

template <bool MODEL, bool GAIN>
__global__ void observe_kernel(const ObserveArgs a, const ObservePrior m, const ObserveGain g) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.batch || a.retire.retired(b)) return;
    const lmpc_observer_params& o = a.obs.of(b);
    const double* y = a.y + (size_t)b * 6;
    double* xe = a.x_est + (size_t)b * 6;
    const bool on = o.mode == 1;
    if (on && !a.blend) a.has_pred[b] = 0;
    double yv[6], p[6];
#pragma unroll
    for (int j = 0; j < 6; ++j) yv[j] = y[j];
    bool prior = on && a.blend && a.has_pred[b];
    bool kal = false;            // GAIN: a mode 1 gain row blends with the model gain K; its fixed gains are not read
    if constexpr (GAIN) kal = on && g.gains.of(b).mode == 1;
    if constexpr (MODEL) {       // a row whose gains are all 1 forms no prior
        bool reads = kal;
#pragma unroll
        for (int j = 0; j < 6; ++j) reads = reads || o.gain[j] != 1.0;
        prior = prior && reads;
    }
    const bool formed = prior;
    if (prior) {
        bool model = false, ok = true;
        if constexpr (MODEL) {
            const lmpc_observer_prior_params& r = m.pri.of(b);
            model = r.source != 0;
            if (model) ok = model_prior(a, m, b, r, yv, p);
        }
        if (!model) {
            const double* pp = a.xPredPrev + ((size_t)b * (a.N + 1) + 1) * 6;
#pragma unroll
            for (int j = 0; j < 6; ++j) p[j] = pp[j];
        }
        wrap_guess_s(p[4], yv[4], a.trk.of(b).TrackLength);
        bool finite = ok;
#pragma unroll
        for (int j = 0; j < 6; ++j) finite = finite && ((!kal && o.gain[j] == 1.0) || isfinite(p[j]));
        if (!finite) {
            a.flags[b] |= LMPC_FLAG_OBSERVER_RESET;
            prior = false;
        }
    }
    if constexpr (MODEL) {
        double* xq = m.x_prior + (size_t)b * 6;
#pragma unroll
        for (int j = 0; j < 6; ++j) xq[j] = formed ? p[j] : __longlong_as_double(0x7ff8000000000000ll);
    }
    if constexpr (GAIN) {
        if (!a.blend) {          // observer_gain_kernel does not run in PID and mode 2 steps: no gain was formed
            const double nan = __longlong_as_double(0x7ff8000000000000ll);
            for (int e = 0; e < 36; ++e) {
                g.jac[(size_t)b * 36 + e] = nan; g.cov[(size_t)b * 36 + e] = nan; g.gain[(size_t)b * 36 + e] = nan;
            }
        }
        if (kal) {               // x_hat_i = p_i + sum_j K_ij (y_j - p_j), left to right, each operation rounded on its own
            if (prior) {
                const double* K = g.gain + (size_t)b * 36;
                bool fin = true;
                for (int e = 0; e < 36; ++e) fin = fin && isfinite(K[e]);
                if (!fin) {
                    a.flags[b] |= LMPC_FLAG_OBSERVER_GAIN;
                    prior = false;
                }
            }
            double e[6];
#pragma unroll
            for (int j = 0; j < 6; ++j) e[j] = prior ? __dsub_rn(yv[j], p[j]) : 0.0;
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                double v = yv[i];
                if (prior) {
                    const double* K = g.gain + (size_t)b * 36 + i * 6;
                    double c = __dmul_rn(K[0], e[0]);
#pragma unroll
                    for (int j = 1; j < 6; ++j) c = __dadd_rn(c, __dmul_rn(K[j], e[j]));
                    v = __dadd_rn(p[i], c);
                }
                xe[i] = v;
            }
            return;
        }
    }
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        const double l = o.gain[j];
        double v = yv[j];
        if (prior && l != 1.0) v = l == 0.0 ? p[j] : __dadd_rn(p[j], __dmul_rn(l, __dsub_rn(yv[j], p[j])));
        xe[j] = v;
    }
}

}  // namespace lmpc
