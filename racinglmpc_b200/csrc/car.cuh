// racinglmpc_b200/csrc/car.cuh — the car: one control period of Simulator.dynModel (SysModel.py:56-137) on the track, defined
// once for every kernel that drives or linearises it.
//
//   sim_step_kernel (plant.cuh)             sim_substep<true> in period_substeps<SURF>
//   the observer's model prior              sim_period: sim_substep<false>
//   nominal_model_kernel                    tyre_forces, velocity_update, kinematic_update and their 3 x 5 sensitivity;
//                                           kinematic_rows
//   K1 (safeset.cuh)                        kinematic_rows
//
// The derivative formulas stay with their kernels: the nominal model's matrix form and the observer's directional form
// (sim_substep_tangent, observer.cuh) round differently, and each is pinned by its own tests.
#pragma once
#include <math.h>
#include "../../include/lmpc_b200.h"

namespace lmpc {

// The track of every controller (lmpc_set_tracks; default: the track of lmpc_store_create); the ABI record is the device record.
using TrackRec = lmpc_track_params;

// Track.py:292-310 — wrap by repeated subtraction, first segment with s in [s0, s0+len)
// (a non-finite or absurdly large s -- an unsolved QP feeding garbage to the simulator -- would spin forever in the
// reference's loop; here it fails the lookup like a negative s does, so the instance is flagged instead of hanging the stream)
__device__ __forceinline__ double curvature_lookup(const TrackRec& m, double s, int* ok) {
    if (!(s <= 64.0 * m.TrackLength)) { *ok = 0; return 0.0; }
    while (s > m.TrackLength) s = s - m.TrackLength;
    for (int i = 0; i < m.nseg; ++i) {
        double s0 = m.seg[i * 3], ln = m.seg[i * 3 + 1];
        if (s >= s0 && s < s0 + ln) return m.seg[i * 3 + 2];
    }
    *ok = 0;   // the reference raises here (negative s / exact end point)
    return 0.0;
}

// 1 / x for a normal, finite x to ~1 ulp: hardware seed (20 bits) + two Newton steps; no slow-path call, so no registers are
// parked in local memory around it
__device__ __forceinline__ double fast_rcp(double x) {
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    r = fma(fma(-x, r, 1.0), r, r);
    return fma(fma(-x, r, 1.0), r, r);
}

// Track surfaces (lmpc_rollout_set_surfaces): the zone of one controller's sub-steps, found by a cursor that follows s.  The
// zones of a row ascend without overlap, so their s_end ascend strictly, and the first zone whose s_end lies above the wrapped s
// is the only one that can hold it.  The cursor walks to that zone from where the last sub-step left it (s moves by at most
// vx h per sub-step), in either direction, so it returns what a scan of every zone returns at any s.
struct SurfaceCursor {
    const lmpc_surface_params* row;
    int c;
    // true and the zone's (mu_f, mu_r) when a zone holds s, wrapped as curvature_lookup wraps it; false when none does, s is not
    // finite or s is beyond 64 laps
    __device__ __forceinline__ bool at(double s, double L, double* muf, double* mur) {
        if (!(s <= 64.0 * L)) return false;
        while (s > L) s = s - L;
        const double* z = row->zone;
        const int n = row->nzone;
        while (c > 0 && z[(c - 1) * 4 + 1] > s) --c;
        while (c < n && z[c * 4 + 1] <= s) ++c;
        if (c >= n || !(z[c * 4] <= s)) return false;
        *muf = z[c * 4 + 2];
        *mur = z[c * 4 + 3];
        return true;
    }
};

// The peak tyre forces of a sub-step at s: fl(mu_f Df), fl(mu_r Dr) in a zone, else Df and Dr exactly
__device__ __forceinline__ void surface_forces(SurfaceCursor& zc, double s, double L, double Df, double Dr, double* Dfi, double* Dri) {
    double muf, mur;
    if (zc.at(s, L, &muf, &mur)) {
        *Dfi = __dmul_rn(muf, Df);
        *Dri = __dmul_rn(mur, Dr);
    } else {
        *Dfi = Df;
        *Dri = Dr;
    }
}

// ---- one explicit-Euler sub-step (SysModel.py:94-137), in pieces: every piece reads the sub-step's starting state ----

constexpr double CAR_H = 0.001;   // the sub-step (SysModel.py:83)

// The lateral tyre forces (SysModel.py:94-97), with the reference's lf in alpha_r, and their intermediates: yf, yr the atan2
// numerators, af, ar the slip angles, tf = atan(Bf af), tr = atan(Br ar).  Dfi, Dri are the sub-step's peak forces.
struct Tyres {
    double yf, yr, af, ar, tf, tr, Fyf, Fyr;
};
__device__ __forceinline__ Tyres tyre_forces(double lf, double Dfi, double Cf, double Bf, double Dri, double Cr, double Br,
                                             double delta, double vx, double vy, double wz) {
    Tyres t;
    t.yf = vy + lf * wz;
    t.af = delta - atan2(t.yf, vx);
    t.yr = vy - lf * wz;
    t.ar = -atan2(t.yr, vx);
    t.tf = atan(Bf * t.af);
    t.Fyf = Dfi * sin(Cf * t.tf);
    t.tr = atan(Br * t.ar);
    t.Fyr = Dri * sin(Cr * t.tr);
    return t;
}

// The updated (vx, vy, wz) (SysModel.py:98-106) under the forces t; sd, cd = sin, cos(delta)
struct Velocities {
    double vx, vy, wz;
};
__device__ __forceinline__ Velocities velocity_update(double mass, double lf, double lr, double Iz, double acc, double sd, double cd,
                                                      double h, const Tyres& t, double vx, double vy, double wz) {
    Velocities n;
    n.vx = vx + h * (acc - 1 / mass * t.Fyf * sd + wz * vy);
    n.vy = vy + h * (1 / mass * (t.Fyf * cd + t.Fyr) - wz * vx);
    n.wz = wz + h * (1 / Iz * (lf * t.Fyf * cd - lr * t.Fyr));
    return n;
}

// The updated (epsi, s, ey) (SysModel.py:107-110) with the curvature at s and ce, se = cos, sin(epsi) it used.  A failed curvature
// lookup clears *okc and goes on with curvature 0.
struct Kinematics {
    double cur, ce, se, epsi, s, ey;
};
__device__ __forceinline__ Kinematics kinematic_update(const TrackRec& trk, int* okc, double h, double vx, double vy, double wz,
                                                       double epsi, double s, double ey) {
    Kinematics k;
    k.cur = curvature_lookup(trk, s, okc);
    k.ce = cos(epsi);
    k.se = sin(epsi);
    k.epsi = epsi + h * (wz - (vx * k.ce - vy * k.se) / (1 - k.cur * ey) * k.cur);
    k.s = s + h * ((vx * k.ce - vy * k.se) / (1 - k.cur * ey));
    k.ey = ey + h * (vx * k.se + vy * k.ce);
    return k;
}

// One sub-step: the curvilinear state (vx, vy, wz, epsi, s, ey) and, GLOBAL, the global pose (psi, X, Y).  Dfi, Dri are the
// sub-step's peak tyre forces (surface_forces), sd, cd = sin, cos(delta).  A failed curvature lookup clears *okc.
template <bool GLOBAL>
__device__ __forceinline__ void sim_substep(double mass, double lf, double lr, double Iz, double Dfi, double Cf, double Bf,
                                            double Dri, double Cr, double Br, double delta, double acc, double sd, double cd,
                                            double h, const TrackRec& trk, int* okc, double& vx, double& vy, double& wz,
                                            double& epsi, double& s, double& ey, double& psi, double& X, double& Y) {
    const Tyres t = tyre_forces(lf, Dfi, Cf, Bf, Dri, Cr, Br, delta, vx, vy, wz);
    const Velocities n = velocity_update(mass, lf, lr, Iz, acc, sd, cd, h, t, vx, vy, wz);
    if constexpr (GLOBAL) {
        const double npsi = psi + h * wz;
        const double nX = X + h * (vx * cos(psi) - vy * sin(psi));
        const double nY = Y + h * (vx * sin(psi) + vy * cos(psi));
        psi = npsi; X = nX; Y = nY;
    }
    const Kinematics k = kinematic_update(trk, okc, h, vx, vy, wz, epsi, s, ey);
    vx = n.vx; vy = n.vy; wz = n.wz; epsi = k.epsi; s = k.s; ey = k.ey;
}

// The sub-steps of one control period (SysModel.py:83): step(Dfi, Dri) for i = 0, 1, .. while (i + 1) CAR_H <= dt, with the
// sub-step's peak tyre forces.  SURF and zoned: they follow the zone of zones that s, the caller's s as it stands before the
// sub-step, lies in on trk (surface_forces); else they are Df and Dr.  Surfaces stay a template flag: a run-time test in this loop
// cost the table-free simulator step 1.5 % per launch on an H100 (DESIGN.md, "Track surfaces").  zones and trk are read only when
// zoned.
template <bool SURF, typename Step>
__device__ __forceinline__ void period_substeps(const double& dt, double Df, double Dr, const lmpc_surface_params* zones, bool zoned,
                                                const TrackRec* trk, const double& s, Step&& step) {
    constexpr double h = CAR_H;
    SurfaceCursor zc{zones, 0};
    int i = 0;
    while ((i + 1) * h <= dt) {
        double Dfi = Df, Dri = Dr;
        if constexpr (SURF) {
            if (zoned) surface_forces(zc, s, trk->TrackLength, Df, Dr, &Dfi, &Dri);
        }
        step(Dfi, Dri);
        ++i;
    }
}

// Phi_car: the simulator's noise-free control period on the curvilinear state x under the input (delta, acc) -- sim_step_kernel's
// sub-steps with car v and, when zones is not null, its surface row, without the global frame.  false when a sub-step's
// curvature lookup failed.  The observer's model prior takes it, so with process noise off the prior is the plant state exactly.
__device__ __forceinline__ bool sim_period(const lmpc_vehicle_params& v, const TrackRec& trk, const lmpc_surface_params* zones,
                                           double dt, double delta, double acc, double (&x)[6]) {
    const double mass = v.m, lf = v.lf, lr = v.lr, Iz = v.Iz;
    const double Df = v.Df, Cf = v.Cf, Bf = v.Bf;
    const double Dr = v.Dr, Cr = v.Cr, Br = v.Br;
    const double sd = sin(delta), cd = cos(delta);
    double vx = x[0], vy = x[1], wz = x[2], epsi = x[3], s = x[4], ey = x[5];
    double psi = 0.0, X = 0.0, Y = 0.0;
    const double h = CAR_H;
    int i = 0;
    int okc = 1;
    SurfaceCursor zc{zones, 0};
    // period_substeps<true> written out: through the helper, observe_kernel<true, *> compiled to other SASS (DESIGN.md,
    // "Observer priors")
    while ((i + 1) * h <= dt) {
        double Dfi = Df, Dri = Dr;
        if (zones) surface_forces(zc, s, trk.TrackLength, Df, Dr, &Dfi, &Dri);
        sim_substep<false>(mass, lf, lr, Iz, Dfi, Cf, Bf, Dri, Cr, Br, delta, acc, sd, cd, h, trk, &okc, vx, vy, wz, epsi, s,
                           ey, psi, X, Y);
        ++i;
    }
    x[0] = vx; x[1] = vy; x[2] = wz; x[3] = epsi; x[4] = s; x[5] = ey;
    return okc != 0;
}

// Rows 3..5 of a stage's (A | B | C) (PM.py:66-135): the Jacobian of the curvilinear kinematics over one period dt at the point
// x, with the curvature cur at x's s.  vals gets the 17 distinct values K1_ABC_SRC indexes: 0, 1, dt, the entries a30 a31 a33 a35,
// a40 a41 a43 a45, a50 a51 a53 of A, and C's c3 c4 c5.
__device__ __forceinline__ void kinematic_rows(const double (&x)[6], double cur, double dt, double (&vals)[17]) {
    const double vx = x[0], vy = x[1], wz = x[2], epsi = x[3], sc = x[4], ey = x[5];
    const double den = 1.0 - cur * ey;
    const double rden = fast_rcp(den), rden2 = rden * rden;
    double se, ce;
    sincos(epsi, &se, &ce);
    const double vl = vx * ce - vy * se;          // longitudinal speed along the centre line
    const double vt = -vx * se - vy * ce;
    const double a30 = -dt * ce * rden * cur, a31 = dt * se * rden * cur, a33 = 1.0 - dt * vt * rden * cur;
    const double a35 = dt * vl * rden2 * cur * (-cur);
    const double a40 = dt * (ce * rden), a41 = -dt * (se * rden), a43 = dt * vt * rden, a45 = -dt * vl * rden2 * (-cur);
    const double a50 = dt * se, a51 = dt * ce, a53 = dt * vl;
    // C_r = f_r(x) - A_r x, products summed left to right like np.dot on 6 terms
    const double f3 = epsi + dt * (wz - vl * rden * cur);
    const double f4 = sc + dt * (vl * rden);
    const double f5 = ey + dt * (vx * se + vy * ce);
    const double c3 = f3 - (a30 * vx + a31 * vy + dt * wz + a33 * epsi + 0.0 * sc + a35 * ey);
    const double c4 = f4 - (a40 * vx + a41 * vy + 0.0 * wz + a43 * epsi + sc + a45 * ey);
    const double c5 = f5 - (a50 * vx + a51 * vy + 0.0 * wz + a53 * epsi + 0.0 * sc + ey);
    vals[0] = 0.0; vals[1] = 1.0; vals[2] = dt;
    vals[3] = a30; vals[4] = a31; vals[5] = a33; vals[6] = a35;
    vals[7] = a40; vals[8] = a41; vals[9] = a43; vals[10] = a45;
    vals[11] = a50; vals[12] = a51; vals[13] = a53;
    vals[14] = c3; vals[15] = c4; vals[16] = c5;
}

}  // namespace lmpc
