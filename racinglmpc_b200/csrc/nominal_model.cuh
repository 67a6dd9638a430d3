// racinglmpc_b200/csrc/nominal_model.cuh — the nominal prediction model of lmpc_set_prediction_models (DESIGN.md,
// "Per-controller prediction models").
//
// A controller of mode 1 or 2 plans with the exact linearisation of a car instead of the k-NN regression of K1: rows 0..2 of
// its stage model are the derivatives of the simulator's own one-period map Phi of (vx, vy, wz) (SysModel.py:94-106,
// sim_step_kernel), rows 3..5 the closed-form kinematic rows K1 writes.  K1 skips such a controller (its NOMINAL instantiation),
// and nominal_model_kernel, launched after it, writes all 54 entries of the controller's stages.
#pragma once
#include "lap_schedule.cuh"
#include "car.cuh"

namespace lmpc {

struct NominalArgs {
    int batch, N;
    double dt;                        // the control period (ModelConst::dt): the sub-steps of period_substeps
    const double* xLin;               // [B][N+1][6]
    const double* uLin;               // [B][N][2]
    PredictionModels pm;              // the mode (and mode 1 vehicle) of every controller
    Table<lmpc_vehicle_params> veh;   // the simulator's vehicle table (mode 2)
    LapSchedule veh_s;                // its lap schedule in the closed loop, else rows == nullptr: the table's own index
    Tracks trk;                       // the curvature of the linearisation point (rows 3..5)
    LapBudget retire;                 // a retired controller identifies nothing
    Shapes shp;                       // stages i >= N_b are not identified
    double* abc;                      // [B][N][54]
    int* status;                      // [B] step flags: 2 (curvature lookup failed), LMPC_FLAG_NOMINAL_NONFINITE
    Table<lmpc_surface_params> surf;  // the simulator's surface table (mode 2; read by the SURF instantiation only)
    LapSchedule surf_s;               // its lap schedule in the closed loop, else rows == nullptr: the table's own index
};

// One thread per (controller, stage).  The state z = (vx, vy, wz) and its forward sensitivity S = dz/d(vx0, vy0, wz0, delta, a)
// (3 x 5) stay in registers through the sub-steps: z <- z + h f(z, u), S <- S + h (f_z S + f_u E), E = [0 | I2], f_z and f_u
// taken at the sub-step's starting state, which is the derivative of the explicit-Euler map itself.
// SURF (a surface table is installed): a mode 2 controller also carries (epsi, s, ey) through the sub-steps with the simulator's
// own curvature lookup, so that each sub-step's peak forces follow the zone the plant's s is in (sim_step_kernel).  The zone is
// piecewise constant in s, so it adds nothing to the derivatives: rows 0..2 of A keep columns 3..5 zero.
template <bool SURF>
__global__ void __launch_bounds__(128) nominal_model_kernel(const NominalArgs a) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = t / a.N, i = t - b * a.N;
    if (b >= a.batch || a.retire.retired(b)) return;
    const PredictionModelRec& row = a.pm.of(b);
    if (row.mode == 0) return;
    if (i >= (a.shp.tab ? a.shp.of(b).N : a.N)) return;
    const lmpc_vehicle_params& v = row.mode == 1 ? row.vehicle : a.veh_s.of(a.veh, b);
    const double mass = v.m, lf = v.lf, lr = v.lr, Iz = v.Iz;
    const double Df = v.Df, Cf = v.Cf, Bf = v.Bf;
    const double Dr = v.Dr, Cr = v.Cr, Br = v.Br;
    const double* xl = a.xLin + ((size_t)b * (a.N + 1) + i) * 6;
    const double* ul = a.uLin + ((size_t)b * a.N + i) * 2;
    const double delta = ul[0], acc = ul[1];
    const double h = CAR_H;
    double vx = xl[0], vy = xl[1], wz = xl[2];
    double S[3][5] = {{1, 0, 0, 0, 0}, {0, 1, 0, 0, 0}, {0, 0, 1, 0, 0}};
    const double sd = sin(delta), cd = cos(delta);
    // SURF: the kinematic states of the plant's sub-steps and the zone row (zoned: a mode 2 controller)
    const bool zoned = SURF && row.mode == 2;
    double epsi = xl[3], sk = xl[4], ey = xl[5];
    SurfaceCursor zc{zoned ? &a.surf_s.of(a.surf, b) : nullptr, 0};
    const TrackRec* trk = zoned ? &a.trk.of(b) : nullptr;
    // the loop of period_substeps<SURF> written out: through the helper, the abc of a mode 2 controller under a surface moved
    int k = 0;
    while ((k + 1) * h <= a.dt) {
        double Dfi = Df, Dri = Dr;
        if constexpr (SURF) {
            if (zoned) surface_forces(zc, sk, trk->TrackLength, Df, Dr, &Dfi, &Dri);
        }
        // the simulator's sub-step (sim_substep)
        const Tyres t = tyre_forces(lf, Dfi, Cf, Bf, Dri, Cr, Br, delta, vx, vy, wz);
        // dFy/dalpha and dalpha/d(vx, vy, wz); d alpha_f / d delta = 1
        const double gf = Dfi * cos(Cf * t.tf) * Cf * Bf / (1.0 + (Bf * t.af) * (Bf * t.af));
        const double gr = Dri * cos(Cr * t.tr) * Cr * Br / (1.0 + (Br * t.ar) * (Br * t.ar));
        const double rf = 1.0 / (vx * vx + t.yf * t.yf), rr = 1.0 / (vx * vx + t.yr * t.yr);
        const double daf[3] = {t.yf * rf, -vx * rf, -lf * vx * rf};
        const double dar[3] = {t.yr * rr, -vx * rr, lf * vx * rr};
        // f_z (3 x 3) and f_u (3 x 2)
        double Fz[3][3], Fu[3][2];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            Fz[0][j] = -sd / mass * gf * daf[j];
            Fz[1][j] = (cd * gf * daf[j] + gr * dar[j]) / mass;
            Fz[2][j] = (lf * cd * gf * daf[j] - lr * gr * dar[j]) / Iz;
        }
        Fz[0][1] += wz; Fz[0][2] += vy;
        Fz[1][0] -= wz; Fz[1][2] -= vx;
        Fu[0][0] = -(gf * sd + t.Fyf * cd) / mass; Fu[0][1] = 1.0;
        Fu[1][0] = (gf * cd - t.Fyf * sd) / mass; Fu[1][1] = 0.0;
        Fu[2][0] = lf * (gf * cd - t.Fyf * sd) / Iz; Fu[2][1] = 0.0;
        double Sn[3][5];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
#pragma unroll
            for (int c = 0; c < 5; ++c) {
                double d = Fz[r][0] * S[0][c] + Fz[r][1] * S[1][c] + Fz[r][2] * S[2][c];
                if (c >= 3) d += Fu[r][c - 3];
                Sn[r][c] = S[r][c] + h * d;
            }
        }
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 5; ++c) S[r][c] = Sn[r][c];
        if constexpr (SURF) {
            if (zoned) {      // the simulator's (epsi, s, ey) update, from the sub-step's starting state
                int okz = 1;
                const Kinematics q = kinematic_update(*trk, &okz, h, vx, vy, wz, epsi, sk, ey);
                epsi = q.epsi; sk = q.s; ey = q.ey;
            }
        }
        const Velocities n = velocity_update(mass, lf, lr, Iz, acc, sd, cd, h, t, vx, vy, wz);
        vx = n.vx; vy = n.vy; wz = n.wz;
        ++k;
    }
    double* out = a.abc + ((size_t)b * a.N + i) * 54;
    const double phi[3] = {vx, vy, wz};
    int flags = 0;
    bool finite = true;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        // C_r = Phi_r - (sum_j A_rj xbar_j + sum_k B_rk ubar_k), left to right, columns 3..5 of A included (they are 0)
        double s = __dmul_rn(S[r][0], xl[0]);
        s = __dadd_rn(s, __dmul_rn(S[r][1], xl[1]));
        s = __dadd_rn(s, __dmul_rn(S[r][2], xl[2]));
        s = __dadd_rn(s, __dmul_rn(0.0, xl[3]));
        s = __dadd_rn(s, __dmul_rn(0.0, xl[4]));
        s = __dadd_rn(s, __dmul_rn(0.0, xl[5]));
        s = __dadd_rn(s, __dmul_rn(S[r][3], delta));
        s = __dadd_rn(s, __dmul_rn(S[r][4], acc));
        const double c = __dsub_rn(phi[r], s);
        out[r * 6 + 0] = S[r][0]; out[r * 6 + 1] = S[r][1]; out[r * 6 + 2] = S[r][2];
        out[r * 6 + 3] = 0.0; out[r * 6 + 4] = 0.0; out[r * 6 + 5] = 0.0;
        out[36 + 2 * r] = S[r][3]; out[36 + 2 * r + 1] = S[r][4];
        out[48 + r] = c;
#pragma unroll
        for (int j = 0; j < 5; ++j) finite = finite && isfinite(S[r][j]);
        finite = finite && isfinite(c);
    }
    if (!finite) flags |= LMPC_FLAG_NOMINAL_NONFINITE;
    // rows 3..5: K1's closed-form block (kinematic_rows), at the entries K1_ABC_SRC gives them
    {
        const double x[6] = {xl[0], xl[1], xl[2], xl[3], xl[4], xl[5]};
        int okc = 1;
        const double cur = curvature_lookup(a.trk.of(b), x[4], &okc);
        if (!okc) flags |= 2;
        double kv[17];
        kinematic_rows(x, cur, a.dt, kv);
        const double row3[6] = {kv[3], kv[4], kv[2], kv[5], kv[0], kv[6]}, row4[6] = {kv[7], kv[8], kv[0], kv[9], kv[1], kv[10]};
        const double row5[6] = {kv[11], kv[12], kv[0], kv[13], kv[0], kv[1]};
#pragma unroll
        for (int j = 0; j < 6; ++j) { out[18 + j] = row3[j]; out[24 + j] = row4[j]; out[30 + j] = row5[j]; out[42 + j] = kv[0]; }
        out[51] = kv[14]; out[52] = kv[15]; out[53] = kv[16];
    }
    if (flags) atomicOr(&a.status[b], flags);
}

}  // namespace lmpc
