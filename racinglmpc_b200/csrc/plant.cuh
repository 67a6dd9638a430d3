// racinglmpc_b200/csrc/plant.cuh — the device-resident closed loop after the QP: the plant and what is measured of it.
//
//   sim_step_kernel       Simulator.dynModel (SysModel.py:56-147): the car of car.cuh, noise and the closed-loop record
//   pid_input_kernel      PID.solve (Utilities.py:42-68)
//   measure_kernel        measurement noise on the state every controller sees
//   ridge_sysid_kernel    Regression (Utilities.py:5-28)
//   seed_from_record_kernel  the seeding of main.py:99-110 from the PID lap
#pragma once
#include <curand_kernel.h>
#include "safeset.cuh"
#include "lap_schedule.cuh"
#include "car.cuh"

namespace lmpc {

// ------------------------------------------------------------------------------------------------
// Simulator.dynModel (src/fnc/simulator/SysModel.py:56-147): 100 explicit-Euler sub-steps (1 ms) of the dynamic
// bicycle model with Pacejka tyres in the curvilinear and the global frame, then clipped Gaussian noise on
// (vx, vy, wz).  One thread per instance.  `z` = three standard-normal draws per instance (the reference consumes
// np.random.randn() in this order: vx, vy, wz); when z == nullptr they come from Philox4x32-10 keyed by
// (seed, stream, step), stream = streams[b] or b when streams is null — statistical, not bit-wise, parity with the reference's
// unseeded global RNG.
// Also appends (x, u) to the closed-loop buffer -- the measured state in place of x when rec_x is set -- and flags lap
// completion (SysModel.py:45-47).
// The ten vehicle constants (SysModel.py:61-70) are read from the instance's row of the vehicle table (a handle without vehicle
// sets holds a one-row table with the reference vehicle).  The arithmetic is the same with the constants in memory as with them
// folded in at compile time (DESIGN.md, "Per-controller vehicles").  The noise constants (SysModel.py:139-145) come the same way
// from the noise table (DESIGN.md, "Per-controller noise and common random numbers").
struct SimArgs {
    int batch;
    const double* x;      // [B][6] curvilinear state
    const double* xg;      // [B][6] global state (psi, X, Y at 3..5)
    const double* u;       // [B][2]  or uPred [B][N][2] with u_stride = N*2
    long long u_stride;
    const double* z;       // [B][3] or nullptr
    unsigned long long seed, step;
    double* xn;            // [B][6]
    double* xgn;           // [B][6]
    double* cl_x;          // [B][Tcl][6] closed-loop record (may be nullptr)
    const double* rec_x;   // [B][6] the state rows the record takes: the measured state (measure_kernel), or nullptr: x
    double* cl_u;          // [B][Tcl][2]
    int* cl_len;           // [B]
    int Tcl;
    int* done;             // [B] 1 when s_next > TrackLength
    const int* flags;     // [B] step flags (K1/K2/addPoint) and QP status of the step that produced u, or nullptr;
    const int* status;     //     accumulated into health[b] (OR of flags) and health[B + b] (steps with status != 1)
    int* health;           //     the simulator's own bits (SIM_LOOKUP_FAILED, SIM_RECORD_FULL) go to health[b] too
    Table<lmpc_vehicle_params> veh;   // vehicle of every instance (lmpc_rollout_set_vehicles)
    Tracks trk;                       // curvature and finish line of every instance (lmpc_set_tracks)
    Table<lmpc_noise_params> noise;   // noise of every instance (lmpc_rollout_set_noise)
    const int* streams;               // [B] Philox stream of every instance (lmpc_rollout_set_noise_streams), or nullptr: b
    LapBudget retire;                 // a retired instance is not driven (the PID lap passes a null budget)
};
// Health bits of the simulator itself (the step flags use 1 .. 64 and 512):
//   SIM_LOOKUP_FAILED  a sub-step's curvature lookup failed (s < 0, s at the finish line after the wrap, s not finite or beyond
//                      64 laps): the reference raises there (Track.py:292-310); the step went on with curvature 0
//   SIM_RECORD_FULL    the closed-loop record already held Tcl rows, so this step's (x, u) was not recorded: the lap is longer
//                      than the record and a hand-over of it files a truncated lap
constexpr int SIM_LOOKUP_FAILED = 128;
constexpr int SIM_RECORD_FULL = 256;

// With reports (rep.rows) the step is also added to the controller's running report row (report_step) with its QP's status
// a.status and iterations rep_iters, both null for a PID step.  The vehicle and noise rows come from the lap schedules veh_s and
// noise_s (lap_schedule.cuh; a null schedule reads the table's own index).  SURF (a surface table is installed): each sub-step's
// peak tyre forces follow the controller's surface row of surf, through the lap schedule surf_s; without one surf is not read.
// Surfaces stay a template flag (period_substeps).
template <bool SURF>
__global__ void sim_step_kernel(const __grid_constant__ ModelConst m, const SimArgs a, const LapReports rep, const int* rep_iters,
                                const LapSchedule veh_s, const LapSchedule noise_s, const Table<lmpc_surface_params> surf,
                                const LapSchedule surf_s) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.batch) return;
    if (a.retire.retired(b)) {
        // no record row, no health count, no draw.  The state (x, xg) is a double buffer whose halves swap every step: carrying
        // the state over to the other half unchanged is what keeps it where the hand-over left it
        for (int j = 0; j < 6; ++j) { a.xn[(size_t)b * 6 + j] = a.x[(size_t)b * 6 + j]; a.xgn[(size_t)b * 6 + j] = a.xg[(size_t)b * 6 + j]; }
        return;
    }
    if (a.health) {
        if (a.flags && a.flags[b]) a.health[b] |= a.flags[b];
        if (a.status && a.status[b] != 1) a.health[a.batch + b] += 1;
    }
    // vehicle parameters, SysModel.py:61-70
    const lmpc_vehicle_params& v = veh_s.of(a.veh, b);
    const double mass = v.m, lf = v.lf, lr = v.lr, Iz = v.Iz;
    const double Df = v.Df, Cf = v.Cf, Bf = v.Bf;
    const double Dr = v.Dr, Cr = v.Cr, Br = v.Br;
    const TrackRec& trk = a.trk.of(b);
    const double* x = a.x + (size_t)b * 6;
    const double* g = a.xg + (size_t)b * 6;
    const double delta = a.u[(size_t)b * a.u_stride], acc = a.u[(size_t)b * a.u_stride + 1];
    double vx = x[0], vy = x[1], wz = x[2], epsi = x[3], s = x[4], ey = x[5];
    double psi = g[3], X = g[4], Y = g[5];
    int sim_bits = 0;
    if (a.cl_x) {
        const int T = a.cl_len[b];
        if (T < a.Tcl) {
            const double* r = a.rec_x ? a.rec_x + (size_t)b * 6 : x;
#pragma unroll
            for (int j = 0; j < 6; ++j) a.cl_x[((size_t)b * a.Tcl + T) * 6 + j] = r[j];
            a.cl_u[((size_t)b * a.Tcl + T) * 2] = delta;
            a.cl_u[((size_t)b * a.Tcl + T) * 2 + 1] = acc;
            a.cl_len[b] = T + 1;
        } else {
            sim_bits = SIM_RECORD_FULL;
        }
    }
    const double sd = sin(delta), cd = cos(delta);
    int okc = 1;
    period_substeps<SURF>(m.dt, Df, Dr, SURF ? &surf_s.of(surf, b) : nullptr, true, &trk, s, [&](double Dfi, double Dri) {
        sim_substep<true>(mass, lf, lr, Iz, Dfi, Cf, Bf, Dri, Cr, Br, delta, acc, sd, cd, CAR_H, trk, &okc, vx, vy, wz, epsi, s, ey,
                          psi, X, Y);
    });
    if (!okc) sim_bits |= SIM_LOOKUP_FAILED;
    if (a.health && sim_bits) a.health[b] |= sim_bits;
    if (rep.rows) report_step(rep, b, x, (a.flags ? a.flags[b] : 0) | sim_bits, a.status, rep_iters);
    double z0, z1, z2;
    if (a.z) {
        z0 = a.z[(size_t)b * 3]; z1 = a.z[(size_t)b * 3 + 1]; z2 = a.z[(size_t)b * 3 + 2];
    } else {
        curandStatePhilox4_32_10_t st;
        const int stream = a.streams ? a.streams[b] : b;
        curand_init(a.seed, (unsigned long long)stream, a.step * 8ull, &st);   // 8 raw 32-bit draws per step: disjoint blocks
        const double2 n01 = curand_normal2_double(&st);
        const double2 n23 = curand_normal2_double(&st);
        z0 = n01.x; z1 = n01.y; z2 = n23.x;
    }
    // noise parameters, SysModel.py:139-145
    const lmpc_noise_params& nz = noise_s.of(a.noise, b);
    const double n_vx = fmax(-nz.sim_clip[0], fmin(z0 * nz.sim_sigma[0], nz.sim_clip[0]));
    const double n_vy = fmax(-nz.sim_clip[1], fmin(z1 * nz.sim_sigma[1], nz.sim_clip[1]));
    const double n_wz = fmax(-nz.sim_clip[2], fmin(z2 * nz.sim_sigma[2], nz.sim_clip[2]));
    const double gain = nz.sim_gain;
    double* xn = a.xn + (size_t)b * 6;
    double* gn = a.xgn + (size_t)b * 6;
    // SysModel.py:143-147: the noise is added to the curvilinear copy only
    gn[0] = vx; gn[1] = vy; gn[2] = wz; gn[3] = psi; gn[4] = X; gn[5] = Y;
    xn[0] = vx + gain * n_vx; xn[1] = vy + gain * n_vy; xn[2] = wz + gain * n_wz;
    xn[3] = epsi; xn[4] = s; xn[5] = ey;
    if (a.done) a.done[b] = (s > trk.TrackLength) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------
// PID path-following controller, Utilities.py:42-68 (PID.solve): u = [-0.6 ey - 0.9 epsi + clip(0.25 z0, +-0.9),
// 1.5 (vt - vx) + clip(0.10 z1, +-0.2)], z ~ N(0,1) drawn in that order.  Writes uPred[b][0] so that sim_step_kernel
// consumes it like a controller's first predicted input.  The noise constants are the instance's row of the noise table, the
// Philox stream is streams[b] (b when streams is null), as in sim_step_kernel.
struct PidArgs {
    int batch;
    const double* x;       // [B][6]
    double vt;
    const double* z;       // [B][2] or nullptr (Philox)
    unsigned long long seed, step;
    double* u;             // [B][u_stride]
    long long u_stride;
    Table<lmpc_noise_params> noise;   // noise of every instance (lmpc_rollout_set_noise)
    const int* streams;               // [B] Philox stream of every instance, or nullptr: b
};
__global__ void pid_input_kernel(const PidArgs a) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.batch) return;
    double z0, z1;
    if (a.z) {
        z0 = a.z[(size_t)b * 2]; z1 = a.z[(size_t)b * 2 + 1];
    } else {
        curandStatePhilox4_32_10_t st;
        const int stream = a.streams ? a.streams[b] : b;
        curand_init(a.seed ^ 0x9E3779B97F4A7C15ull, (unsigned long long)stream, a.step * 8ull, &st);
        const double2 n01 = curand_normal2_double(&st);
        z0 = n01.x; z1 = n01.y;
    }
    const lmpc_noise_params& nz = a.noise.of(b);
    const double* x = a.x + (size_t)b * 6;
    // -0.6 ey - 0.9 epsi with the one contraction the device has always computed (ptxas fused it so when the noise constants were
    // immediates); written out because the compiler otherwise picks its contraction from the surrounding code
    a.u[(size_t)b * a.u_stride] = fma(-0.6, x[5], -(0.9 * x[3])) +
                                  fmax(-nz.pid_clip[0], fmin(z0 * nz.pid_sigma[0], nz.pid_clip[0]));
    a.u[(size_t)b * a.u_stride + 1] = 1.5 * (a.vt - x[0]) + fmax(-nz.pid_clip[1], fmin(z1 * nz.pid_sigma[1], nz.pid_clip[1]));
}

// ------------------------------------------------------------------------------------------------
// Measurement noise (DESIGN.md, "Per-controller measurement noise"): the state a controller sees, y = x + n on the six
// curvilinear channels, n_j = clip(z_j * sigma_j, +-clip_j) in the form of the process noise, z_j standard normal from Philox keyed
// by (seed ^ K_MEAS, stream, clock) -- three curand_normal2_double calls, 12 raw 32-bit draws, in blocks of 16 per step.  Where
// n_j == 0 the state is copied, so a zero set gives y == x bit for bit (-0.0 + 0.0 would be +0.0).  One thread per controller; a
// retired controller draws nothing and writes nothing.  The row comes from the lap schedule meas_s (lap_schedule.cuh; a null
// schedule reads the table's own index).
constexpr unsigned long long K_MEAS = 0xD1B54A32D192ED03ull;     // distinct from the PID's key constant
struct MeasArgs {
    int batch;
    const double* x;       // [B][6] plant state
    double* y;             // [B][6] measured state
    unsigned long long seed, step;
    Table<lmpc_measurement_params> meas;   // measurement noise of every instance (lmpc_rollout_set_measurement_noise)
    const int* streams;                    // [B] Philox stream of every instance, or nullptr: b
    LapBudget retire;
};
__global__ void measure_kernel(const MeasArgs a, const LapSchedule meas_s) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.batch || a.retire.retired(b)) return;
    curandStatePhilox4_32_10_t st;
    const int stream = a.streams ? a.streams[b] : b;
    curand_init(a.seed ^ K_MEAS, (unsigned long long)stream, a.step * 16ull, &st);
    const double2 n01 = curand_normal2_double(&st);
    const double2 n23 = curand_normal2_double(&st);
    const double2 n45 = curand_normal2_double(&st);
    const double z[6] = {n01.x, n01.y, n23.x, n23.y, n45.x, n45.y};
    const lmpc_measurement_params& m = meas_s.of(a.meas, b);
    const double* x = a.x + (size_t)b * 6;
    double* y = a.y + (size_t)b * 6;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        const double n = fmax(-m.clip[j], fmin(z[j] * m.sigma[j], m.clip[j]));
        y[j] = n == 0.0 ? x[j] : x[j] + n;
    }
}

// LTI system identification by ridge regression, Utilities.py:5-28 (Regression): rows t = 1 .. T-2 of the closed-loop
// record, z_t = [x_t u_t] (8), y_t = x_{t+1} (6); W = (Z'Z + lamb I)^-1 Z'Y; A = W'[:, 0:6], B = W'[:, 6:8].
// One warp per instance: lane e < 36 owns one entry of the upper triangle of Z'Z, lanes own the 48 entries of Z'Y in two
// rounds; the 8 x 8 system with 6 right-hand sides is solved by Gaussian elimination with partial pivoting in shared memory.
// Output abc[b][54] = A (36, row-major) | B (12) | C = 0 (6): the per-instance LTI model in the layout ftocp_kernel reads.
__global__ void __launch_bounds__(32) ridge_sysid_kernel(int batch, const double* cl_x, const double* cl_u, const int* cl_len, int Tcl,
                                                         double lamb, double* abc, int* status) {
    const int b = blockIdx.x;
    if (b >= batch) return;
    const int lane = threadIdx.x;
    __shared__ double S[8][14];      // [Z'Z + lamb I | Z'Y]
    const int T = cl_len[b];
    const double* X = cl_x + (size_t)b * Tcl * 6;
    const double* U = cl_u + (size_t)b * Tcl * 2;
    auto zval = [&](int t, int j) { return j < 6 ? X[(size_t)t * 6 + j] : U[(size_t)t * 2 + (j - 6)]; };
    for (int e = lane; e < 36 + 48; e += 32) {
        int r, c;
        if (e < 36) { r = 0; int k = e; while (k >= 8 - r) { k -= 8 - r; ++r; } c = k + r; }
        else { r = (e - 36) / 6; c = 8 + (e - 36) % 6; }
        double acc = 0.0;
        for (int t = 1; t <= T - 2; ++t) {
            const double zr = zval(t, r);
            const double other = (c < 8) ? zval(t, c) : X[(size_t)(t + 1) * 6 + (c - 8)];
            acc += zr * other;
        }
        if (c < 8) {
            if (r == c) acc += lamb;
            S[r][c] = acc; S[c][r] = acc;
        } else {
            S[r][c] = acc;
        }
    }
    __syncwarp();
    bool ok = T >= 12;
    for (int p = 0; p < 8; ++p) {
        int piv = p;
        double best = fabs(S[p][p]);
        for (int r = p + 1; r < 8; ++r) { const double v = fabs(S[r][p]); if (v > best) { best = v; piv = r; } }
        if (!(best > 0.0)) ok = false;
        __syncwarp();
        if (lane < 14 && piv != p) { const double t = S[p][lane]; S[p][lane] = S[piv][lane]; S[piv][lane] = t; }
        __syncwarp();
        const double inv = (S[p][p] != 0.0) ? 1.0 / S[p][p] : 0.0;
        double f[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) f[r] = S[r][p] * inv;
        const double prow = lane < 14 ? S[p][lane] : 0.0;
        __syncwarp();
        if (lane < 14 && lane > p) {
#pragma unroll
            for (int r = 0; r < 8; ++r) if (r != p) S[r][lane] -= f[r] * prow;     // Gauss-Jordan: eliminate above and below
        }
        __syncwarp();
    }
    // W[r][c] = S[r][8 + c] / S[r][r];  A = W'[:, 0:6] -> A[i][j] = W[j][i];  B[i][k] = W[6 + k][i]
    double* out = abc + (size_t)b * 54;
    for (int e = lane; e < 54; e += 32) {
        double v = 0.0;
        if (e < 36) { const int i = e / 6, j = e % 6; v = S[j][8 + i] / S[j][j]; }
        else if (e < 48) { const int i = (e - 36) / 2, k = (e - 36) % 2; v = S[6 + k][8 + i] / S[6 + k][6 + k]; }
        out[e] = v;
    }
    if (lane == 0 && !ok) atomicOr(&status[b], 1);
}

// Seed a controller from the closed-loop record the way main.py:99-110 does from the PID lap: the record is stored `copies`
// times in the safe set (slots ss_slot0 ..) and in the regression model (slots model_slot0 ..), cost-to-go by computeCost,
// the controller state from the record (seed_state_block), timeStep = 0, no previous prediction; the record restarts.  One CTA
// per instance.  With reports the report table starts afresh.
__global__ void __launch_bounds__(256) seed_from_record_kernel(int batch, LapPool ss, LapPool model, int copies, int ss_slot0, int model_slot0,
                                                              const double* cl_x, const double* cl_u, int* cl_len, int Tcl, int N,
                                                              double* xLin, double* uLin, double* zt, double* OldInput, int* timeStep,
                                                              int* hasPred, int* done, Tracks trk, Shapes shp, LapReports rep) {
    const int b = blockIdx.x;
    if (b >= batch) return;
    const int Trec = cl_len[b];
    const double TrackLength = trk.of(b).TrackLength;
    const double* cx = cl_x + (size_t)b * Tcl * 6;
    const double* cu = cl_u + (size_t)b * Tcl * 2;
    for (int c = 0; c < copies; ++c) {
        copy_ss_lap_block(ss, ss.lap_index(b, ss_slot0 + c), cx, cu, Trec, TrackLength);
        copy_lap_block(model, model.lap_index(b, model_slot0 + c), cx, cu, Trec);
    }
    seed_state_block(b, N, shp, cx, cu, xLin, uLin, zt, OldInput);
    if (threadIdx.x == 0) {
        timeStep[b] = 0; hasPred[b] = 0; cl_len[b] = 0; done[b] = 0;
        if (rep.rows) report_restart(rep, b);
    }
}

}  // namespace lmpc
