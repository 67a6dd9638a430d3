// racinglmpc_b200/csrc/safeset.cuh — device-resident lap stores and the HBM-scan kernels of the LMPC step.
//
//   K1 knn_ltv_regress   PredictiveModel.regressionAndLinearization + computeIndices + compute_Q_M +
//                        compute_b + LMPC_LocLinReg (PredictiveModel.py:48-197), Map.curvature (Track.py:292-310)
//   K2 ss_select         LMPC.addTerminalComponents / selectPoints (PredictiveControllers.py:386-416,478-514)
//   K6 ss_add_point      LMPC.addPoint (PC.py:466-476);  rollout_cost = LMPC.computeCost (PC.py:447-464)
//   K5 shift_state       xLin/uLin/OldInput/timeStep update of MPC.solve (PC.py:129-137)
//
// Lap store layout (one pool for the safe set, one for the regression model), per instance b, slot j:
//   x  [b][j][Tmax][6]   row-major states      u [b][j][Tmax][2]      q [b][j][Tmax] (safe set only)
//   len[b][j]            valid rows
// Rows are contiguous, so a warp scanning a lap issues fully coalesced 48 B/row (x) + 16 B/row (u) loads.
#pragma once
#include <math.h>
#include <math_constants.h>
#include <stdint.h>
#include "lap_budget.cuh"
#include "ftocp_launch.cuh"
#include "car.cuh"

namespace lmpc {

// What stays per handle of the regression model: the store's trToUse (strides of the usedIt books, K1's scratch) and dt (the
// simulator's control period too).  The regression constants are per controller (Regressions below).
struct ModelConst {
    int trToUse;
    double dt;
};

// A per-controller table as the kernels read it (DESIGN.md, "Per-controller tables"): controller b reads row idx[b] of tab, or
// row 0 when idx is null (the one-row default table of a handle without sets).
template <typename T>
struct Table {
    const T* tab;
    const int* idx;
    __device__ __forceinline__ const T& of(int b) const { return tab[idx ? idx[b] : 0]; }
};

// The regression constants of every controller (lmpc_set_regression_sets; default: those of lmpc_store_create, |scaling|
// included)
using RegressionRec = lmpc_regression_params;
using Regressions = Table<RegressionRec>;

// The track of every controller (TrackRec, car.cuh)
using Tracks = Table<TrackRec>;

// The shape of every controller (lmpc_set_shapes): horizon N_b and safe-set size M_b, or no table (tab == null) for the handle's
// own (N, numSS_Points).  Buffers keep the handle's N and M as their per-controller strides; a controller uses the leading part.
using ShapeRec = lmpc_shape_params;
using Shapes = Table<ShapeRec>;
// K1, K2 and the state shift come in two instantiations, SHAPED = a table is installed: without one the kernels are the code they
// were before shapes existed (a branch on a null table cost the closed loop of configs[3] about 1 %)
__device__ __forceinline__ int horizon_of(const Shapes& s, int b, int N) { return s.tab ? s.of(b).N : N; }
__device__ __forceinline__ int ss_points_of(const Shapes& s, int b, int M) { return s.tab ? s.of(b).numSS_Points : M; }

// The safe-set lap count numSS_it_b of every controller (lmpc_set_ss_laps), or no table (tab == null) for the handle's numSS_it,
// which stays the stride of sel / is_prev / min_index and K2's block size.  K2 takes SHAPED when either table is installed; the
// lap-book kernels (lapbooks.cuh) read the table through ss_laps_of.
// The prediction model of every controller (lmpc_set_prediction_models), or no table (tab == null): the k-NN regression for all.
// K1 takes NOMINAL when a table is installed and then skips the controllers of a nominal mode (nominal_model.cuh).
using PredictionModelRec = lmpc_prediction_model_params;
using PredictionModels = Table<PredictionModelRec>;

using SsLapsRec = lmpc_ss_laps_params;
using SsLaps = Table<SsLapsRec>;
__device__ __forceinline__ int ss_laps_of(const SsLaps& l, int b, int nit) { return l.tab ? l.of(b).numSS_it : nit; }

// Per-lap reports (lmpc_rollout_enable_lap_reports, DESIGN.md "Per-lap reports"): rows[B][L] filed at the lap hand-overs, and the
// running row of the record under way with the count n of rows filed.  Without reports every pointer is null and the kernels
// that file reports test rows.
struct LapRun {
    lmpc_lap_report row;
    int n, pad[3];
};
static_assert(sizeof(lmpc_lap_report) == 32 && sizeof(LapRun) == 48, "report rows are 32 bytes, running rows 48");
struct LapReports {
    lmpc_lap_report* rows;       // [B][L]
    LapRun* run;                 // [B]
    int L;
    Table<FtocpConstRec> qp;     // the QP constants (Fx, bx) of every controller: its parameter-set row, else the handle's
};
__device__ __forceinline__ void report_reset(lmpc_lap_report& r) {
    r.steps = 0; r.flags = 0; r.unsolved = 0; r.viol_steps = 0; r.ipm_iters = 0; r.ipm_iters_max = 0;
    r.viol_max = -CUDART_INF;
}
// A hand-over: the running row becomes report n (stored while n < L), n counts on, the row restarts with the record.  One thread.
__device__ __forceinline__ void report_file(const LapReports& rep, int b) {
    LapRun& r = rep.run[b];
    const int n = r.n;
    if ((unsigned)n < (unsigned)rep.L) rep.rows[(size_t)b * rep.L + n] = r.row;
    r.n = n + 1;
    report_reset(r.row);
}
// The seeding: the PID record is consumed without a report and the table starts afresh.  One thread.
__device__ __forceinline__ void report_restart(const LapReports& rep, int b) {
    rep.run[b].n = 0;
    report_reset(rep.run[b].row);
}
// One closed-loop step of controller b driven from plant state x: flags = the step flags | the simulator's bits, status / iters of
// the step's QP (null for a PID step).  The lane rows are evaluated without contraction so that a host restatement gives the same
// bits (tests/support/lap_reports.py).
__device__ __forceinline__ void report_step(const LapReports& rep, int b, const double* x, int flags, const int* status,
                                            const int* iters) {
    const FtocpConst& c = rep.qp.of(b).c;
    lmpc_lap_report r = rep.run[b].row;
    bool finite = true, viol = false;
#pragma unroll
    for (int j = 0; j < 6; ++j) finite = finite && isfinite(x[j]);
    if (!finite) {
        viol = true;
        r.viol_max = CUDART_INF;
    } else {
#pragma unroll
        for (int i = 0; i < 2; ++i) {                            // ncx == 2 lane rows (lmpc_create)
            double s = __dmul_rn(c.Fx[i * 6], x[0]);
#pragma unroll
            for (int j = 1; j < 6; ++j) s = __dadd_rn(s, __dmul_rn(c.Fx[i * 6 + j], x[j]));
            const double d = __dsub_rn(s, c.bx[i]);
            viol = viol || d > 0.0;
            r.viol_max = fmax(r.viol_max, d);
        }
    }
    r.steps += 1;
    r.flags |= flags;
    r.viol_steps += viol ? 1 : 0;
    if (status) {
        r.unsolved += status[b] != 1 ? 1 : 0;
        const int it = iters[b];
        r.ipm_iters += it;
        r.ipm_iters_max = max(r.ipm_iters_max, it);
    }
    rep.run[b].row = r;
}

struct LapPool {
    double* x;      // [B][cap][Tmax][6]
    double* u;      // [B][cap][Tmax][2]
    double* q;      // [B][cap][Tmax]   (nullptr for the model pool)
    int* len;       // [B][cap]
    int cap, Tmax;
    __host__ __device__ size_t lap_index(int b, int slot) const { return (size_t)b * cap + slot; }
};

// (dist, idx) lexicographic "less": ties go to the lower row index
__device__ __forceinline__ bool cand_less(double d1, int i1, double d2, int i2) { return d1 < d2 || (d1 == d2 && i1 < i2); }

// Gaussian elimination with partial pivoting, n = 5, NR right-hand sides; lane-redundant.
template <int NR>
__device__ __forceinline__ bool solve5(double (&A)[5][5], double (&b)[NR][5]) {
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 5; ++c) {
        int piv = c;
        double best = fabs(A[c][c]);
#pragma unroll
        for (int r = c + 1; r < 5; ++r) {
            double v = fabs(A[r][c]);
            if (v > best) { best = v; piv = r; }
        }
        if (!(best > 0.0)) { ok = false; best = 1.0; }
#pragma unroll
        for (int r = c + 1; r < 5; ++r) {
            if (piv == r) {
#pragma unroll
                for (int j = 0; j < 5; ++j) { double t = A[c][j]; A[c][j] = A[r][j]; A[r][j] = t; }
#pragma unroll
                for (int k = 0; k < NR; ++k) { double t = b[k][c]; b[k][c] = b[k][r]; b[k][r] = t; }
            }
        }
        double inv = 1.0 / A[c][c];
#pragma unroll
        for (int r = c + 1; r < 5; ++r) {
            double f = A[r][c] * inv;
#pragma unroll
            for (int j = c + 1; j < 5; ++j) A[r][j] -= f * A[c][j];
#pragma unroll
            for (int k = 0; k < NR; ++k) b[k][r] -= f * b[k][c];
        }
    }
#pragma unroll
    for (int k = 0; k < NR; ++k) {
#pragma unroll
        for (int r = 4; r >= 0; --r) {
            double v = b[k][r];
#pragma unroll
            for (int j = r + 1; j < 5; ++j) v -= A[r][j] * b[k][j];
            b[k][r] = v / A[r][r];
        }
    }
    return ok;
}

constexpr int K1_MAXPTS = 7;     // MaxNumPoint supported by the register top-k
constexpr int K1_MAXLAPS = 8;    // trToUse supported
#ifndef LMPC_K1_TILE
#define LMPC_K1_TILE 512
#endif
constexpr int K1_TILE = LMPC_K1_TILE;     // lap rows staged in shared memory per pass (fp32 features)
constexpr int K1_LOCAL = 3;      // entries of the lane-local candidate list
constexpr int K1_CAND = 32;      // exact re-scoring buffer per warp
constexpr unsigned K1_JBITS = 7; // low mantissa bits of a scan key that hold the lane's row counter: laps of up to 32 * 128 rows
constexpr unsigned K1_JMASK = (1u << K1_JBITS) - 1u;
constexpr float K1_FAR = 1.0e18f; // feature value of the padding rows of a tile (farther than any stored row, no overflow)

struct K1Args {
    int batch, N, wpb, pts_stride;   // warps per block; doubles of per-warp scratch (see k1_pts_stride)
    // Always 0: every launch covers the whole batch.  Kept because with the instance index read as b0 + blockIdx.x ptxas
    // rematerialises it instead of holding it in a register; with b = blockIdx.x the kernel spills 16 B at its 56-register cap and
    // the closed loop of configs[3] ran about 1 % slower (H100 80GB HBM3, profiles/h100_one_step_sequence_ab.txt).
    int b0 = 0;
    const double* xLin;  // [B][N+1][6]
    const double* uLin;   // [B][N][2]
    LapPool pool;         // model pool
    const int* used;      // [B][trToUse] slot ids, in usedIt order (the store's trToUse; a controller reads its first reg.trToUse)
    Tracks trk;           // the curvature of the linearisation point
    Regressions reg;      // MaxNumPoint, h, lamb, scaling and laps used of every controller (lmpc_set_regression_sets)
    LapBudget retire;     // the CTAs of a retired controller identify nothing
    double* abc;          // [B][N][54]
    int* status;          // [B] : 0 ok, else bit flags (1 = singular regression, 2 = curvature lookup failed,
                          //        4 = a single neighbour in a lap — cases where the reference raises,
                          //        32 = more than K1_CAND rows within rounding distance of the k-th neighbour)
    Shapes shp;           // the horizon of every controller: stages i >= N_b are not identified
    PredictionModels pm;  // NOMINAL: the prediction model of every controller; a controller of mode 1 or 2 is not regressed
};
// per-warp scratch: selected points [7*trToUse][15] (x0 x1 x2 delta a 1 | y0 y1 y2 | K*(x0 x1 x2 delta a 1)) | normal
//                   equations 45 (+3 pad) | staging of the closed-form record entries (17, +3 pad)
//                   | re-scoring buffer: K1_CAND exact distances + K1_CAND row indices | the query point (5 doubles, +1 pad)
//                   | the controller's regression row (RegressionRec, 8 doubles)
constexpr int K1_PW = 15;        // doubles per selected point
constexpr int K1_REGW = 8;       // doubles of a regression row
static_assert(sizeof(RegressionRec) == K1_REGW * sizeof(double), "a regression row is staged as 8 doubles");
__host__ __device__ inline int k1_pts_stride(int trToUse) {
    return K1_MAXPTS * trToUse * K1_PW + 48 + 20 + K1_CAND + K1_CAND / 2 + 6 + K1_REGW;
}
constexpr int K1_MAXWPB = 12;    // warps per block (__launch_bounds__ below)
// dynamic shared memory of a launch: the fp32 tile + the per-warp scratch
inline size_t k1_smem_bytes(int trToUse, int wpb) {
    return sizeof(float) * 5 * K1_TILE + sizeof(double) * (size_t)k1_pts_stride(trToUse) * wpb;
}

// The reference's distance of one stored row to the query (PM.py:185-186): diff = (Data - x) * scaling, 1-norm summed left to
// right (numpy semantics for 5 columns), in IEEE fp64 with no contraction: the value np.argsort ranks.
__device__ __noinline__ double k1_exact_dist(const double* sc, const double* X, const double* U, int t, const double* q) {
    const double* xr = X + (size_t)t * 6;
    const double* ur = U + (size_t)t * 2;
    double d = fabs(__dmul_rn(__dsub_rn(xr[0], q[0]), sc[0]));
    d = __dadd_rn(d, fabs(__dmul_rn(__dsub_rn(xr[1], q[1]), sc[1])));
    d = __dadd_rn(d, fabs(__dmul_rn(__dsub_rn(xr[2], q[2]), sc[2])));
    d = __dadd_rn(d, fabs(__dmul_rn(__dsub_rn(ur[0], q[3]), sc[3])));
    d = __dadd_rn(d, fabs(__dmul_rn(__dsub_rn(ur[1], q[4]), sc[4])));
    return d;
}

// grid = (B, ceil(N / wpb)); one warp per horizon step (= query point).  Per stored lap:
//   1. the CTA stages the lap's five regression features as fp32 in shared memory (tiles of K1_TILE rows, padded to whole
//      batches of 32 with far-away rows) and every warp scans the tile for its own query with an fp32 distance -- ten full-rate
//      instructions per row instead of fourteen half-rate fp64 ones.  Each lane keeps its K1_LOCAL smallest rows as packed keys
//      (distance bits | row counter) maintained by five integer min / max: the loop has no branch;
//   2. G = the k-th smallest lane minimum bounds the k-th smallest distance from above; every listed row with a key within the
//      rounding margin of G is re-scored with the reference's exact fp64 distance (global memory, ~9 rows) and the exact k
//      nearest are selected on the key (distance, row) -- bit for bit the rows np.argsort picks (PM.py:189), ties to the lower
//      row; the bandwidth test (PM.py:187-191) is made on the exact distances of the candidates;
//   3. a lane list that may have dropped such a row (all its entries are within the margin) makes the warp re-collect from
//      global memory with the now known threshold (rare: K1_LOCAL + 1 of the ~9 nearest rows in one lane).
// HBM traffic is one pass over the used laps per CTA; the scan is instruction-issue bound (SURVEY §8d).
// record entry e of (A | B | C) -> staged value (see the kernel's last block); -1 = written by the regression lanes
__constant__ signed char K1_ABC_SRC[54] = {
    -1, -1, -1, 0, 0, 0,   -1, -1, -1, 0, 0, 0,   -1, -1, -1, 0, 0, 0,      // A rows 0..2
    3, 4, 2, 5, 0, 6,      7, 8, 0, 9, 1, 10,     11, 12, 0, 13, 0, 1,      // A rows 3..5
    0, -1,  -1, 0,  -1, 0,  0, 0,  0, 0,  0, 0,                             // B
    -1, -1, -1, 14, 15, 16};                                                // C
#ifndef LMPC_K1_MINBLOCKS
#define LMPC_K1_MINBLOCKS 3
#endif
template <bool SHAPED, bool NOMINAL>
__global__ void __launch_bounds__(32 * K1_MAXWPB, LMPC_K1_MINBLOCKS) knn_ltv_regress_kernel(const __grid_constant__ ModelConst m, const K1Args a) {
    extern __shared__ __align__(16) unsigned char k1_smem[];
    const int b = a.b0 + blockIdx.x;
    if (a.retire.retired(b)) return;          // uniform over the CTA: no barrier is skipped by part of it
    if (NOMINAL && a.pm.of(b).mode != 0) return;   // nominal_model_kernel identifies this controller (uniform over the CTA)
    // every stage of this CTA lies past the controller's horizon (uniform over the CTA).  The shape is read where it is tested, not
    // held as a horizon: as one int across the scan it cost K1 a 12-byte spill at its 56-register cap
    if (SHAPED && (int)blockIdx.y * a.wpb >= a.shp.of(b).N) return;
    const int wib = threadIdx.x >> 5;
    const int i = blockIdx.y * a.wpb + wib;   // horizon step
    const int lane = threadIdx.x & 31;
    const int nthr = blockDim.x;
    const bool active = SHAPED ? i < a.shp.of(b).N : i < a.N;             // all warps take part in the tile loads
    float4* tile4 = reinterpret_cast<float4*>(k1_smem);                // [K1_TILE] : (vx, vy, wz, delta) of a row, one 16-byte load
    float* tile1 = reinterpret_cast<float*>(k1_smem) + 4 * K1_TILE;    // [K1_TILE] : a
    double* wbase = reinterpret_cast<double*>(k1_smem + sizeof(float) * 5 * K1_TILE) + (size_t)wib * a.pts_stride;
    double* pts = wbase;                                               // this warp's scratch
    const int np_max = K1_MAXPTS * m.trToUse;
    double* ne = pts + (size_t)np_max * K1_PW;                         // 48
    double* sys = ne + 48;                                             // 17 (+3)
    double* cbd = sys + 20;                                            // exact distances of the re-scored rows [K1_CAND]
    int* cbi = reinterpret_cast<int*>(cbd + K1_CAND);                  // their row indices [K1_CAND]

    const int ii = active ? i : 0;
    const double* xl = a.xLin + ((size_t)b * (a.N + 1) + ii) * 6;
    const double* ul = a.uLin + ((size_t)b * a.N + ii) * 2;
    // the fp64 query lives in shared memory (read on the rare exact paths only); the scan keeps its fp32 copy in registers
    double* qv = reinterpret_cast<double*>(cbi + K1_CAND);
    if (lane < 5) qv[lane] = (lane < 3) ? xl[lane] : ul[lane - 3];
    // this controller's regression constants: one 64 B row per warp, staged next to the query (b is uniform per CTA).  Read from
    // shared memory where they are used, they hold no register across the scan (the row pointer and h would cost K1 a spill at
    // its 56-register cap: DESIGN.md, "Per-controller regression models")
    double* rw = qv + 6;
    if (lane < K1_REGW) rw[lane] = reinterpret_cast<const double*>(&a.reg.of(b))[lane];
    __syncwarp();
    const RegressionRec& rg = *reinterpret_cast<const RegressionRec*>(rw);
    const float f0 = (float)qv[0], f1 = (float)qv[1], f2 = (float)qv[2], f3 = (float)qv[3], f4 = (float)qv[4];
    const float s0 = (float)rg.scaling[0], s1 = (float)rg.scaling[1], s2 = (float)rg.scaling[2], s3 = (float)rg.scaling[3], s4 = (float)rg.scaling[4];
    const float qsum = s0 * fabsf(f0) + s1 * fabsf(f1) + s2 * fabsf(f2) + s3 * fabsf(f3) + s4 * fabsf(f4);
    const int kk = rg.MaxNumPoint;
    int flags = 0, npts = 0;

    for (int c = 0; c < rg.trToUse; ++c) {      // rg.trToUse <= m.trToUse, the stride of the usedIt books
        const int slot = a.used[(size_t)b * m.trToUse + c];
        const size_t lap = a.pool.lap_index(b, slot);
        const double* X = a.pool.x + lap * a.pool.Tmax * 6;
        const double* U = a.pool.u + lap * a.pool.Tmax * 2;
        const int T = a.pool.len[lap];
        // lane-local candidate lists: the K1_LOCAL smallest KEYS a lane has seen, ascending.  A key is the fp32 distance with its
        // low K1_JBITS mantissa bits replaced by the lane's row counter j (row t = 32 j + lane): non-negative floats order like
        // their bit patterns, so three unsigned min / two max per row keep the list sorted -- no branch, no index registers.
        unsigned k0 = 0xffffffffu, k1 = 0xffffffffu, k2 = 0xffffffffu;
        for (int t0 = 0; t0 < T - 1; t0 += K1_TILE) {
            const int rows = min(K1_TILE, T - 1 - t0);      // rows 0..T-2 are candidates (PM.py:183)
            const int rows32 = (rows + 31) & ~31;            // the last batch is padded with far-away rows: the scan has no bounds test
            __syncthreads();                                 // previous tile fully consumed
            for (int r = threadIdx.x; r < rows32; r += nthr) {          // one 48 B + one 16 B row per thread -> fp32
                if (r < rows) {
                    const double2 v01 = *reinterpret_cast<const double2*>(X + (size_t)(t0 + r) * 6);
                    const double v2 = X[(size_t)(t0 + r) * 6 + 2];
                    const double2 uu = *reinterpret_cast<const double2*>(U + (size_t)(t0 + r) * 2);
                    tile4[r] = make_float4((float)v01.x, (float)v01.y, (float)v2, (float)uu.x);
                    tile1[r] = (float)uu.y;
                } else {
                    tile4[r] = make_float4(K1_FAR, K1_FAR, K1_FAR, K1_FAR);
                    tile1[r] = K1_FAR;
                }
            }
            __syncthreads();
            if (active) {
                unsigned j = (unsigned)(t0 >> 5);
#pragma unroll 4
                for (int rb = 0; rb < rows32; rb += 32, ++j) {
                    const float4 xv = tile4[rb + lane];
                    const float x4 = tile1[rb + lane];
                    float d = s0 * fabsf(xv.x - f0);
                    d = fmaf(s1, fabsf(xv.y - f1), d);
                    d = fmaf(s2, fabsf(xv.z - f2), d);
                    d = fmaf(s3, fabsf(xv.w - f3), d);
                    d = fmaf(s4, fabsf(x4 - f4), d);
                    const unsigned key = (__float_as_uint(d) & ~K1_JMASK) | j;
                    const unsigned a1 = max(k0, key), a2 = max(k1, key);
                    k0 = min(k0, key);
                    k1 = min(k1, a1);
                    k2 = min(k2, a2);
                }
            }
        }
        if (!active) continue;
        // ---- G = an upper bound of the k-th smallest key: the k-th smallest of the 32 lane minima (k distinct rows are at or
        //      below it); one REDUX.MIN per round.  At least two rounds: the flag-4 count below needs every row inside h as a
        //      candidate whenever fewer than two are, also at MaxNumPoint = 1
        unsigned G = 0xffffffffu;
        {
            unsigned cur = k0;
            const int kg = kk > 2 ? kk : 2;
            for (int rnd = 0; rnd < kg; ++rnd) {
                G = __reduce_min_sync(0xffffffffu, cur);
                cur = (cur == G) ? 0xffffffffu : cur;
            }
        }
        // Threshold.  A key understates its fp32 distance by < 2^-(23-K1_JBITS) relative (1.53e-5); |d32 - d64| < (|row| + |query|)
        // 4.2e-7 in the scaled 1-norm (inputs rounded to fp32, five fused terms) and |row| <= d + |query|.  The k rows behind G have
        // d64 < G (1 + 1.53e-5) + (G + 2 qsum) 4.3e-7, so every row of the exact top-k -- and, when fewer than k rows lie inside the
        // bandwidth h, every row inside it (then G >= h - margin) -- has a key below
        //     thr = G (1 + 3.2e-5) + (G + 2 qsum) 1.3e-6.
        // Per-controller scaling and h (lmpc_set_regression_sets).  Every bound above is relative: the fp32 scaling is the fp64 one
        // rounded once (2^-24, like a feature), and scaling every s_j by one factor scales the exact distances, the fp32 partial
        // distances, G, qsum, thr and h by it too -- by a power of two exactly.  What is not relative is the fp32 range: (float)s
        // must be normal, the padding rows' distance (K1_FAR s, five terms) must be finite and farther than every stored row, and
        // the partial distances must stay normal and below K1_FAR 1e-3 (the `open` bound) for rows of physical size.  The sets
        // admit |s| == 0 or 2^-32 <= |s| <= 2^32: then (float)s is normal; K1_FAR s <= 1e18 2^32 (x5 = 2.1e28) is finite and
        // farther than any row with features below 1e17; a stored distance with features below 2^10 is at most 5 2^32 2^11 =
        // 4.4e13 < 1e15, so a real G is never taken for `open`; and a partial distance stays normal down to feature differences
        // of 2^-94.  (`open` only labels the padding: below that bound G of a lap shorter than k rows is a padding key, and thr
        // then admits every stored row as `open` does.)  h enters only through the exact fp64 test d < h.
        const float Gf = __uint_as_float(G & ~K1_JMASK);
        const bool open = !(Gf < K1_FAR * 1e-3f);                   // fewer than k lanes hold a row: everything stored is a candidate
        const float thrf = open ? 3.0e38f : fmaf(Gf, 3.2e-5f, Gf) + (Gf + 2.0f * qsum) * 1.3e-6f;
        const unsigned thrk = __float_as_uint(thrf) | K1_JMASK;
        const int nrow = T - 1;
        const bool in0 = k0 <= thrk && (int)(((k0 & K1_JMASK) << 5) + lane) < nrow && k0 != 0xffffffffu;
        const bool in1 = k1 <= thrk && (int)(((k1 & K1_JMASK) << 5) + lane) < nrow && k1 != 0xffffffffu;
        const bool in2 = k2 <= thrk && (int)(((k2 & K1_JMASK) << 5) + lane) < nrow && k2 != 0xffffffffu;
        const unsigned m0 = __ballot_sync(0xffffffffu, in0), m1 = __ballot_sync(0xffffffffu, in1), m2 = __ballot_sync(0xffffffffu, in2);
        int nc = 0;
        if (m2 == 0u) {                                    // no lane list is full of candidates: nothing was dropped
            const unsigned lt = (1u << lane) - 1u;
            const int c0 = __popc(m0), c1 = __popc(m1);
            if (in0) { const int pos = __popc(m0 & lt); cbi[pos] = (int)(((k0 & K1_JMASK) << 5) + lane); }
            if (in1) { const int pos = c0 + __popc(m1 & lt); if (pos < K1_CAND) cbi[pos] = (int)(((k1 & K1_JMASK) << 5) + lane); }
            nc = c0 + c1;
        } else {                                           // rare: re-collect from global memory with the known threshold
            for (int t0 = 0; t0 < T - 1; t0 += 32) {
                const int t = t0 + lane;
                bool in = false;
                if (t < T - 1) {
                    const double* xr = X + (size_t)t * 6;
                    const double* ur = U + (size_t)t * 2;
                    float d = s0 * fabsf((float)xr[0] - f0);
                    d = fmaf(s1, fabsf((float)xr[1] - f1), d);
                    d = fmaf(s2, fabsf((float)xr[2] - f2), d);
                    d = fmaf(s3, fabsf((float)ur[0] - f3), d);
                    d = fmaf(s4, fabsf((float)ur[1] - f4), d);
                    in = d <= thrf;
                }
                const unsigned mask = __ballot_sync(0xffffffffu, in);
                const int pos = nc + __popc(mask & ((1u << lane) - 1u));
                if (in && pos < K1_CAND) cbi[pos] = t;
                nc += __popc(mask);
            }
        }
        if (nc > K1_CAND) { flags |= 32; nc = K1_CAND; }
        __syncwarp();
        int ksel = 0;
        // ---- exact re-scoring and selection of the k nearest on the key (distance, row): every candidate lane counts the
        //      candidates that precede it (a handful of broadcast shared-memory reads) -- its rank in np.argsort's order.
        // The lane that holds a winning candidate writes that point itself: features, next-row targets and the kernel-weighted
        // features (PM.py:193) -- no second pass over the selected rows.
        {
            double cd = 1e300;
            int ci = 0x7fffffff;
            if (lane < nc) { ci = cbi[lane]; cd = k1_exact_dist(rg.scaling, X, U, ci, qv); cbd[lane] = cd; }
            // PM.py:187-191: >= MaxNumPoint neighbours inside the bandwidth -> the MaxNumPoint closest, else all inside.  Every row
            // inside the bandwidth is a candidate whenever fewer than k are (see the threshold), so counting candidates decides it.
            const int inside = __popc(__ballot_sync(0xffffffffu, cd < rg.h));
            ksel = inside >= kk ? kk : inside;
            if (inside == 1) flags |= 4;    // np.squeeze() makes this case raise in the reference
            __syncwarp();
            int rank = 0;
            for (int j = 0; j < nc; ++j) {
                const double dj = cbd[j];
                const int ij = cbi[j];
                rank += (dj < cd || (dj == cd && ij < ci)) ? 1 : 0;
            }
            if (lane < nc && rank < ksel) {
                double* P = pts + (size_t)(npts + rank) * K1_PW;
                const double* xr = X + (size_t)ci * 6;
                const double* ur = U + (size_t)ci * 2;
                const double rr = cd * fast_rcp(rg.h);
                const double Kw = (1.0 - rr * rr) * 3.0 / 4.0;
                const double z0 = xr[0], z1 = xr[1], z2 = xr[2], z3 = ur[0], z4 = ur[1];
                P[0] = z0; P[1] = z1; P[2] = z2; P[3] = z3; P[4] = z4; P[5] = 1.0;
                P[6] = xr[6]; P[7] = xr[7]; P[8] = xr[8];       // row + 1 (PM.py:163: y = xStored[it][index + 1, yIndex])
                P[9] = Kw * z0; P[10] = Kw * z1; P[11] = Kw * z2; P[12] = Kw * z3; P[13] = Kw * z4; P[14] = Kw;
            }
            __syncwarp();                                   // cbd / cbi are rewritten for the next lap
        }
        npts += ksel;
    }
    if (!active) return;
    __syncwarp();

    // ---- normal equations (PM.py:141-168).  entries: Qvx(15) Qlat(15) bvx(5) bvy(5) bwz(5) ----
    for (int e = lane; e < 45; e += 32) {
        // entry e = sum_p (K z)[ir] * P[ic]; columns of a point row: 0..2 state, 3 delta, 4 a, 5 the constant 1, 6..8 targets,
        // 9..14 the kernel-weighted features
        int ir, ic;
        bool diag = false;
        if (e < 30) {
            const int lat = e >= 15;
            const int idx = lat ? e - 15 : e;
            // (r, cc), r <= cc, of the idx-th entry of the upper triangle of a 5 x 5 matrix
            const int r = (idx >= 5) + (idx >= 9) + (idx >= 12) + (idx >= 14);
            const int cc = idx - (r * 5 - r * (r - 1) / 2) + r;
            ir = (r < 3) ? r : (r == 3 ? (lat ? 3 : 4) : 5);
            ic = (cc < 3) ? cc : (cc == 3 ? (lat ? 3 : 4) : 5);
            diag = (r == cc);
        } else {
            const int which = (e - 30) / 5, r = (e - 30) % 5;   // 0 vx, 1 vy, 2 wz
            const int lat = which > 0;
            ir = (r < 3) ? r : (r == 3 ? (lat ? 3 : 4) : 5);
            ic = 6 + which;
        }
        double acc = 0.0;
        const double* P = pts;
        for (int p = 0; p < npts; ++p, P += K1_PW) acc = fma(P[9 + ir], P[ic], acc);
        if (diag) acc += rg.lamb;
        ne[e] = acc;
    }
    __syncwarp();
    // ---- three 5 x 5 solves in registers, one per lane (0: vx, 1: vy, 2: wz): the matrices are Gram matrices, so symmetric
    //      elimination without pivoting is stable; only the upper triangle is kept
    double th[5];
    {
        const int sy = lane < 2 ? lane : 2;
        const double* qa = ne + (sy == 0 ? 0 : 15);
        const double* qr = ne + 30 + 5 * sy;
        double A5[5][5];                      // upper triangle; a pivot is replaced by its reciprocal once used
#pragma unroll
        for (int r = 0; r < 5; ++r) {
#pragma unroll
            for (int cc = r; cc < 5; ++cc) A5[r][cc] = qa[r * 5 - r * (r - 1) / 2 + (cc - r)];
            th[r] = qr[r];
        }
        bool ok = true;
#pragma unroll
        for (int c = 0; c < 5; ++c) {
            const double pv = A5[c][c];
            if (!(pv > 1e-280)) ok = false;
            const double inv = (pv > 1e-280) ? fast_rcp(pv) : 0.0;
            A5[c][c] = inv;
#pragma unroll
            for (int r = c + 1; r < 5; ++r) {
                const double f = A5[c][r] * inv;
#pragma unroll
                for (int j = r; j < 5; ++j) A5[r][j] = fma(-f, A5[c][j], A5[r][j]);
                th[r] = fma(-f, th[c], th[r]);
            }
        }
#pragma unroll
        for (int r = 4; r >= 0; --r) {
            double v = th[r];
#pragma unroll
            for (int j = r + 1; j < 5; ++j) v = fma(-A5[r][j], th[j], v);
            th[r] = v * A5[r][r];
        }
        if (__any_sync(0xffffffffu, !ok && lane < 3)) flags |= 1;
    }

    // ---- A, B, C (PM.py:66-135) ----
    double* out = a.abc + ((size_t)b * a.N + i) * 54;
    if (lane < 3) {                          // rows 0..2: regression coefficients on (vx, vy, wz), the input and the constant
        out[lane * 6 + 0] = th[0]; out[lane * 6 + 1] = th[1]; out[lane * 6 + 2] = th[2];
        out[36 + 2 * lane + (lane == 0 ? 1 : 0)] = th[3];   // vx uses the acceleration input, the lateral rows the steering (PM.py:29-30)
        out[48 + lane] = th[4];
    }
    // rows 3..5: Jacobian of the curvilinear kinematics (kinematic_rows); every lane evaluates the few distinct values, lane 3
    // stages them and the warp writes the record through an index table
    {
        const double x[6] = {xl[0], xl[1], xl[2], xl[3], xl[4], xl[5]};
        int okc = 1;
        const double cur = curvature_lookup(a.trk.of(b), x[4], &okc);
        if (!okc) flags |= 2;
        double kv[17];
        kinematic_rows(x, cur, m.dt, kv);
        double* vals = sys;
        if (lane == 3) {
            vals[0] = kv[0]; vals[1] = kv[1]; vals[2] = kv[2];
            vals[3] = kv[3]; vals[4] = kv[4]; vals[5] = kv[5]; vals[6] = kv[6];
            vals[7] = kv[7]; vals[8] = kv[8]; vals[9] = kv[9]; vals[10] = kv[10];
            vals[11] = kv[11]; vals[12] = kv[12]; vals[13] = kv[13];
            vals[14] = kv[14]; vals[15] = kv[15]; vals[16] = kv[16];
        }
        __syncwarp();
        for (int e = lane; e < 54; e += 32) {
            const int k = K1_ABC_SRC[e];
            if (k >= 0) out[e] = vals[k];
        }
    }
    if (lane == 0 && flags) atomicOr(&a.status[b], flags);
}

// ------------------------------------------------------------------------------------------------
struct K2Args {
    int batch, N, numSS_it, P;   // P = numSS_Points / numSS_it (the handle's; under SHAPED controller b has P_b = M_b / numSS_it_b)
    Tracks trk;
    const double* x0;        // [B][6]
    const double* zt;        // [B][6]
    LapPool pool;            // safe-set pool
    const int* sel;          // [B][numSS_it] slot ids in sortedLapTime order (PC.py:395,402)
    const int* is_prev;      // [B][numSS_it] 1 if that lap is iteration it-1 (PC.py:506-512)
    const int* timeStep;     // [B]
    const int* has_pred;     // [B]
    const double* xPred;     // [B][N+1][6] previous prediction
    double* SS_sel;          // [B][6][M]
    double* Qfun_sel;        // [B][M]
    double* Succ_SS;         // [B][6][M]
    double* Succ_uSS;        // [B][2][M]
    double* zt_fixed;        // [B][6] zt after the lap-wrap fix (PC.py:392-393)
    int* status;             // [B] bit 8 = selection window ran past the stored lap (reference: IndexError)
    int* min_index;          // [B][numSS_it] argmin row (for tests)
    LapBudget retire;        // the CTA of a retired controller selects nothing
    Shapes shp;              // N_b and M_b of every controller: the [6,M_b] block at the start of the controller's [6,M] region
    SsLaps laps;             // numSS_it_b of every controller: warps c >= numSS_it_b select nothing
};

// Lap-wrap fix of a guess of s made before the finish line (PC.py:392-393): after a hand-over the state's s has moved back by
// TrackLength and the guess has not.  K2's terminal guess and the state observer's prior (observe_kernel) both take it.
__device__ __forceinline__ void wrap_guess_s(double& guess_s, double x_s, double TrackLength) {
    if (guess_s - x_s > TrackLength / 2) guess_s = fmax(guess_s - TrackLength, 0.0);
}

// One CTA per instance, one warp per selected lap.  SHAPED: a shape table or a lap-count table (or both) is installed.
template <bool SHAPED>
__global__ void __launch_bounds__(32 * 8) ss_select_kernel(const K2Args a) {
    const int b = blockIdx.x;
    const int c = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (b >= a.batch || c >= a.numSS_it || a.retire.retired(b)) return;
    const int Mh = a.P * a.numSS_it;                         // the handle's M: the per-controller stride of the outputs
    const int nit = SHAPED ? ss_laps_of(a.laps, b, a.numSS_it) : a.numSS_it;
    if (SHAPED && c >= nit) return;                          // uniform over the warp; K2 has no block barrier
    const int M = SHAPED ? ss_points_of(a.shp, b, Mh) : Mh, P = SHAPED ? M / nit : a.P, Nb = SHAPED ? horizon_of(a.shp, b, a.N) : a.N;
    const double TrackLength = a.trk.of(b).TrackLength;
    // lap-wrap fix of the terminal guess (PC.py:392-393)
    double z[6];
#pragma unroll
    for (int j = 0; j < 6; ++j) z[j] = a.zt[(size_t)b * 6 + j];
    wrap_guess_s(z[4], a.x0[(size_t)b * 6 + 4], TrackLength);
    if (c == 0 && lane < 6) a.zt_fixed[(size_t)b * 6 + lane] = z[lane];

    const int slot = a.sel[(size_t)b * a.numSS_it + c];
    const size_t lap = a.pool.lap_index(b, slot);
    const double* X = a.pool.x + lap * a.pool.Tmax * 6;
    const double* U = a.pool.u + lap * a.pool.Tmax * 2;
    const double* Q = a.pool.q + lap * a.pool.Tmax;
    const int T = a.pool.len[lap];
    // 1-nearest neighbour in the 1-norm over all six states (PC.py:486-490) in np.argmin's order: the first NaN distance if there
    // is one (a NaN counts as -1, below every distance), else the first minimum.  A minimum of +inf is no candidate below: then
    // every distance is +inf, and np.argmin returns row 0
    double bd = CUDART_INF;
    int bi = 0x7fffffff;
    for (int t = lane; t < T; t += 32) {
        const double* xr = X + (size_t)t * 6;
        double d = fabs(__dsub_rn(xr[0], z[0]));
        d = __dadd_rn(d, fabs(__dsub_rn(xr[1], z[1])));
        d = __dadd_rn(d, fabs(__dsub_rn(xr[2], z[2])));
        d = __dadd_rn(d, fabs(__dsub_rn(xr[3], z[3])));
        d = __dadd_rn(d, fabs(__dsub_rn(xr[4], z[4])));
        d = __dadd_rn(d, fabs(__dsub_rn(xr[5], z[5])));
        if (isnan(d)) d = -1.0;
        if (d < bd) { bd = d; bi = t; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        double od = __shfl_xor_sync(0xffffffffu, bd, o);
        int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (cand_less(od, oi, bd, bi)) { bd = od; bi = oi; }
    }
    const int mn = bi == 0x7fffffff ? 0 : bi;
    if (mn >= T) {                                            // a lap without rows (np.argmin of an empty array raises)
        if (lane == 0) atomicOr(&a.status[b], 8);
        return;
    }
    // window (PC.py:492-495), numPoints = P + 1
    const int npt = P + 1;
    const int half = npt / 2;
    int start, count;
    if ((double)mn - (double)npt / 2.0 >= 0.0) { start = mn - half; count = 2 * half + 1; }
    else { start = mn; count = npt; }
    if (lane == 0) a.min_index[(size_t)b * a.numSS_it + c] = mn;
    if (start + count > T || count != npt) {
        if (lane == 0) atomicOr(&a.status[b], 8);
        return;
    }
    // Q-function shift when the prediction has crossed the finish line (PC.py:501-512)
    double adj = 0.0;
    if (a.has_pred[b]) {
        int over = 0;
        for (int k = 0; k <= Nb; ++k) over += (a.xPred[((size_t)b * (a.N + 1) + k) * 6 + 4] > TrackLength) ? 1 : 0;
        if (over > 0) {
            if (!a.is_prev[(size_t)b * a.numSS_it + c]) adj = Q[0];
            else adj = (double)a.timeStep[b] + (double)(Nb - over);
        }
    }
    for (int l = lane; l < count; l += 32) {
        const int row = start + l;
        const double* xr = X + (size_t)row * 6;
        if (l < P) {
            const int col = c * P + l;
#pragma unroll
            for (int j = 0; j < 6; ++j) a.SS_sel[SHAPED ? (size_t)b * 6 * Mh + j * M + col : ((size_t)b * 6 + j) * M + col] = xr[j];
            a.Qfun_sel[(size_t)b * (SHAPED ? Mh : M) + col] = Q[row] + adj;
        }
        if (l >= 1) {
            const int col = c * P + (l - 1);
#pragma unroll
            for (int j = 0; j < 6; ++j) a.Succ_SS[SHAPED ? (size_t)b * 6 * Mh + j * M + col : ((size_t)b * 6 + j) * M + col] = xr[j];
            a.Succ_uSS[SHAPED ? (size_t)b * 2 * Mh + 0 * M + col : ((size_t)b * 2 + 0) * M + col] = U[(size_t)row * 2];
            a.Succ_uSS[SHAPED ? (size_t)b * 2 * Mh + 1 * M + col : ((size_t)b * 2 + 1) * M + col] = U[(size_t)row * 2 + 1];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// LMPC.addPoint (PC.py:466-476): append x + [0,0,0,0,L,0], u to lap it-1; Qfun extends by last - 1.
// A point with a non-finite value is not appended (the reference would store it): flag 512.  Lap it-1 is the lap the pooled
// exchange exports, so a diverged controller would otherwise hand NaN rows to every importer of its group.
__global__ void ss_add_point_kernel(int batch, LapPool pool, const int* prev_slot, const double* x, const double* u,
                                    long long u_stride, Tracks trk, int* status, int* dropped, LapBudget retire) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch || retire.retired(b)) return;
    const int slot = prev_slot[b];
    if (slot < 0) return;
    bool finite = isfinite(u[(size_t)b * u_stride]) && isfinite(u[(size_t)b * u_stride + 1]);
#pragma unroll
    for (int j = 0; j < 6; ++j) finite = finite && isfinite(x[(size_t)b * 6 + j]);
    if (!finite) {
        atomicOr(&status[b], 512);
        return;
    }
    const size_t lap = pool.lap_index(b, slot);
    const int T = pool.len[lap];
    if (T >= pool.Tmax || T < 1) {       // the lap cannot grow (the reference would keep appending): flag it, count it
        atomicOr(&status[b], 16);
        if (dropped) atomicAdd(dropped, 1);
        return;
    }
    double* X = pool.x + (lap * pool.Tmax + T) * 6;
    double* U = pool.u + (lap * pool.Tmax + T) * 2;
    double* Q = pool.q + lap * pool.Tmax;
    const double TrackLength = trk.of(b).TrackLength;
#pragma unroll
    for (int j = 0; j < 6; ++j) X[j] = x[(size_t)b * 6 + j] + (j == 4 ? TrackLength : 0.0);
    U[0] = u[(size_t)b * u_stride];
    U[1] = u[(size_t)b * u_stride + 1];
    Q[T] = Q[T - 1] - 1.0;
    pool.len[lap] = T + 1;
}

// LMPC.computeCost (PC.py:447-464) for one stored lap, block-parallel: the reference counts backwards
//   Q[T-1] = 0;  Q[j] = Q[j+1] + 1 if s_j < TrackLength else 0
// i.e. Q[j] = (first row r >= j that is the last row or has s_r >= TrackLength) - j.  Chunks of blockDim rows are walked from
// the end; inside a chunk the nearest such row is a suffix-minimum (Hillis-Steele in shared memory).  blockDim.x == 256.
__device__ void lap_cost_block(const LapPool& pool, size_t lap, double TrackLength) {
    __shared__ int nxt[256];
    __shared__ int carry_s;
    const int T = pool.len[lap];
    const double* X = pool.x + lap * pool.Tmax * 6;
    double* Q = pool.q + lap * pool.Tmax;
    if (threadIdx.x == 0) carry_s = 0x7fffffff;
    __syncthreads();
    for (int hi = T; hi > 0; hi -= 256) {
        const int lo = max(hi - 256, 0);
        const int j = lo + threadIdx.x;
        int v = 0x7fffffff;
        if (j < hi && (j == T - 1 || !(X[(size_t)j * 6 + 4] < TrackLength))) v = j;
        nxt[threadIdx.x] = v;
        __syncthreads();
        for (int o = 1; o < 256; o <<= 1) {
            const int w = (threadIdx.x + o < 256) ? nxt[threadIdx.x + o] : 0x7fffffff;
            __syncthreads();
            if (w < nxt[threadIdx.x]) nxt[threadIdx.x] = w;
            __syncthreads();
        }
        const int carry = carry_s;
        const int r = min(nxt[threadIdx.x], carry);
        if (j < hi) Q[j] = (double)(r - j);
        __syncthreads();
        if (threadIdx.x == 0) carry_s = min(nxt[0], carry);
        __syncthreads();
    }
}

// ---- lap hand-over primitives ---------------------------------------------------------------------------------------------
// The host-slot kernels below (slots chosen by the Python lap books) and the device-book kernels of lapbooks.cuh (slots chosen
// on the device) copy laps only through these, so both keep stored laps bit-identical.  The *_block functions are called by
// every thread of the CTA; those with a barrier only from a path that is uniform across the CTA.

// Copy the first min(T, Tmax) rows of (x | u) of a closed-loop record into a pool slot.
__device__ inline void copy_lap_block(const LapPool& pool, size_t lap, const double* cx, const double* cu, int T) {
    T = min(T, pool.Tmax);
    for (int e = threadIdx.x; e < T * 6; e += blockDim.x) pool.x[lap * pool.Tmax * 6 + e] = cx[e];
    for (int e = threadIdx.x; e < T * 2; e += blockDim.x) pool.u[lap * pool.Tmax * 2 + e] = cu[e];
    if (threadIdx.x == 0) pool.len[lap] = T;
}

// The same into a safe-set slot, followed by the lap's cost-to-go (LMPC.computeCost).
__device__ inline void copy_ss_lap_block(const LapPool& ss, size_t lap, const double* cx, const double* cu, int T, double TrackLength) {
    copy_lap_block(ss, lap, cx, cu, T);
    __syncthreads();
    lap_cost_block(ss, lap, TrackLength);
}

// Exchange row: one lap as both lap exchanges ship it, [Tpad][XR_COLS] doubles, each lap row (x 6 | u 2 | Qfun 1), zero past
// the lap's length.  A model slot takes the first XR_Q columns.
constexpr int XR_U = 6;       // first column of u
constexpr int XR_Q = 8;       // column of Qfun
constexpr int XR_COLS = 9;

// Pack the first T rows of a stored safe-set lap into exchange row R.
__device__ inline void pack_lap_row_block(const LapPool& ss, size_t lap, int T, int Tpad, double* R) {
    const double* X = ss.x + lap * ss.Tmax * 6;
    const double* U = ss.u + lap * ss.Tmax * 2;
    const double* Q = ss.q + lap * ss.Tmax;
    for (int e = threadIdx.x; e < Tpad * XR_COLS; e += blockDim.x) {
        const int t = e / XR_COLS, j = e - t * XR_COLS;
        double v = 0.0;
        if (t < T) v = (j < XR_U) ? X[t * 6 + j] : (j < XR_Q ? U[t * 2 + (j - XR_U)] : Q[t]);
        R[e] = v;
    }
}

// File the first T rows of exchange row R into a safe-set slot, Qfun included, and count the lap in *filed when given (here,
// in thread 0's one block of writes: counted by the caller after the call, pool_import_kernel takes 40 registers instead of 32).
__device__ inline void file_ss_row_block(const LapPool& ss, size_t lap, const double* R, int T, int* filed = nullptr) {
    for (int e = threadIdx.x; e < T * XR_COLS; e += blockDim.x) {
        const int t = e / XR_COLS, j = e - t * XR_COLS;
        const double v = R[e];
        if (j < XR_U) ss.x[(lap * ss.Tmax + t) * 6 + j] = v;
        else if (j < XR_Q) ss.u[(lap * ss.Tmax + t) * 2 + (j - XR_U)] = v;
        else ss.q[lap * ss.Tmax + t] = v;
    }
    if (threadIdx.x == 0) { ss.len[lap] = T; if (filed) atomicAdd(filed, 1); }
}

// File the first Tm rows of exchange row R into a model slot.
__device__ inline void file_model_row_block(const LapPool& model, size_t lap, const double* R, int Tm) {
    for (int e = threadIdx.x; e < Tm * XR_Q; e += blockDim.x) {
        const int t = e / XR_Q, j = e - t * XR_Q;
        const double v = R[t * XR_COLS + j];
        if (j < XR_U) model.x[(lap * model.Tmax + t) * 6 + j] = v;
        else model.u[(lap * model.Tmax + t) * 2 + (j - XR_U)] = v;
    }
    if (threadIdx.x == 0) model.len[lap] = Tm;
}

// Restart the record of a finished lap (one thread): s -= TrackLength (SysModel.py:50), timeStep = 0 (PC.py:445), done = 0.
__device__ __forceinline__ void restart_record(int b, int* cl_len, double* x_cur, int* timeStep, int* done, double TrackLength) {
    cl_len[b] = 0;
    x_cur[(size_t)b * 6 + 4] -= TrackLength;
    timeStep[b] = 0;
    done[b] = 0;
}

// The controller state a seeded controller starts from: xLin / uLin = rows 1..N_b+1 / 1..N_b of its record cx / cu
// (PC.py:432-433) at the handle's stride N, zt = [0,0,0,0,10,0] (PC.py:330), OldInput = 0.
__device__ inline void seed_state_block(int b, int N, const Shapes& shp, const double* cx, const double* cu, double* xLin, double* uLin,
                                        double* zt, double* OldInput) {
    const int Nb = horizon_of(shp, b, N);
    for (int e = threadIdx.x; e < (Nb + 1) * 6; e += blockDim.x) xLin[(size_t)b * (N + 1) * 6 + e] = cx[6 + e];
    for (int e = threadIdx.x; e < Nb * 2; e += blockDim.x) uLin[(size_t)b * N * 2 + e] = cu[2 + e];
    __syncthreads();
    if (threadIdx.x < 6) zt[(size_t)b * 6 + threadIdx.x] = (threadIdx.x == 4) ? 10.0 : 0.0;
    if (threadIdx.x < 2) OldInput[(size_t)b * 2 + threadIdx.x] = 0.0;
}

__global__ void __launch_bounds__(256) rollout_cost_kernel(LapPool pool, int b, int slot, Tracks trk) {
    lap_cost_block(pool, pool.lap_index(b, slot), trk.of(b).TrackLength);
}

// Lap hand-over of every instance with fin[b] != 0, one CTA per instance (main.py:113-119 + SysModel.py:50 + PC.py:445):
// the closed-loop record goes to safe-set slot ss_slot[b] (>= 0) with its cost-to-go and to regression slot model_slot[b]
// (>= 0); then the record restarts (with reports, its running report row is filed first).
__global__ void __launch_bounds__(256) commit_laps_kernel(int batch, LapPool ss, LapPool model, const int* fin, const int* ss_slot,
                                                          const int* model_slot, const double* cl_x, const double* cl_u, int* cl_len,
                                                          int Tcl, double* x_cur, int* timeStep, int* done, Tracks trk, LapReports rep) {
    const int b = blockIdx.x;
    if (b >= batch || !fin[b]) return;
    const int Trec = cl_len[b];
    const double TrackLength = trk.of(b).TrackLength;
    const size_t rec = (size_t)b * Tcl;     // an offset, not two record pointers, lives across the safe-set store: 28 registers, not 31
    if (ss_slot[b] >= 0) copy_ss_lap_block(ss, ss.lap_index(b, ss_slot[b]), cl_x + rec * 6, cl_u + rec * 2, Trec, TrackLength);
    if (model_slot[b] >= 0) copy_lap_block(model, model.lap_index(b, model_slot[b]), cl_x + rec * 6, cl_u + rec * 2, Trec);
    __syncthreads();
    if (threadIdx.x == 0) {
        if (rep.rows) report_file(rep, b);
        restart_record(b, cl_len, x_cur, timeStep, done, TrackLength);
    }
}

// Pooled-safe-set exchange (SURVEY §8e): pack one stored lap per instance, slot[b] (< 0: none), into exchange rows
// rows[B][Tpad][XR_COLS] + lens[B] -- the send buffer of the once-per-lap all-gather ...
__global__ void ss_export_laps_kernel(int batch, LapPool pool, const int* slot, int Tpad, double* rows, int* lens) {
    const int b = blockIdx.x;
    if (b >= batch) return;
    const int sl = slot[b];
    const size_t lap = pool.lap_index(b, sl < 0 ? 0 : sl);
    const int T = sl < 0 ? 0 : min(pool.len[lap], Tpad);
    pack_lap_row_block(pool, lap, T, Tpad, rows + (size_t)b * Tpad * XR_COLS);
    if (threadIdx.x == 0) lens[b] = T;
}

// ... and its receive side: instance b stores gathered lap src[b] (index into rows[G][Tpad][XR_COLS], < 0: skip) in safe-set
// slot ss_slot[b] and, when model_slot[b] >= 0, in the regression-model pool too (main.py:117-119 adds a lap to both).
__global__ void ss_import_laps_kernel(int batch, LapPool ss, LapPool model, const int* ss_slot, const int* model_slot, const int* src,
                                      int Tpad, const double* rows, const int* lens) {
    const int b = blockIdx.x;
    if (b >= batch) return;
    const int g = src[b];
    if (g < 0) return;
    const double* R = rows + (size_t)g * Tpad * XR_COLS;
    const int T = min(lens[g], min(Tpad, ss.Tmax));
    if (ss_slot[b] >= 0) file_ss_row_block(ss, ss.lap_index(b, ss_slot[b]), R, T);
    if (model_slot && model_slot[b] >= 0) {
        // the model stores the lap as driven (rows up to the finish line, Qfun > 0 ... = 0), not the addPoint overrun
        int Tm = 0;
        for (int t = 0; t < T; ++t) { if (R[t * XR_COLS + XR_Q] >= 0.0) Tm = t + 1; }
        file_model_row_block(model, model.lap_index(b, model_slot[b]), R, min(Tm, model.Tmax));
    }
}

// MPC.solve tail (PC.py:129-137): xLin = [xPred[1:]; zt], uLin = [uPred[1:]; zt_u], OldInput = uPred[0], timeStep += 1
struct ShiftArgs {
    int batch, N, lmpc;
    const double* xPred;  // [B][N+1][6]
    const double* uPred;   // [B][N][2]
    const double* zt_in;   // [B][6]  (LMPC: Succ_SS lam; MPC: unused -> xPred[N])
    const double* ztu_in;  // [B][2]
    double* xLin;          // [B][N+1][6]
    double* uLin;          // [B][N][2]
    double* zt;            // [B][6]
    double* OldInput;      // [B][2]
    double* xPredPrev;     // [B][N+1][6]
    int* timeStep;
    int* has_pred;
    LapBudget retire;      // the state of a retired controller is not shifted
    Shapes shp;            // the horizon N_b of every controller (the blocks keep the handle's stride N)
};
template <bool SHAPED>
__global__ void shift_state_kernel(const ShiftArgs a) {
    const int b = blockIdx.x;
    if (b >= a.batch || a.retire.retired(b)) return;
    const int N = a.N, Nb = SHAPED ? a.shp.of(b).N : N;
    for (int e = threadIdx.x; e < (Nb + 1) * 6; e += blockDim.x) {
        const int k = e / 6, j = e % 6;
        double v;
        if (k < Nb) v = a.xPred[((size_t)b * (N + 1) + k + 1) * 6 + j];
        else v = a.lmpc ? a.zt_in[(size_t)b * 6 + j] : a.xPred[((size_t)b * (N + 1) + Nb) * 6 + j];
        a.xLin[(size_t)b * (N + 1) * 6 + e] = v;
        a.xPredPrev[(size_t)b * (N + 1) * 6 + e] = a.xPred[(size_t)b * (N + 1) * 6 + e];
        if (k == Nb) a.zt[(size_t)b * 6 + j] = v;
    }
    for (int e = threadIdx.x; e < Nb * 2; e += blockDim.x) {
        const int k = e / 2, j = e % 2;
        double v;
        if (k < Nb - 1) v = a.uPred[((size_t)b * N + k + 1) * 2 + j];
        else v = a.lmpc ? a.ztu_in[(size_t)b * 2 + j] : a.uPred[((size_t)b * N + Nb - 1) * 2 + j];
        a.uLin[(size_t)b * N * 2 + e] = v;
    }
    if (threadIdx.x < 2) a.OldInput[(size_t)b * 2 + threadIdx.x] = a.uPred[(size_t)b * N * 2 + threadIdx.x];
    if (threadIdx.x == 0) { a.timeStep[b] += 1; a.has_pred[b] = 1; }
}

}  // namespace lmpc
