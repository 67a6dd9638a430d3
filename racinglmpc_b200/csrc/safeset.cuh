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

// The track of every controller (lmpc_set_tracks; default: the track of lmpc_store_create); the ABI record is the device record.
using TrackRec = lmpc_track_params;
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
    // rows 3..5: Jacobian of the curvilinear kinematics; every lane evaluates the few distinct values, lane 3 stages them and the
    // warp writes the record through an index table
    {
        const double vx = xl[0], vy = xl[1], wz = xl[2], epsi = xl[3], sc = xl[4], ey = xl[5];
        const double dt = m.dt;
        int okc = 1;
        const double cur = curvature_lookup(a.trk.of(b), sc, &okc);
        if (!okc) flags |= 2;
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
        double* vals = sys;
        if (lane == 3) {
            vals[0] = 0.0; vals[1] = 1.0; vals[2] = dt;
            vals[3] = a30; vals[4] = a31; vals[5] = a33; vals[6] = a35;
            vals[7] = a40; vals[8] = a41; vals[9] = a43; vals[10] = a45;
            vals[11] = a50; vals[12] = a51; vals[13] = a53;
            vals[14] = c3; vals[15] = c4; vals[16] = c5;
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

}  // namespace lmpc
#include <curand_kernel.h>
#include "lap_schedule.cuh"
namespace lmpc {

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

// One explicit-Euler sub-step of Simulator.dynModel (SysModel.py:94-137), with the reference's lf in alpha_r: the curvilinear
// state (vx, vy, wz, epsi, s, ey) and, GLOBAL, the global pose (psi, X, Y), all updated from the sub-step's starting state.  Dfi,
// Dri are the sub-step's peak tyre forces (surface_forces), sd, cd = sin, cos(delta).  A failed curvature lookup clears *okc.
// sim_step_kernel and the observer's model prior (sim_period) both take it, so the prior is the plant's arithmetic exactly.
template <bool GLOBAL>
__device__ __forceinline__ void sim_substep(double mass, double lf, double lr, double Iz, double Dfi, double Cf, double Bf,
                                            double Dri, double Cr, double Br, double delta, double acc, double sd, double cd,
                                            double h, const TrackRec& trk, int* okc, double& vx, double& vy, double& wz,
                                            double& epsi, double& s, double& ey, double& psi, double& X, double& Y) {
    const double af = delta - atan2(vy + lf * wz, vx);
    const double ar = -atan2(vy - lf * wz, vx);
    const double Fyf = Dfi * sin(Cf * atan(Bf * af));
    const double Fyr = Dri * sin(Cr * atan(Br * ar));
    const double nvx = vx + h * (acc - 1 / mass * Fyf * sd + wz * vy);
    const double nvy = vy + h * (1 / mass * (Fyf * cd + Fyr) - wz * vx);
    const double nwz = wz + h * (1 / Iz * (lf * Fyf * cd - lr * Fyr));
    if constexpr (GLOBAL) {
        const double npsi = psi + h * wz;
        const double nX = X + h * (vx * cos(psi) - vy * sin(psi));
        const double nY = Y + h * (vx * sin(psi) + vy * cos(psi));
        psi = npsi; X = nX; Y = nY;
    }
    const double cur = curvature_lookup(trk, s, okc);
    const double ce = cos(epsi), se = sin(epsi);
    const double nepsi = epsi + h * (wz - (vx * ce - vy * se) / (1 - cur * ey) * cur);
    const double ns = s + h * ((vx * ce - vy * se) / (1 - cur * ey));
    const double ney = ey + h * (vx * se + vy * ce);
    vx = nvx; vy = nvy; wz = nwz; epsi = nepsi; s = ns; ey = ney;
}

// With reports (rep.rows) the step is also added to the controller's running report row (report_step) with its QP's status
// a.status and iterations rep_iters, both null for a PID step.  The vehicle and noise rows come from the lap schedules veh_s and
// noise_s (lap_schedule.cuh; a null schedule reads the table's own index).  SURF (a surface table is installed): each sub-step's
// peak tyre forces follow the controller's surface row of surf, through the lap schedule surf_s; without one surf is not read.
// Surfaces stay a template flag: a run-time test in the sub-step loop cost the table-free step 1.5 % per launch on an H100
// (DESIGN.md, "Track surfaces").
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
    const double h = 0.001;
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
    int i = 0;
    int okc = 1;
    SurfaceCursor zc{SURF ? &surf_s.of(surf, b) : nullptr, 0};
    while ((i + 1) * h <= m.dt) {
        double Dfi = Df, Dri = Dr;
        if constexpr (SURF) surface_forces(zc, s, trk.TrackLength, Df, Dr, &Dfi, &Dri);
        sim_substep<true>(mass, lf, lr, Iz, Dfi, Cf, Bf, Dri, Cr, Br, delta, acc, sd, cd, h, trk, &okc, vx, vy, wz, epsi, s, ey,
                          psi, X, Y);
        ++i;
    }
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

// Phi_car: the simulator's noise-free control period on the curvilinear state x under the input (delta, acc) -- sim_step_kernel's
// sub-step loop with car v and, when zones is not null, its surface row, without the global frame.  false when a sub-step's
// curvature lookup failed.
__device__ __forceinline__ bool sim_period(const lmpc_vehicle_params& v, const TrackRec& trk, const lmpc_surface_params* zones,
                                           double dt, double delta, double acc, double (&x)[6]) {
    const double mass = v.m, lf = v.lf, lr = v.lr, Iz = v.Iz;
    const double Df = v.Df, Cf = v.Cf, Bf = v.Bf;
    const double Dr = v.Dr, Cr = v.Cr, Br = v.Br;
    const double h = 0.001;
    const double sd = sin(delta), cd = cos(delta);
    double vx = x[0], vy = x[1], wz = x[2], epsi = x[3], s = x[4], ey = x[5];
    double psi = 0.0, X = 0.0, Y = 0.0;
    int i = 0;
    int okc = 1;
    SurfaceCursor zc{zones, 0};
    while ((i + 1) * h <= dt) {
        double Dfi = Df, Dri = Dr;
        if (zones) surface_forces(zc, s, trk.TrackLength, Df, Dr, &Dfi, &Dri);
        sim_substep<false>(mass, lf, lr, Iz, Dfi, Cf, Bf, Dri, Cr, Br, delta, acc, sd, cd, h, trk, &okc, vx, vy, wz, epsi, s, ey,
                           psi, X, Y);
        ++i;
    }
    x[0] = vx; x[1] = vy; x[2] = wz; x[3] = epsi; x[4] = s; x[5] = ey;
    return okc != 0;
}

// The model prior of controller b (source 1: the row's car, no surface; source 2: the car and surface the plant drove the
// previous step with -- the lap before lap_n when a hand-over came in between, seen as x_hat_{k-1}.s - y.s > TrackLength / 2).
// false when an input is not finite or a curvature lookup failed.
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
// differentiated.  A separate function, so that sim_substep's code, and the simulator's, stay as they are.
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
    const double h = 0.001;
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
