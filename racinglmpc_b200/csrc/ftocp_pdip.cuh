// racinglmpc_b200/csrc/ftocp_pdip.cuh
//
// One warp = one finite-time optimal control QP (the FTOCP that the reference assembles in
// src/fnc/controller/PredictiveControllers.py:166-257 (MPC) and :340-362 (LMPC terminal set)
// and hands to OSQP at :259-283).  Nothing is assembled: the solver works directly on the
// stage data (A_k,B_k,C_k, x(t), u(t-1), SS_sel, Qfun_sel) and solves
//
//   min  sum_k (x_k-xRef)'Q(x_k-xRef) + (x_N-xRef)'Qf(x_N-xRef) + u_k'R u_k
//        + sum_k (u_k-u_{k-1})'dR(u_k-u_{k-1}) + qs_quad|s|^2 + qs_lin 1's + Qfun'lam + xi'Qts xi
//   s.t. x_{k+1} = A_k x_k + B_k u_k + C_k,  Fx x_k - s_k <= bx (k<N),  Fu u_k <= bu,
//        s >= 0,  lam >= 0,  x_N - SS lam + xi = 0,  1'lam = 1
//
// with a Mehrotra predictor-corrector primal-dual interior-point method.  The Newton system is
// solved by (i) analytic elimination of the lane slacks and bound multipliers, (ii) a 6x6
// covariance-form elimination of the simplex/terminal block (centred at the D^-1-weighted
// centroid so the simplex multiplier decouples), (iii) a Riccati recursion over the horizon
// with the input-rate coupling carried as a 2-dim augmented state.  All in IEEE fp64.
// Executable specification + derivation: oracle/pdip_model.py (NumPy, test-only).
//
// Execution model: every function below is called by all 32 lanes of a warp with identical
// arguments.  Three idioms only, so that the same source also compiles as a 1-lane host
// emulation (tests/host_core.cpp; never part of the product path):
//   FOR_LANES(e, n) {..}  +  wsync()     work items spread over lanes, shared-memory results
//   lane-redundant scalar code           every lane computes the same value (free under SIMT)
//   FOR_SLOTS(r,row,CNT) + wsum/wmin     per-constraint state held in registers, row = lane + 32 r
// A "phase" never reads shared memory that another lane writes in the same phase.
#pragma once
#include <math.h>
#include <type_traits>

#if defined(__CUDACC__)
#define LMPC_HD __host__ __device__ __forceinline__
#else
#define LMPC_HD inline
#endif

// Device formulation of the Riccati sweeps: fp64 tensor-core fragments (mma.sync.m8n8k4.f64, "DMMA") when compiled by nvcc,
// the scalar shared-memory formulation on the host (tests/support/host_core.cpp) or with -DLMPC_NO_MMA (A/B measurements).
// The choice changes the layout of Work<>, so it must not depend on __CUDA_ARCH__ (host and device passes of one TU agree).
#if defined(__CUDACC__) && !defined(LMPC_NO_MMA)
#define LMPC_MMA 1
#else
#define LMPC_MMA 0
#endif
// unroll factor of the stage loops of the sweeps (2 lets the compiler rename the one-stage-ahead operand registers instead
// of copying them; more only grows the code, which 16 resident warps at different places keep missing in the instruction cache)
#ifndef LMPC_SWEEP_UNROLL_N
#define LMPC_SWEEP_UNROLL_N 2
#endif
#define LMPC_PRAGMA_(x) _Pragma(#x)
#define LMPC_PRAGMA(x) LMPC_PRAGMA_(x)
#define LMPC_SWEEP_UNROLL LMPC_PRAGMA(unroll LMPC_SWEEP_UNROLL_N)

// Algorithmic constants of the interior-point method's starting point and step rule.  Macros so that the 1-lane host emulation
// (tests/support/host_core.cpp) can sweep them on the CPU; the expressions may use the horizon N and LMPC (= a safe set is present).
// The MPC-type defaults are the result of such a sweep over the BASELINE workloads (4096 LTV-MPC QPs at N = 6 / 12 / 24 / 48;
// DESIGN.md §2): mean iterations 7.84 / 8.60 / 8.96 / 10.96 with the round-1 constants (0.3, 1, 0.995, back-off 0.8) -> 6.11 / 6.99 /
// 7.64 / 9.17, confirmed on the device (DESIGN.md §4).  LMPC-type QPs keep the
// round-1 constants: on 953 closed-loop QPs the same change saves 2.6 % of the iterations, and on the device it made the kernel
// 2.5 % slower and the Monte-Carlo rollouts less robust (12 instead of 2 unsolved steps in 5 M).
//   LMPC_TUNE_S0        offset of the initial lane slacks above the violation: long roll-outs of the initial input guess start
//                       farther from the lanes and want more room (N = 48: 18.9 iterations with 0.02, 9.4 with 0.5), short ones
//                       converge faster from a tight start
//   LMPC_TUNE_MU0SCALE  initial complementarity of the input bounds and the simplex relative to the mean lane-row product
//   LMPC_TUNE_MUFLOOR   floor of those products
//   LMPC_TUNE_STEP      fraction of the step to the boundary
// An end-game rule was tried and dropped: once the affine step is almost full, step to within max(fraction, 1 - mu) of the boundary
// with no neighbourhood test; it saved 3-9 % of the iterations on the host emulation and made configs[1] and [2] 1-2 % faster, but
// the Monte-Carlo rollouts left 67 instead of 2 of 5 M closed-loop QPs unsolved (DESIGN.md section 8).
#ifndef LMPC_TUNE_S0
#define LMPC_TUNE_S0 (LMPC ? 0.3 : (N <= 16 ? 0.1 : (N <= 24 ? 0.2 : 0.5)))
#endif
#ifndef LMPC_TUNE_MUFLOOR
#define LMPC_TUNE_MUFLOOR 1e-3
#endif
#ifndef LMPC_TUNE_MU0SCALE
#define LMPC_TUNE_MU0SCALE (LMPC ? 1.0 : 0.05)
#endif
#ifndef LMPC_TUNE_STEP
#define LMPC_TUNE_STEP (LMPC ? 0.995 : 0.999)
#endif
#ifndef LMPC_TUNE_SIGMA
#define LMPC_TUNE_SIGMA(s) ((s) * (s) * (s))      // Mehrotra's centring parameter from the affine complementarity ratio
#endif
#ifndef LMPC_TUNE_BACKOFF
#define LMPC_TUNE_BACKOFF (LMPC ? 0.8 : 0.9)       // step reduction until the iterate is back inside the neighbourhood
#endif
namespace lmpc {

// ------------------------------------------------------------------------------------------
// lane abstraction
// ------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
#define LMPC_NLANE 32
#define LMPC_LANE ((int)(threadIdx.x & 31))
__device__ __forceinline__ void wsync() { __syncwarp(); }
#ifndef LMPC_RED_INLINE
#define LMPC_RED_INLINE 1
#endif
#if LMPC_RED_INLINE
#define LMPC_RED_ATTR __forceinline__
#else
#define LMPC_RED_ATTR __noinline__      // one copy of each butterfly: the kernels are instruction-cache bound (DESIGN.md §8)
#endif
__device__ LMPC_RED_ATTR double wsum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ LMPC_RED_ATTR double wmin(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ LMPC_RED_ATTR double wmax(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// max / min of NON-NEGATIVE values (|.|, step bounds): such doubles order like their bit patterns, so two 32-bit REDUX
// (high word, then the low words of the lanes that tie on it) replace five shuffle + NaN-aware fmax rounds (~50 instructions)
__device__ __forceinline__ double wmax_nn(double v) {
    const unsigned hi = (unsigned)__double2hiint(v);
    const unsigned mh = __reduce_max_sync(0xffffffffu, hi);
    const unsigned ml = __reduce_max_sync(0xffffffffu, hi == mh ? (unsigned)__double2loint(v) : 0u);
    return __hiloint2double((int)mh, (int)ml);
}
__device__ __forceinline__ double wmin_nn(double v) {
    const unsigned hi = (unsigned)__double2hiint(v);
    const unsigned mh = __reduce_min_sync(0xffffffffu, hi);
    const unsigned ml = __reduce_min_sync(0xffffffffu, hi == mh ? (unsigned)__double2loint(v) : 0xffffffffu);
    return __hiloint2double((int)mh, (int)ml);
}
#else
#define LMPC_NLANE 1
#define LMPC_LANE 0
inline double wmax_nn(double v) { return v; }
inline double wmin_nn(double v) { return v; }
inline void wsync() {}
inline double wsum(double v) { return v; }
inline double wmin(double v) { return v; }
inline double wmax(double v) { return v; }
#endif

#if defined(__CUDA_ARCH__)
#define FOR_LANES(e, n) _Pragma("unroll") for (int e = LMPC_LANE; e < (n); e += LMPC_NLANE)
#else
#define FOR_LANES(e, n) for (int e = LMPC_LANE; e < (n); e += LMPC_NLANE)
#endif
#define NSLOT(CNT) (((CNT) + LMPC_NLANE - 1) / LMPC_NLANE)
// Horizons from LMPC_STREAM_MIN_N on do not stage the stage model (A | B | C, 44 % of the per-stage footprint) in shared memory:
// the tensor-core sweeps read their fragments of it straight from global memory / L2, one stage ahead of their use, which
// doubles the warps an SM holds at N = 48 (DESIGN.md §8).  Tensor-core build only.
#ifndef LMPC_STREAM_MIN_N
#define LMPC_STREAM_MIN_N 32
#endif
constexpr bool stream_model(int N) { return LMPC_MMA && N >= LMPC_STREAM_MIN_N; }
// condensed Hessian weight of lane row (k, i) / input-bound row (k, j): per-stage 8-vector (tensor-core path) or flat arrays
#if LMPC_MMA
#define LMPC_WDT(w, k, i, row) (w).Wd[k][i]
#define LMPC_WD2(w, k, j, row) (w).Wd[k][NCX + (j)]
#else
#define LMPC_WDT(w, k, i, row) (w).Dt[row]
#define LMPC_WD2(w, k, j, row) (w).d2[row]
#endif
// row = lane + 32*r ; the body runs only for valid rows.  No warp collectives inside.
#define FOR_SLOTS(r, row, CNT) \
    _Pragma("unroll") for (int r = 0, row = LMPC_LANE; r < NSLOT(CNT); ++r, row += LMPC_NLANE) if (row < (CNT))

// ------------------------------------------------------------------------------------------
// problem constants (one copy per controller configuration; __constant__ on the device)
// ------------------------------------------------------------------------------------------
constexpr int NX = 6;       // state dimension  (reference: n = 6, main.py:44)
constexpr int NU = 2;       // input dimension  (reference: d = 2)
constexpr int MAX_NCX = 4;  // rows of Fx supported
constexpr int MAX_NCU = 8;  // rows of Fu supported

struct FtocpConst {
    double Q2[36], Qf2[36], R2[4];  // 2Q, 2Qf, 2R           (buildCost: H = 2*blkdiag, PC.py:257)
    double qx[6], qxN[6];           // -2 Q xRef, -2 Qf xRef  (PC.py:245)
    double dR2[2];                  // 2 dR                   (PC.py:233-242)
    double qs2, ql;                 // 2*Qslack[0], Qslack[1] (PC.py:249-250)
    double Fx[MAX_NCX * 6], bx[MAX_NCX], Fu[MAX_NCU * 2], bu[MAX_NCU];  // PC.py:166-198
    double T[36], Tinv[36];         // 2*QterminalSlack and its inverse (PC.py:361)
    double eps_res, eps_gap, d4_min;
    double eps_step;                // convergence also needs the last primal step |alpha (dx, du)|_inf <= eps_step
    int max_iter;
    int pad_;
};

enum Status : int {
    ST_SOLVED = 1,
    ST_MAX_ITER = 2,
    ST_NUMERICAL = 3,   // non-positive pivot / non-finite step
    ST_BAD_INPUT = 4
};

// ------------------------------------------------------------------------------------------
// per-instance workspace (shared memory on the device)
// ------------------------------------------------------------------------------------------
template <int N, int M, int NCX, int NCU>
struct Work {
    static constexpr int MM = (M > 0 ? M : 1);
    static constexpr int TM = (M > 0 ? 36 : 1);
    // --- model (filled by the loader; ABC via cp.async.bulk) ---
    // As loaded: per stage A (36, row major a*6+b) | B (12, a*2+q) | C (6).  prepare_model() transposes A and B in
    // place, after which ABC[k][j*6 + c] = [A_k B_k](c, j), j < 8: every dot product of the sweeps then runs over a
    // contiguous, 16 B-aligned 6-vector (LDS.128).
    static constexpr bool STREAM = stream_model(N);
    alignas(16) double ABC[STREAM ? 1 : N][54];
    const double* gabc;             // STREAM: this instance's stage model in global memory (stage k at gabc + k * gstage)
    int gstage;                     // STREAM: doubles between two stage records
    alignas(16) double SS[6 * MM];  // SS[a*M + l]      (PC.py:411 SS_PointSelectedTot, 6 x M)
    double Qfun[MM];                // Qfun_SelectedTot (PC.py:412)
    alignas(16) double uOld[2];     // OldInput         (PC.py:136,247)
    // --- iterate ---
    alignas(16) double x[(N + 1) * 6];
    alignas(16) double dx[(N + 1) * 6];
    alignas(16) double u[N * 2];
    alignas(16) double du[N * 2];
    // (dx also stages nu1 | nu2 for the stage-gradient pre-pass: it is dead between the update and the next forward sweep)
    static_assert(N * (NCX + NCU) <= (N + 1) * 6, "staging area too small");
    // --- per-row quantities shared between lanes ---
    double ex[N * NCX];               // right-hand sides of the condensed lane constraints
    double eu[N * NCU];               // right-hand sides of the input bounds
    double d4i[MM];                   // 1 / max(nu4/lam, d4_min)
    alignas(16) double ru[N][2];      // input-stationarity residual
#if LMPC_MMA
    // ---- tensor-core formulation of the sweeps: cost-to-go Hessian / gradient live in register fragments; per stage only the
    //      barrier weights, the stage gradients, the feedback gain (or the closed-loop rows built from it), the inverse input
    //      Hessian and the feed-forward term are kept
    static_assert(NCX + NCU <= 6, "barrier weights of one stage must fit six entries of one 8-vector");
    alignas(16) double Wd[N][8];    // (Dt[0..NCX) | d2[0..NCU) | 0.. | input-rate weights at 6,7): diagonal of the stage's Fa' W Fa term
    alignas(16) double gv[N][16];   // row 0: stage gradient incl. the eliminated rows' right-hand side; row 1: -(stage gradient)
    // K = -Suu^-1 [Sux | -diag(dR2)]  (2 x 8, row major): u_k = K (x_k, u_{k-1}) + f.  Closed-loop sweeps (M == 0): K_k A~_{k-1}
    // instead, rows 6,7 of Phi_k = [A_{k-1} B_{k-1}; K_k A~_{k-1}], which maps (x, u)_{k-1} to (x, u)_k - (0, f_k); Kst[0] unused
    alignas(16) double Kst[N][16];
    alignas(16) double Sinv[N][4];  // Suu^-1 = (s00, s01, s11, -)
    alignas(16) double fst[N][2];   // f = -Suu^-1 g0 for the current right-hand side
    alignas(16) double tN[8];       // Qf2 x_N + qxN + yT  (= -costate at the end of the horizon)
    alignas(16) double cst[6];      // (1,0 | 0,1 | 0,0): identity / zero fragments read like stage data
#else
    double Dt[N * NCX];               // condensed lane-constraint Hessian weights
    double d2[N * NCU];               // input-bound Hessian weights
    alignas(16) double gst[N][8];   // stage gradient: (2Q x + qx + Fx'nu1 | 2R u + rate + Fu'nu2)
    alignas(16) double Zt[N][16];   // Z~ = L^-1 [ (B'Pxx+Pxv')A | -diag(dR2) ]  (2 x 8, row major)
    double Li[N][3];                // 1/L00, L10, 1/L11   (L = chol of the 2x2 input Hessian)
    double z0[N][2];                // L^-1 g0 for the current right-hand side
    // --- sweep scratch (augmented state (x, v = previous input), 8 x 8) ---
    static constexpr int PS = 10;   // padded row stride of Paug / Gt (80 B: the 8 rows hit distinct 16 B bank groups)
    alignas(16) double Paug[8 * PS];  // cost-to-go Hessian of stage k+1
    alignas(16) double Gt[8 * PS];    // Gt[j][a] = (Paug A~)(a, j),  A~ = [A B; 0 I]
    alignas(16) double S[64];       // A~' Paug A~ + stage Hessian
    alignas(16) double pb[2][8];    // cost-to-go gradient (px | pv), double buffered
    alignas(16) double pi[2][8];    // costate (6 used), double buffered
    double hv[8];                   // h~ = r~ + A~' p
#endif
    // --- terminal block ---
    alignas(16) double Wm[TM], Wi[TM];
    double sbar[6], yT[6];
    alignas(16) double red[8];      // warp sums of up to eight values at once (wsumv)
    alignas(16) double tv[8];       // 6-vectors handed from the lanes that compute them to the whole warp
    int flag;
};

// per-lane register state -------------------------------------------------------------------
template <int N, int M, int NCX, int NCU>
struct Regs {
    static constexpr int R1 = N * NCX, R2 = N * NCU, R4 = (M > 0 ? M : 1);
    // lane-constraint pair (k,i):  Fx_i x_k - s <= bx_i  and  s >= 0
    double s[NSLOT(R1)], nu1[NSLOT(R1)], nu3[NSLOT(R1)];
    double w1[NSLOT(R1)], rs[NSLOT(R1)], d1[NSLOT(R1)], p1[NSLOT(R1)], p3[NSLOT(R1)];
    double iw1[NSLOT(R1)], is_[NSLOT(R1)], ihs[NSLOT(R1)];   // reciprocals of w1, s, hs = qs2 + nu1/w1 + nu3/s (one division each per iteration)
    // input bound (k,j):  Fu_j u_k <= bu_j
    double nu2[NSLOT(R2)], w2[NSLOT(R2)], iw2[NSLOT(R2)], p2[NSLOT(R2)];
    // simplex multiplier l:  lam_l >= 0
    double lam[NSLOT(R4)], ilam[NSLOT(R4)], nu4[NSLOT(R4)], rl[NSLOT(R4)], p4[NSLOT(R4)], rho[NSLOT(R4)], dlam[NSLOT(R4)];
    double y1;
};

#if defined(LMPC_HOST_COUNT) && !defined(__CUDA_ARCH__)
static long g_host_count[3];     // host emulation only (parameter sweeps): corrector passes, recentring passes, step reductions
#endif
#ifndef LMPC_TUNE_GAMMA
#define LMPC_TUNE_GAMMA (LMPC ? 0.01 : 0.003)   // width of the central-path neighbourhood: min_i w_i nu_i >= gamma * mean
#endif
constexpr int LATE_ACCEPT_IT = 20;
constexpr int RECENTRE_AFTER = 3;   // step reductions before the corrector is replaced by a centring step

struct SolveInfo {
    int status, iters;
    int late;            // 1 = reported solved by the late-acceptance safety net (1e-6 contract), not at eps_res / eps_gap
    double r_prim, r_dual, gap;
};

// ------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------
LMPC_HD double dot6(const double* a, const double* b) {
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3] + a[4] * b[4] + a[5] * b[5];
}
// dot product of two contiguous, 16 B-aligned 6-vectors in shared memory (three LDS.128 per operand)
LMPC_HD double dot6v(const double* a, const double* b) {
#if defined(__CUDA_ARCH__)
    const double2 a0 = *reinterpret_cast<const double2*>(a), a1 = *reinterpret_cast<const double2*>(a + 2),
                  a2 = *reinterpret_cast<const double2*>(a + 4);
    const double2 b0 = *reinterpret_cast<const double2*>(b), b1 = *reinterpret_cast<const double2*>(b + 2),
                  b2 = *reinterpret_cast<const double2*>(b + 4);
    return (a0.x * b0.x + a0.y * b0.y) + (a1.x * b1.x + a1.y * b1.y) + (a2.x * b2.x + a2.y * b2.y);
#else
    return (a[0] * b[0] + a[1] * b[1]) + (a[2] * b[2] + a[3] * b[3]) + (a[4] * b[4] + a[5] * b[5]);
#endif
}
// 1/sqrt(v) and 1/v for positive, normal v (every call site guards its argument).  Device: the hardware approximation
// (MUFU.RSQ64H / MUFU.RCP64H, about 2^-20) refined to full double accuracy -- one cubic step for rsqrt (error e^3), two Newton
// steps for the reciprocal (e^4) -- without the library's slow-path branches for subnormal / infinite arguments.
LMPC_HD double rsqrt_f64(double v) {
#if defined(__CUDA_ARCH__)
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(v));
    const double e = fma(-v, y * y, 1.0);
    return fma(fma(0.375, e, 0.5), y * e, y);
#else
    return 1.0 / sqrt(v);
#endif
}
LMPC_HD double recip(double v) {
#if defined(__CUDA_ARCH__)
    double y;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(v));
    y = fma(y, fma(-v, y, 1.0), y);
    return fma(y, fma(-v, y, 1.0), y);
#else
    return 1.0 / v;
#endif
}
// (i, j), i <= j, of the e-th entry of the upper triangle of an 8 x 8 matrix (row-wise)
LMPC_HD void tri8(int e, int& i, int& j) {
    i = 0;
    while (e >= 8 - i) { e -= 8 - i; ++i; }
    j = e + i;
}
// Ratio test without divisions: (rn, rd) is the largest -dv/v seen so far as a fraction (start 0/1; v, rd > 0).
// The step bound of the lane is rd/rn, one division per test instead of one per constraint.
LMPC_HD void ratio_update(double v, double dv, double& rn, double& rd) {
    const double nn = -dv;
    if (nn * rd > rn * v) { rn = nn; rd = v; }
}
LMPC_HD double ratio_bound(double rn, double rd, double a) { return (rn > 0.0) ? fmin(a, rd * recip(rn)) : a; }

template <int N, int M, int NCX, int NCU>
struct Pdip {
    using W = Work<N, M, NCX, NCU>;
    using RG = Regs<N, M, NCX, NCU>;
    static constexpr int R1 = N * NCX, R2 = N * NCU, R4 = (M > 0 ? M : 1);
    static constexpr bool LMPC = (M > 0);
    static constexpr int TMW = (M > 0 ? 36 : 1);
#if !LMPC_MMA
    static constexpr int PS = W::PS;
#endif

    // ---------------------------------------------------------------- warm-start record ---
    // Per-controller snapshot of an interior-point iterate, taken at the first iteration (>= 1) whose complementarity gap is
    // below WARM_SNAP_MU, for the NEXT solve of the same controller (SURVEY §8f rank 2; the reference always starts cold,
    // PC.py:124,276).  Starting the next QP from the converged solution does not help an interior-point method (it sits on the
    // boundary); an iterate from the middle of the central path, shifted by one stage, does (oracle/pdip_model.py `warm=`).
    // Layout (doubles): u [N*2] | s, w1, nu1, nu3 [R1 each] | nu2 [R2] | lam, nu4 [M each] | y1.
    static constexpr int WS_U = 0, WS_S = N * 2, WS_W1 = WS_S + R1, WS_N1 = WS_W1 + R1, WS_N3 = WS_N1 + R1, WS_N2 = WS_N3 + R1,
                         WS_LAM = WS_N2 + R2, WS_N4 = WS_LAM + (LMPC ? M : 0), WS_Y1 = WS_N4 + (LMPC ? M : 0), WS_SIZE = WS_Y1 + 2;
    // The snapshot is the first iterate (the starting point included) whose gap lies in [WARM_MIN_MU, WARM_SNAP_MU]: an iterate
    // closer to the boundary makes a poor start (measured: snapshots at mu <= 1e-2 cost iterations and can stall).  A record is
    // re-used for at most WARM_MAX_AGE consecutive solves before a cold start re-anchors it, and it is dropped whenever a solve
    // started from it does not finish cleanly within WARM_MAX_ITERS iterations (max_iter if that is smaller) -- the solve then
    // restarts cold inside the same call with the full max_iter budget, and the next solve of that controller is cold.
    static constexpr double WARM_SNAP_MU = 0.1, WARM_MIN_MU = 0.01, WARM_THETA = 0.25;
    static constexpr int WARM_MAX_AGE = 8, WARM_MAX_ITERS = 16;

    static LMPC_HD void warm_snapshot(const W& w, const RG& g, double* wb) {
        FOR_LANES(e, N * 2) wb[WS_U + e] = w.u[e];
        FOR_SLOTS(r, row, R1) { wb[WS_S + row] = g.s[r]; wb[WS_W1 + row] = g.w1[r]; wb[WS_N1 + row] = g.nu1[r]; wb[WS_N3 + row] = g.nu3[r]; }
        FOR_SLOTS(r, row, R2) { wb[WS_N2 + row] = g.nu2[r]; }
        if (LMPC) {
            FOR_SLOTS(r, row, R4) { wb[WS_LAM + row] = g.lam[r]; wb[WS_N4 + row] = g.nu4[r]; }
            if (LMPC_LANE == 0) wb[WS_Y1] = g.y1;
        }
    }

    // Start from the snapshot of the previous solve shifted by one stage (stage k takes stage k+1, the last stage repeats):
    // inputs, lane slacks and all multipliers are taken over, the states are rolled out from the new x0 with the new model, and a
    // derived slack that shrank below WARM_THETA of its old value is restored through its lane slack.
    static LMPC_HD void warm_point(W& w, RG& g, const FtocpConst& c, const double* x0, const double* wb) {
        FOR_LANES(e, N * 2) { const int k = e >> 1, ks = (k + 1 < N) ? k + 1 : N - 1; w.u[e] = wb[WS_U + ks * 2 + (e & 1)]; }
        FOR_LANES(e, 6) w.x[e] = x0[e];
        prepare_model(w, c);
        wsync();
        rollout(w, x0);
        FOR_SLOTS(r, row, R1) {
            const int k = row / NCX, i = row % NCX;
            const int rs = (k + 1 < N) ? row + NCX : row;
            const double fx = dot6(&c.Fx[i * 6], &w.x[k * 6]) - c.bx[i];
            double s = wb[WS_S + rs];
            const double floor1 = WARM_THETA * wb[WS_W1 + rs];
            if (s - fx < floor1) s = fx + floor1;
            g.s[r] = s;
            g.nu1[r] = wb[WS_N1 + rs];
            g.nu3[r] = wb[WS_N3 + rs];
        }
        FOR_SLOTS(r, row, R2) {
            const int k = row / NCU;
            g.nu2[r] = wb[WS_N2 + ((k + 1 < N) ? row + NCU : row)];
        }
        if (LMPC) {
            FOR_SLOTS(r, row, R4) { g.lam[r] = wb[WS_LAM + row]; g.nu4[r] = wb[WS_N4 + row]; }
            g.y1 = wb[WS_Y1];
        }
    }

    // one-time preparation of the stage data (constants of the tensor-core sweeps / in-place transposition for the scalar sweeps)
    static LMPC_HD void prepare_model(W& w, const FtocpConst& c) {
#if LMPC_MMA
        FOR_LANES(e, 6) w.cst[e] = (e == 0 || e == 3) ? 1.0 : 0.0;
        FOR_LANES(e, N * 8) {           // rows 6,7: weight of u_k^2 in the input-rate cost (PC.py:233-242), rest written every iteration
            const int k = e >> 3, j = e & 7;
            w.Wd[k][j] = (j >= 6) ? ((k < N - 1) ? 2.0 : 1.0) * c.dR2[j - 6] : 0.0;
        }
#else
        FOR_LANES(k, N) {               // transpose A and B in place: ABC[k][j*6+c] = [A B](c, j)
            double* A = &w.ABC[k][0];
#pragma unroll
            for (int a = 0; a < 6; ++a)
#pragma unroll
                for (int b = a + 1; b < 6; ++b) { double t = A[a * 6 + b]; A[a * 6 + b] = A[b * 6 + a]; A[b * 6 + a] = t; }
            double bt[12];
#pragma unroll
            for (int e = 0; e < 12; ++e) bt[e] = A[36 + e];
#pragma unroll
            for (int cc = 0; cc < 6; ++cc) { A[36 + cc] = bt[cc * 2]; A[42 + cc] = bt[cc * 2 + 1]; }
        }
#endif
    }

#if !LMPC_MMA
    // roll the model out with the inputs in w.u (dynamics hold from the start); scalar formulation, transposed stage records
    static LMPC_HD void rollout(W& w, const double* x0) {
        (void)x0;
        for (int k = 0; k < N; ++k) {
            FOR_LANES(a, 6) {
                const double* T = &w.ABC[k][0];
                double v = T[48 + a] + T[36 + a] * w.u[k * 2] + T[42 + a] * w.u[k * 2 + 1];
#pragma unroll
                for (int b = 0; b < 6; ++b) v += T[b * 6 + a] * w.x[k * 6 + b];
                w.x[(k + 1) * 6 + a] = v;
            }
            wsync();
        }
    }
#endif

    // ---------------------------------------------------------------- initial point ------
    static LMPC_HD void init_point(W& w, RG& g, const FtocpConst& c, const double* x0, bool prepare = true) {
        // inputs: a strictly feasible multiple of the previous input, held over the horizon
        double tau = 1.0;
#pragma unroll
        for (int j = 0; j < NCU; ++j) {
            double v = c.Fu[j * 2] * w.uOld[0] + c.Fu[j * 2 + 1] * w.uOld[1];
            if (v > 0.9 * c.bu[j]) tau = fmin(tau, 0.9 * c.bu[j] / v);
        }
        FOR_LANES(e, N * 2) w.u[e] = tau * w.uOld[e & 1];
        FOR_LANES(e, 6) w.x[e] = x0[e];
        if (prepare) prepare_model(w, c);   // (a restart inside a solve finds the stage data prepared already)
        wsync();
        rollout(w, x0);                 // dynamics hold from the start
        // Dual-feasible, centred start (oracle/pdip_model.py, mu0 = "auto"): the slack-stationarity row
        // nu1 + nu3 = 2 qs s + ql holds exactly with w1 nu1 = s nu3 = mu_row; every other constraint
        // family starts at the mean of those products.
        double mu_acc = 0.0;
        FOR_SLOTS(r, row, R1) {
            int k = row / NCX, i = row % NCX;
            double fx = dot6(&c.Fx[i * 6], &w.x[k * 6]) - c.bx[i];
            double s = fmax(fx, 0.0) + LMPC_TUNE_S0;
            double w1 = s - fx;
            double mur = fmax((c.qs2 * s + c.ql) * (w1 * s) / (w1 + s), LMPC_TUNE_MUFLOOR);
            g.s[r] = s;
            g.nu1[r] = mur / w1;
            g.nu3[r] = mur / s;
            mu_acc += mur;
        }
        const double mu0 = fmax(LMPC_TUNE_MU0SCALE * wsum(mu_acc) / (double)R1, LMPC_TUNE_MUFLOOR);
        FOR_SLOTS(r, row, R2) {
            int k = row / NCU, j = row % NCU;
            double w2 = c.bu[j] - (c.Fu[j * 2] * w.u[k * 2] + c.Fu[j * 2 + 1] * w.u[k * 2 + 1]);
            g.nu2[r] = mu0 / w2;
        }
        if (LMPC) {
            FOR_SLOTS(r, row, R4) { g.lam[r] = 1.0 / M; }
            terminal_state(w, g, c);           // xi, yT for lam = 1/M
            double red_min = 1e300;
            FOR_SLOTS(r, row, R4) {
                double red = w.Qfun[row];
#pragma unroll
                for (int a = 0; a < 6; ++a) red -= w.SS[a * M + row] * w.yT[a];
                g.nu4[r] = red;
                red_min = fmin(red_min, red);
            }
            red_min = wmin(red_min);
            g.y1 = -red_min + mu0 * (double)M;
            FOR_SLOTS(r, row, R4) { g.nu4[r] += g.y1; }
        }
    }

    // Warp sums of NV <= 8 per-lane values at once; every lane receives all of them (and w.red keeps a copy until the next
    // call).  Tensor-core form: A = e_i 1' selects row i, B carries value i of the 32 lanes, so D[i][n] collects the four-lane
    // partial sums of value i; a product with the all-ones matrix then adds the eight partial sums: NV + 2 MMAs instead of
    // 15 NV shuffle / add instructions.
    template <int NV>
    static LMPC_HD void wsumv(W& w, double (&v)[NV]) {
        static_assert(NV >= 1 && NV <= 8, "up to eight values");
        wsync();                                    // earlier readers of red are done
#if LMPC_MMA
        const int lane = LMPC_LANE;
        const int r = lane >> 2;
        Frag Da{0.0, 0.0}, Db{0.0, 0.0};
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const double sel = (r == i) ? 1.0 : 0.0;
            if (i & 1) dmma(Db.a, Db.b, sel, v[i], Db.a, Db.b);
            else dmma(Da.a, Da.b, sel, v[i], Da.a, Da.b);
        }
        const Frag T = prod(Frag{1.0, 1.0}, Frag{Da.a + Db.a, Da.b + Db.b});   // T[m][i] = sum_n D[i][n]
        if (lane < 4) st2(&w.red[2 * lane], T.a, T.b);
        wsync();
#pragma unroll
        for (int i = 0; i < NV; ++i) v[i] = w.red[i];
#else
#pragma unroll
        for (int i = 0; i < NV; ++i) w.red[i] = v[i];
#endif
    }

    // xi = SS lam - x_N, yT = -T xi (both derived every iteration: the terminal equality and the
    // xi-stationarity row then hold by construction).  Returns sum(lam) - 1.
    static LMPC_HD double terminal_state(W& w, RG& g, const FtocpConst& c) {
        double acc[6] = {0, 0, 0, 0, 0, 0}, sl = 0.0;
        FOR_SLOTS(r, row, R4) {
#pragma unroll
            for (int a = 0; a < 6; ++a) acc[a] += w.SS[a * M + row] * g.lam[r];
            sl += g.lam[r];
        }
        double xi[6];
        {
            double v[7] = {acc[0], acc[1], acc[2], acc[3], acc[4], acc[5], sl};
            wsumv<7>(w, v);
#pragma unroll
            for (int a = 0; a < 6; ++a) xi[a] = v[a] - w.x[N * 6 + a];
            sl = v[6];
        }
        wsync();   // previous readers of yT are done
        FOR_LANES(a, 6) {
            double y = 0.0;
#pragma unroll
            for (int b = 0; b < 6; ++b) y -= c.T[a * 6 + b] * xi[b];
            w.yT[a] = y;
        }
        wsync();
        return sl - 1.0;
    }

    // ---------------------------------------------------------------- terminal factor ----
    // d4i, centroid, W = sum d4i s~ s~' + Tinv, Wi = W^-1 via Cholesky (PSD by construction).
    static LMPC_HD double terminal_factor(W& w, RG& g, const FtocpConst& c, double d4_floor) {
        double acc[6] = {0, 0, 0, 0, 0, 0}, dl = 0.0;
        FOR_SLOTS(r, row, R4) {
            double d4 = fmax(g.nu4[r] * g.ilam[r], d4_floor);
            double di = recip(d4);
            w.d4i[row] = di;
            dl += di;
#pragma unroll
            for (int a = 0; a < 6; ++a) acc[a] += w.SS[a * M + row] * di;
        }
        double sums[7] = {acc[0], acc[1], acc[2], acc[3], acc[4], acc[5], dl};
        wsumv<7>(w, sums);
        const double delta = sums[6];
        const double idelta = recip(delta);
#pragma unroll
        for (int a = 0; a < 6; ++a)
            if (LMPC_LANE == (a % LMPC_NLANE)) w.sbar[a] = sums[a] * idelta;   // same value on every lane
        wsync();
#if LMPC_MMA
        // W = Tinv + S~ diag(d4i) S~' on the tensor cores: one m8n8k4 step per four safe-set points.  Lane (r, q) supplies
        // S~[r][4j+q] d4i[4j+q] as the A element and S~[r][4j+q] as the B element (rows 6, 7 are zero); two accumulators.
        {
            static_assert(M % 4 == 0 || M == 0, "safe-set size must be a multiple of four");
            const int lane = sweep_lane();
            const int r = lane >> 2, q = lane & 3;
            const double m6 = (r < 6) ? 1.0 : 0.0;
            const double sb_r = w.sbar[r < 6 ? r : 0];
            const double* Sr = &w.SS[(r < 6 ? r : 0) * M + q];
            const double* Dq = &w.d4i[q];
            Frag Wa{0.0, 0.0}, Wb{0.0, 0.0};
#pragma unroll 4
            for (int j = 0; j + 1 < M / 4; j += 2) {
                const double s0 = (Sr[4 * j] - sb_r) * m6, s1 = (Sr[4 * j + 4] - sb_r) * m6;
                dmma(Wa.a, Wa.b, s0 * Dq[4 * j], s0, Wa.a, Wa.b);
                dmma(Wb.a, Wb.b, s1 * Dq[4 * j + 4], s1, Wb.a, Wb.b);
            }
            if ((M / 4) & 1) {
                const int j = M / 4 - 1;
                const double s0 = (Sr[4 * j] - sb_r) * m6;
                dmma(Wa.a, Wa.b, s0 * Dq[4 * j], s0, Wa.a, Wa.b);
            }
            if (r < 6 && q < 3)
                st2(&w.Wm[r * 6 + 2 * q], Wa.a + Wb.a + c.Tinv[r * 6 + 2 * q], Wa.b + Wb.b + c.Tinv[r * 6 + 2 * q + 1]);
        }
#else
        // W (21 unique entries), four partial accumulators each
        FOR_LANES(e, 21) {
            int a = 0, b = e;
            while (b >= 6 - a) { b -= 6 - a; ++a; }
            b += a;   // (a,b), a <= b
            double sa = w.sbar[a], sbb = w.sbar[b];
            double t0 = 0, t1 = 0, t2 = 0, t3 = 0;
            const double* Sa = &w.SS[a * M];
            const double* Sb = &w.SS[b * M];
            int l = 0;
            for (; l + 3 < M; l += 4) {
                t0 += (Sa[l] - sa) * (Sb[l] - sbb) * w.d4i[l];
                t1 += (Sa[l + 1] - sa) * (Sb[l + 1] - sbb) * w.d4i[l + 1];
                t2 += (Sa[l + 2] - sa) * (Sb[l + 2] - sbb) * w.d4i[l + 2];
                t3 += (Sa[l + 3] - sa) * (Sb[l + 3] - sbb) * w.d4i[l + 3];
            }
            for (; l < M; ++l) t0 += (Sa[l] - sa) * (Sb[l] - sbb) * w.d4i[l];
            double v = (t0 + t1) + (t2 + t3) + c.Tinv[a * 6 + b];
            w.Wm[a * 6 + b] = v;
            w.Wm[b * 6 + a] = v;
        }
#endif
        wsync();
        // lane-redundant 6x6 Cholesky, triangular inverse and Wi = Linv' Linv
        double L[21];   // packed lower, row i: i(i+1)/2 + j
        bool ok = true;
#pragma unroll
        for (int i = 0; i < 6; ++i) {
#pragma unroll
            for (int j = 0; j <= i; ++j) {
                double v = w.Wm[i * 6 + j];
#pragma unroll
                for (int k = 0; k < j; ++k) v -= L[i * (i + 1) / 2 + k] * L[j * (j + 1) / 2 + k];
                if (i == j) {
                    if (!(v > 0.0)) { ok = false; v = 1.0; }
                    L[i * (i + 1) / 2 + i] = rsqrt_f64(v);           // store the reciprocal pivot
                } else {
                    L[i * (i + 1) / 2 + j] = v * L[j * (j + 1) / 2 + j];
                }
            }
        }
        double X[21];   // Linv, packed lower
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            X[j * (j + 1) / 2 + j] = L[j * (j + 1) / 2 + j];
#pragma unroll
            for (int i = j + 1; i < 6; ++i) {
                double v = 0.0;
#pragma unroll
                for (int k = j; k < i; ++k) v -= L[i * (i + 1) / 2 + k] * X[k * (k + 1) / 2 + j];
                X[i * (i + 1) / 2 + j] = v * L[i * (i + 1) / 2 + i];
            }
        }
#pragma unroll
        for (int a = 0; a < 6; ++a) {
#pragma unroll
            for (int b = 0; b <= a; ++b) {
                double v = 0.0;
#pragma unroll
                for (int k = a; k < 6; ++k) v += X[k * (k + 1) / 2 + a] * X[k * (k + 1) / 2 + b];
                if (LMPC_LANE == ((a * (a + 1) / 2 + b) % LMPC_NLANE)) {
                    w.Wi[a * 6 + b] = v;
                    w.Wi[b * 6 + a] = v;
                }
            }
        }
        if (!ok) w.flag = ST_NUMERICAL;
        wsync();
        return delta;
    }

    // right-hand side of the terminal block for one solve: c1 (all lanes) and beta.
    // b1 = rhs of the simplex row (= -(sum lam - 1)).
    static LMPC_HD void terminal_rhs(W& w, RG& g, double b1, double* c1, double& beta) {
        double acc[6] = {0, 0, 0, 0, 0, 0}, sb = 0.0;
        FOR_SLOTS(r, row, R4) {
            double t = w.d4i[row] * g.rho[r];
            sb += t;
#pragma unroll
            for (int a = 0; a < 6; ++a) acc[a] += (w.SS[a * M + row] - w.sbar[a]) * t;
        }
        double v[7] = {acc[0], acc[1], acc[2], acc[3], acc[4], acc[5], sb};
        wsumv<7>(w, v);
#pragma unroll
        for (int a = 0; a < 6; ++a) c1[a] = -v[a] - w.sbar[a] * b1;
        beta = b1 - v[6];
    }

    // ---------------------------------------------------------------- backward sweeps ----
#if !LMPC_MMA
    // Start of a backward sweep: terminal cost-to-go into (Paug | pb[N&1]) and pi_N.
    template <bool FACTOR>
    static LMPC_HD void backward_start(W& w, const FtocpConst& c, const double* c1) {
        if (FACTOR) {
            FOR_LANES(e, 64) {
                const int i = e >> 3, j = e & 7;
                w.Paug[i * PS + j] = (i < 6 && j < 6) ? c.Qf2[i * 6 + j] + (LMPC ? w.Wi[(i * 6 + j) % TMW] : 0.0) : 0.0;
            }
            FOR_LANES(a, 8) {   // pi_N = -(Qf2 x_N + qxN + yT)
                double v = 0.0;
                if (a < 6) {
                    v = c.qxN[a] + (LMPC ? w.yT[a] : 0.0);
#pragma unroll
                    for (int b = 0; b < 6; ++b) v += c.Qf2[a * 6 + b] * w.x[N * 6 + b];
                }
                w.pi[N & 1][a] = -v;
            }
        }
        FOR_LANES(a, 8) {
            double v = 0.0;
            if (LMPC && a < 6) {
#pragma unroll
                for (int b = 0; b < 6; ++b) v += w.Wi[(a * 6 + b) % TMW] * c1[b];
            }
            w.pb[N & 1][a] = v;
        }
        wsync();
    }

#endif

    // r~_k: right-hand side contribution of the eliminated inequality rows (state part j < 6, input part r < 2)
    static LMPC_HD double rhs_x(const W& w, const FtocpConst& c, int k, int j) {
        double v = 0.0;
#pragma unroll
        for (int i = 0; i < NCX; ++i) v += c.Fx[i * 6 + j] * w.ex[k * NCX + i];
        return v;
    }
    static LMPC_HD double rhs_u(const W& w, const FtocpConst& c, int k, int r) {
        double v = 0.0;
#pragma unroll
        for (int jj = 0; jj < NCU; ++jj) v += c.Fu[jj * 2 + r] * w.eu[k * NCU + jj];
        return v;
    }

#if !LMPC_MMA
    // Stage gradients for the costate / input-residual recursion (embarrassingly parallel over stages).
    static LMPC_HD void stage_gradients(W& w, const FtocpConst& c) {
        FOR_LANES(e, N * 8) {
            const int k = e >> 3, j = e & 7;
            double v;
            if (j < 6) {
                v = c.qx[j];
#pragma unroll
                for (int b = 0; b < 6; ++b) v += c.Q2[j * 6 + b] * w.x[k * 6 + b];
#pragma unroll
                for (int i = 0; i < NCX; ++i) v += c.Fx[i * 6 + j] * w.dx[k * NCX + i];
            } else {
                const int r = j - 6;
                const double uk = w.u[k * 2 + r];
                const double up = (k == 0) ? w.uOld[r] : w.u[(k - 1) * 2 + r];
                v = c.R2[r * 2] * w.u[k * 2] + c.R2[r * 2 + 1] * w.u[k * 2 + 1] + c.dR2[r] * (uk - up);
                if (k < N - 1) v += c.dR2[r] * (uk - w.u[(k + 1) * 2 + r]);
#pragma unroll
                for (int jj = 0; jj < NCU; ++jj) v += c.Fu[jj * 2 + r] * w.dx[N * NCX + k * NCU + jj];
            }
            w.gst[k][j] = v;
        }
    }
#endif

    static constexpr int KF = (NCX > NCU ? NCX : NCU);
#if !LMPC_MMA
    // work item e < 36 of phase b/e: entry (i, j), i <= j, of the 8 x 8 stage matrix and its constant data
    struct SEnt {
        int i, j, cls;       // class 0 = state-state, 1 = input-state, 2 = input-input
        double kq, kf[KF];
    };
    static LMPC_HD void s_entry(const FtocpConst& c, int e, SEnt& q) {
        q.i = q.j = 0; q.cls = 1; q.kq = 0.0;
#pragma unroll
        for (int z = 0; z < KF; ++z) q.kf[z] = 0.0;
        if (e >= 36) return;
        tri8(e, q.i, q.j);
        if (q.j < 6) {
            q.cls = 0;
            q.kq = c.Q2[q.i * 6 + q.j];
#pragma unroll
            for (int z = 0; z < NCX; ++z) q.kf[z] = c.Fx[z * 6 + q.i] * c.Fx[z * 6 + q.j];
        } else if (q.i >= 6) {
            q.cls = 2;
            q.kq = c.R2[(q.i - 6) * 2 + (q.j - 6)];
#pragma unroll
            for (int z = 0; z < NCU; ++z) q.kf[z] = c.Fu[z * 2 + (q.i - 6)] * c.Fu[z * 2 + (q.j - 6)];
        }
    }

    // Factorising backward sweep on the augmented state (x, v): Riccati matrices, gradient recursion for the
    // predictor right-hand side and the costate / input-residual recursion.  Four uniform phases per stage.
    static LMPC_HD double backward_factor(W& w, const FtocpConst& c) {
        double ru_max = 0.0;
        // loop-invariant per-lane work assignment, cached in registers on the device (2 items per lane)
        constexpr bool CACHED = (LMPC_NLANE == 32);
        SEnt se[CACHED ? 2 : 1];
        if (CACHED) {
            s_entry(c, LMPC_LANE, se[0]);
            s_entry(c, LMPC_LANE + 32, se[CACHED ? 1 : 0]);
        }
        for (int k = N - 1; k >= 0; --k) {
            const double* T = &w.ABC[k][0];           // T[j*6 + c] = [A B](c, j)
            const double* pn = w.pb[(k + 1) & 1];     // px | pv of stage k+1
            const double* pin = w.pi[(k + 1) & 1];    // pi_{k+1}
            // ---- phase a: Gt[j][a] = (Paug A~)(a, j)
            FOR_LANES(e, 64) {
                const int j = e >> 3, a = e & 7;
                double v = dot6v(&T[j * 6], &w.Paug[a * PS]);
                if (j >= 6) v += w.Paug[a * PS + j];
                w.Gt[j * PS + a] = v;
            }
            wsync();
            // ---- phase b: S = A~' G~ + stage Hessian (36 entries), then the vector recursions (8 items)
            {
                int t = 0;
                FOR_LANES(e, 44) {
                    if (e < 36) {
                        SEnt qq;
                        if (!CACHED) s_entry(c, e, qq);
                        const SEnt& q = CACHED ? se[t] : qq;
                        const int i = q.i, j = q.j;
                        double v = dot6v(&T[i * 6], &w.Gt[j * PS]);
                        if (i >= 6) v += w.Gt[j * PS + i];
                        if (q.cls == 0) {
                            v += q.kq;
#pragma unroll
                            for (int z = 0; z < NCX; ++z) v += w.Dt[k * NCX + z] * q.kf[z];
                        } else if (q.cls == 2) {
                            v += q.kq;
                            if (i == j) v += ((k < N - 1) ? 2.0 : 1.0) * c.dR2[i - 6];
#pragma unroll
                            for (int z = 0; z < NCU; ++z) v += w.d2[k * NCU + z] * q.kf[z];
                        }
                        w.S[i * 8 + j] = v;
                        w.S[j * 8 + i] = v;
                    } else {
                        const int j = e - 36;                       // 0..7
                        const double hp = dot6v(&T[j * 6], pn);     // A~' p
                        const double tp = dot6v(&T[j * 6], pin);    // A~' pi
                        if (j < 6) {
                            w.hv[j] = rhs_x(w, c, k, j) + hp;
                            w.pi[k & 1][j] = tp - w.gst[k][j];
                        } else {
                            const double ru = w.gst[k][j] - tp;
                            w.ru[k][j - 6] = ru;
                            w.hv[j] = ru + rhs_u(w, c, k, j - 6) + hp + pn[j];
                        }
                    }
                    ++t;
                }
            }
            wsync();
            // ---- phase c/d: 2x2 Cholesky (lane redundant), Z~, z0
            {
                double l00s = w.S[6 * 8 + 6], l10 = w.S[7 * 8 + 6], l11s = w.S[7 * 8 + 7];
                bool bad = !(l00s > 0.0);
                if (bad) l00s = 1.0;
                const double i00 = rsqrt_f64(l00s);
                l10 *= i00;
                double tt = l11s - l10 * l10;
                if (!(tt > 0.0)) { bad = true; tt = 1.0; }
                const double i11 = rsqrt_f64(tt);
                ru_max = fmax(ru_max, fmax(fabs(w.ru[k][0]), fabs(w.ru[k][1])));
                FOR_LANES(j, 9) {
                    if (j < 8) {
                        const double y0 = (j < 6) ? w.S[6 * 8 + j] : (j == 6 ? -c.dR2[0] : 0.0);
                        const double y1 = (j < 6) ? w.S[7 * 8 + j] : (j == 7 ? -c.dR2[1] : 0.0);
                        const double z0c = y0 * i00;
                        w.Zt[k][j] = z0c;
                        w.Zt[k][8 + j] = (y1 - l10 * z0c) * i11;
                    } else {
                        const double a0 = w.hv[6] * i00;
                        w.z0[k][0] = a0;
                        w.z0[k][1] = (w.hv[7] - l10 * a0) * i11;
                        w.Li[k][0] = i00;
                        w.Li[k][1] = l10;
                        w.Li[k][2] = i11;
                        if (bad) w.flag = ST_NUMERICAL;
                    }
                }
            }
            wsync();
            // ---- phase e: cost-to-go of stage k: Paug = [Sxx 0; 0 0] - Z~'Z~ ; p = [hx; 0] - Z~' z0
            {
                const double* Z = w.Zt[k];
                const double a0 = w.z0[k][0], a1 = w.z0[k][1];
                double* po = w.pb[k & 1];
                int t = 0;
                FOR_LANES(e, 44) {
                    if (e < 36) {
                        SEnt qq;
                        if (!CACHED) s_entry(c, e, qq);
                        const SEnt& q = CACHED ? se[t] : qq;
                        const int i = q.i, j = q.j;
                        const double v = ((q.cls == 0) ? w.S[i * 8 + j] : 0.0) - Z[i] * Z[j] - Z[8 + i] * Z[8 + j];
                        w.Paug[i * PS + j] = v;
                        w.Paug[j * PS + i] = v;
                    } else {
                        const int a = e - 36;
                        po[a] = ((a < 6) ? w.hv[a] : 0.0) - Z[a] * a0 - Z[8 + a] * a1;
                    }
                    ++t;
                }
            }
            wsync();
        }
        return ru_max;
    }

    // Gradient-only backward sweep for a new right-hand side (corrector), one phase per stage.
    static LMPC_HD void backward_rhs(W& w, const FtocpConst& c) {
        for (int k = N - 1; k >= 0; --k) {
            const double* T = &w.ABC[k][0];
            const double* pn = w.pb[(k + 1) & 1];
            double* po = w.pb[k & 1];
            double g0[2];
#pragma unroll
            for (int r = 0; r < 2; ++r) g0[r] = w.ru[k][r] + rhs_u(w, c, k, r) + pn[6 + r] + dot6v(&T[(6 + r) * 6], pn);
            const double a0 = g0[0] * w.Li[k][0];
            const double a1 = (g0[1] - w.Li[k][1] * a0) * w.Li[k][2];
            FOR_LANES(a, 8) {
                double v = 0.0;
                if (a < 6) v = rhs_x(w, c, k, a) + dot6v(&T[a * 6], pn);
                po[a] = v - w.Zt[k][a] * a0 - w.Zt[k][8 + a] * a1;
                if (a >= 6) w.z0[k][a - 6] = (a == 6) ? a0 : a1;
            }
            wsync();
        }
    }

    // ---------------------------------------------------------------- forward sweep ------
    static LMPC_HD void forward(W& w) {
        FOR_LANES(a, 6) w.dx[a] = 0.0;
        wsync();
        double dv0 = 0.0, dv1 = 0.0;
        for (int k = 0; k < N; ++k) {
            const double* T = &w.ABC[k][0];
            const double* Z = w.Zt[k];
            const double* d = &w.dx[k * 6];
            const double t0 = w.z0[k][0] + dot6v(Z, d) + Z[6] * dv0 + Z[7] * dv1;
            const double t1 = w.z0[k][1] + dot6v(Z + 8, d) + Z[14] * dv0 + Z[15] * dv1;
            const double du1 = -t1 * w.Li[k][2];
            const double du0 = (-t0 - w.Li[k][1] * du1) * w.Li[k][0];
            FOR_LANES(a, 8) {
                if (a < 6) {
                    double v = T[36 + a] * du0 + T[42 + a] * du1;
#pragma unroll
                    for (int b = 0; b < 6; ++b) v += T[b * 6 + a] * d[b];
                    w.dx[(k + 1) * 6 + a] = v;
                } else {
                    w.du[k * 2 + (a - 6)] = (a == 6) ? du0 : du1;
                }
            }
            dv0 = du0;
            dv1 = du1;
            wsync();
        }
    }

#else   // ======================================================================== LMPC_MMA: tensor-core sweeps
    // The sweeps of one interior-point iteration on fp64 tensor-core fragments (mma.sync.m8n8k4.f64, SASS DMMA).
    //
    // Fragment convention ("D layout" of an 8 x 8 matrix X): lane l = 4 r + q (r = l >> 2, q = l & 3) holds
    //   X.a = X[r][2q],  X.b = X[r][2q+1]                       -- the accumulator layout of m8n8k4.
    // With the summation index split into even / odd columns, two MMAs give a full 8 x 8 x 8 product WITHOUT any register
    // shuffle between chained products:
    //   prod(X, YT) = X Y    where YT is the D layout of Y' :   mma(X.a, YT.a) + mma(X.b, YT.b)
    // (A operand X[r][2q] = X.a; B operand Y[2q][r] = Y'[r][2q] = YT.a; same for the odd half.)  The result is again in D
    // layout, so products chain; a symmetric matrix serves as both X and YT.  Row vectors ride in rows 0 / 1 of a fragment.
    //
    // Augmented state w = (x, v) with v_k = u_{k-1}; A~ = [A B; 0 I] maps (x_k, u_k) to w_{k+1}.  Per stage, with the cost-to-go
    // Hessian P of stage k+1:   S = A~' P A~ + H_k,   H_k = blkdiag(2Q, 2R + rate) + Fa' diag(Wd_k) Fa,  Fa = [Fx 0; 0 Fu],
    //   Y = [Sux | -dR2],  W = Suu^-1 Y (2 x 2 adjugate, no square roots),  K = -W,  M = [I 0; K],  P_k = [Sxx 0; 0 0] - Y'W,
    //   gradient  c_k = M'(A~' c + g_k),   f_k = -Suu^-1 (A~' c + g_k)_u,        g_k = stage gradient + eliminated-row terms,
    //   where c = (cost-to-go gradient) - (costate, 0): the costate recursion pi_k = A' pi - gst_x drops out of the solve and is
    //   only carried (row 1) in the factorising sweep to report the input-stationarity residual ru = gst_u - B' pi.
    // forward (open loop, M > 0):  (x_k, u_k) = M w_k + (0, f_k),  w_{k+1} = A~ (x_k, u_k).
    // Closed loop (M == 0): the vector sweeps run on the stage variables z_k = (x_k, u_k) with Phi_k = M_k A~_{k-1} (k >= 1),
    // one 8 x 8 x 8 product per stage; its rows 0..5 are [A B]_{k-1} as staged, rows 6,7 = K_k A~_{k-1} are stored (Kst):
    //   backward:  h_{N-1} = A~'_{N-1} c_N + g_{N-1},  h_{k-1} = Phi_k' h_k + g_{k-1}   (h_k = A~' c_{k+1} + g_k, c_k = M' h_k)
    //   forward:   z_0 = (0, f_0),  z_k = Phi_k z_{k-1} + (0, f_k),  x_N = [A B]_{N-1} z_{N-1}.
    // Both forms solve the same system; they round differently.  On MPC-type QPs the closed-loop solutions agree with the
    // open-loop ones to rounding and take the same iterations.  The LMPC terminal block (covariance form, degenerate simplex)
    // amplifies any reordering of the sweep arithmetic to ~1e-10 in the solution and an iteration more or less on some QPs, and
    // closed-loop LMPC roll-outs are chaotic, so a kernel with a safe set keeps the open-loop sweeps and its results.
    static constexpr bool CLOSED = (M == 0);
    struct Frag { double a, b; };

    static LMPC_HD void dmma(double& d0, double& d1, double a, double b, double c0, double c1) {
#if defined(__CUDA_ARCH__)
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%4,%5};"
                     : "=d"(d0), "=d"(d1) : "d"(a), "d"(b), "d"(c0), "d"(c1));
#endif
    }
    // LMPC_PROD_CHAIN: accumulate the odd half through the C operand of the second MMA (two dependent MMAs, no extra adds)
    // instead of two independent MMAs and a pair of DADDs (shorter chain, two more fp64 instructions per product).
#ifndef LMPC_PROD_CHAIN
#define LMPC_PROD_CHAIN 1
#endif
    static LMPC_HD Frag prod(const Frag& X, const Frag& YT) {
        Frag e, o;
        dmma(e.a, e.b, X.a, YT.a, 0.0, 0.0);
#if LMPC_PROD_CHAIN
        dmma(o.a, o.b, X.b, YT.b, e.a, e.b);
        return o;
#else
        dmma(o.a, o.b, X.b, YT.b, 0.0, 0.0);
        return Frag{e.a + o.a, e.b + o.b};
#endif
    }
    static LMPC_HD Frag prod_add(const Frag& X, const Frag& YT, const Frag& C) {
        Frag e, o;
        dmma(e.a, e.b, X.a, YT.a, C.a, C.b);
#if LMPC_PROD_CHAIN
        dmma(o.a, o.b, X.b, YT.b, e.a, e.b);
        return o;
#else
        dmma(o.a, o.b, X.b, YT.b, 0.0, 0.0);
        return Frag{e.a + o.a, e.b + o.b};
#endif
    }
    static LMPC_HD double bcast(double v, int src) {
#if defined(__CUDA_ARCH__)
        return __shfl_sync(0xffffffffu, v, src);
#else
        return v;
#endif
    }
    static LMPC_HD Frag ld2(const double* p) {
        const double2 v = *reinterpret_cast<const double2*>(p);
        return Frag{v.x, v.y};
    }
    static LMPC_HD void st2(double* p, double a, double b) { *reinterpret_cast<double2*>(p) = make_double2(a, b); }

    // Lane-constant addressing of the stage-data fragments.  A lane whose fragment entry is a structural constant (identity /
    // zero rows of A~ and M) reads it from w.cst with stride 0, so the sweeps contain no lane-dependent branches.
    // Offsets are doubles from sweep_base(): the staged model in shared memory, or -- STREAM -- the instance's model in global
    // memory, in which case the shared-memory operands (constants, gains) sit at 64-bit generic-address distances from it.
    static constexpr bool STREAM = W::STREAM;
    using Off = typename std::conditional<STREAM, long long, int>::type;
    struct LaneMap {
        int r, q;
        Off at_a, at_b; int at_step;   // D layout of A~' : (A~[2q][r], A~[2q+1][r]); per-stage step
        Off af; int af_step;           // D layout of A~  : (A~[r][2q], A~[r][2q+1]) as one 16-byte load
        // open loop (M > 0)
        Off mf; int mf_step;           // D layout of M   : rows 6,7 = K (from Kst), identity elsewhere
        Off mt_a, mt_b; int mt_step;   // D layout of M'  : (M[2q][r], M[2q+1][r]); q == 3 -> (K0[r], K1[r])
        // closed loop (M == 0): Phi_k (k >= 1) at Phi_1 + (k - 1) * step; rows / columns 0..5 from the stage model of k - 1,
        // 6,7 from Kst[k]
        Off pf; int pf_step;           // D layout of Phi : (Phi[r][2q], Phi[r][2q+1]); r >= 6 -> one 16-byte load from Kst
        Off pt_a, pt_b; int pt_step;   // D layout of Phi': (Phi[2q][r], Phi[2q+1][r]); q == 3 -> (Kst[0][r], Kst[1][r])
        Off cst;                       // the constant block (1,0 | 0,1 | 0,0)
    };
    // base address of the stage model as the sweeps see it.  STREAM: a global pointer made opaque, so that the compiler treats
    // base + offset as a generic address (the offsets of the shared-memory operands leave the global allocation)
    static LMPC_HD const double* sweep_base(const W& w) {
#if defined(__CUDA_ARCH__)
        if constexpr (STREAM) {
            const double* p = w.gabc;
            asm volatile("" : "+l"(p));
            return p;
        }
#endif
        return &w.ABC[0][0];
    }
    static LMPC_HD Off base_off(const W& w, const double* base, const double* p) {
#if defined(__CUDA_ARCH__)
        if constexpr (STREAM) {
            (void)w;
            const double* q = p;                    // generic address of the shared-memory operand
            asm volatile("" : "+l"(q));
            return (Off)(((long long)(size_t)q - (long long)(size_t)base) / 8);
        }
#endif
        (void)base;
        return (Off)(p - &w.ABC[0][0]);
    }
    static constexpr int STAGE = 54;
    static LMPC_HD int stage_step(const W& w) { if constexpr (STREAM) return w.gstage; else return STAGE; }
    // The lane id the sweeps derive their roles from.  Made opaque to the optimiser on purpose: otherwise every role mask and
    // address of a sweep is hoisted out of the interior-point loop and stays live (in registers or spilled) across the row loops.
    static LMPC_HD int sweep_lane() {
        int lane = LMPC_LANE;
#if defined(__CUDA_ARCH__)
        asm volatile("" : "+r"(lane));
#endif
        return lane;
    }
    static LMPC_HD LaneMap lane_map(const W& w, int lane) {
        LaneMap m{};
        m.r = lane >> 2;
        m.q = lane & 3;
        const int r = m.r, q = m.q;
        const double* base = sweep_base(w);
        const Off abc0 = 0;
        const Off cst0 = base_off(w, base, &w.cst[0]);
        const Off kst0 = base_off(w, base, &w.Kst[0][0]);
        const int stg = stage_step(w);
        m.cst = cst0;
        // A~ = [A B; 0 I], A row major (a*6+b) at 0, B (a*2+j) at 36
        if (q < 3) {
            m.at_a = abc0 + ((r < 6) ? (2 * q) * 6 + r : 36 + (2 * q) * 2 + (r - 6));
            m.at_b = abc0 + ((r < 6) ? (2 * q + 1) * 6 + r : 36 + (2 * q + 1) * 2 + (r - 6));
            m.at_step = stg;
        } else {                       // rows 6,7 of A~: (delta(r==6), delta(r==7))
            m.at_a = cst0 + ((r == 6) ? 0 : 1);
            m.at_b = cst0 + ((r == 7) ? 0 : 1);
            m.at_step = 0;
        }
        if (r < 6) { m.af = abc0 + ((q < 3) ? r * 6 + 2 * q : 36 + 2 * r); m.af_step = stg; }
        else { m.af = cst0 + ((q == 3) ? ((r == 6) ? 0 : 2) : 4); m.af_step = 0; }
        if constexpr (CLOSED) {
            if (r < 6) { m.pf = m.af; m.pf_step = stg; }
            else { m.pf = kst0 + 16 + (r - 6) * 8 + 2 * q; m.pf_step = 16; }
            if (q < 3) { m.pt_a = m.at_a; m.pt_b = m.at_b; m.pt_step = stg; }
            else { m.pt_a = kst0 + 16 + r; m.pt_b = kst0 + 24 + r; m.pt_step = 16; }
        } else {
            if (r >= 6) { m.mf = kst0 + (r - 6) * 8 + 2 * q; m.mf_step = 16; }
            else { m.mf = cst0 + ((r == 2 * q) ? 0 : ((r == 2 * q + 1) ? 2 : 4)); m.mf_step = 0; }
            if (q == 3) { m.mt_a = kst0 + r; m.mt_b = kst0 + 8 + r; m.mt_step = 16; }
            else { m.mt_a = cst0 + ((r == 2 * q) ? 0 : 1); m.mt_b = cst0 + ((r == 2 * q + 1) ? 0 : 1); m.mt_step = 0; }
        }
        return m;
    }

    // Right-hand side rows of the eliminated inequality constraints for a NEW right-hand side (corrector): row 0 of gv becomes
    // stage gradient + (Fx' ex | Fu' eu); row 1 (= -stage gradient, written by stage_gradients) is kept.
    static LMPC_HD void stage_rhs(W& w, const FtocpConst& c) {
        const int lane = sweep_lane();
        const int r = lane >> 2, q = lane & 3;
        const Frag FaT = fa_t_frag(c, r, q);
#pragma unroll
        for (int t = 0; t < (N + 7) / 8; ++t) {
            const int k = 8 * t + r;
            const bool live = k < N;
            const int kk = live ? k : N - 1;
            const Frag R = prod(row_frag(&w.ex[kk * NCX], &w.eu[kk * NCU], q), FaT);
            if (live) {
                const Frag G = ld2(&w.gv[k][8 + 2 * q]);
                st2(&w.gv[k][2 * q], R.a - G.a, R.b - G.b);
            }
        }
    }

    // D layout of Fa', Fa = [Fx 0; 0 Fu; 0 I2] (constraint rows x stage variables)
    static LMPC_HD Frag fa_t_frag(const FtocpConst& c, int r, int q) {
        Frag FaT{0.0, 0.0};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = 2 * q + h;
            double v = 0.0;
            if (row < NCX) v = (r < 6) ? c.Fx[row * 6 + r] : 0.0;
            else if (row < NCX + NCU) v = (r >= 6) ? c.Fu[(row - NCX) * 2 + (r - 6)] : 0.0;
            else if (row >= 6) v = (r == row) ? 1.0 : 0.0;
            if (h == 0) FaT.a = v; else FaT.b = v;
        }
        return FaT;
    }
    // entries (2q, 2q+1) of one stage's per-constraint-row vector (lane rows | input rows | 0 0), as an A operand
    static LMPC_HD Frag row_frag(const double* px, const double* pu, int q) {
        Frag v{0.0, 0.0};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = 2 * q + h;
            double t = 0.0;
            if (row < NCX) t = px[row];
            else if (row < NCX + NCU) t = pu[row - NCX];
            if (h == 0) v.a = t; else v.b = t;
        }
        return v;
    }

    // Stage gradients for the costate / input-residual recursion, eight stages per tensor-core tile:
    //   G = (x_k | u_k) blkdiag(2Q, 2R) + (nu1_k | nu2_k) Fa + (qx | input-rate terms),   R = (ex_k | eu_k) Fa
    // gv row 0 = G + R (predictor right-hand side incl. the eliminated rows' contribution), row 1 = -G.
    static LMPC_HD void stage_gradients(W& w, const FtocpConst& c) {
        const int lane = sweep_lane();
        const int r = lane >> 2, q = lane & 3;
        Frag Hc{0.0, 0.0};
        if (r < 6 && q < 3) Hc = Frag{c.Q2[r * 6 + 2 * q], c.Q2[r * 6 + 2 * q + 1]};
        if (r >= 6 && q == 3) Hc = Frag{c.R2[(r - 6) * 2], c.R2[(r - 6) * 2 + 1]};
        const Frag FaT = fa_t_frag(c, r, q);
        const Frag Cq = (q < 3) ? Frag{c.qx[2 * q], c.qx[2 * q + 1]} : Frag{0.0, 0.0};
#pragma unroll
        for (int t = 0; t < (N + 7) / 8; ++t) {
            const int k = 8 * t + r;
            const bool live = k < N;
            const int kk = live ? k : N - 1;
            const Frag Z = ld2((q < 3) ? &w.x[kk * 6 + 2 * q] : &w.u[kk * 2]);
            // input-rate terms (PC.py:233-242): dR2 (u_k - u_{k-1}) + dR2 (u_k - u_{k+1}), the latter not at the last stage
            const Frag uk = ld2(&w.u[kk * 2]);
            const Frag up = ld2((kk == 0) ? &w.uOld[0] : &w.u[(kk - 1) * 2]);
            const Frag un = ld2(&w.u[((kk < N - 1) ? kk + 1 : kk) * 2]);      // (last stage: u_k - u_k = 0)
            Frag C0 = Cq;
            if (q == 3) C0 = Frag{c.dR2[0] * ((uk.a - up.a) + (uk.a - un.a)), c.dR2[1] * ((uk.b - up.b) + (uk.b - un.b))};
            Frag G = prod_add(Z, Hc, C0);
            G = prod_add(row_frag(&w.dx[kk * NCX], &w.dx[N * NCX + kk * NCU], q), FaT, G);
            const Frag R = prod(row_frag(&w.ex[kk * NCX], &w.eu[kk * NCU], q), FaT);
            if (live) {
                st2(&w.gv[k][2 * q], G.a + R.a, G.b + R.b);
                st2(&w.gv[k][8 + 2 * q], -G.a, -G.b);
            }
        }
    }

    // tN = Qf2 x_N + qxN + yT (minus the costate at the end of the horizon), once per iteration
    static LMPC_HD void terminal_costate(W& w, const FtocpConst& c) {
        FOR_LANES(a, 8) {
            double t = 0.0;
            if (a < 6) {
                t = c.qxN[a] + (LMPC ? w.yT[a] : 0.0);
#pragma unroll
                for (int b = 0; b < 6; ++b) t += c.Qf2[a * 6 + b] * w.x[N * 6 + b];
            }
            w.tN[a] = t;
        }
    }
    // Row vectors at the end of the horizon: row 0 = Wi c1 + tN (gradient minus costate), row 1 = -tN (costate; FACTOR only)
    template <bool FACTOR>
    static LMPC_HD Frag terminal_vec(const W& w, const double* c1, int r, int q) {
        Frag V{0.0, 0.0};
        if (r <= (FACTOR ? 1 : 0)) {
            const Frag t = ld2(&w.tN[2 * q]);
            if (r == 1) { V.a = -t.a; V.b = -t.b; }
            else {
                V = t;
                if (LMPC && q < 3) {
#pragma unroll
                    for (int b = 0; b < 6; ++b) {
                        V.a += w.Wi[((2 * q) * 6 + b) % TMW] * c1[b];
                        V.b += w.Wi[((2 * q + 1) * 6 + b) % TMW] * c1[b];
                    }
                }
            }
        }
        return V;
    }

    // Factorising backward sweep; carries the gradient recursion of the predictor right-hand side (row 0) and the costate
    // recursion (row 1, only to report the input-stationarity residual).  Returns max |ru|.
    // The loop body is branch-free: lane roles are encoded in 0/1 masks and per-lane addresses, stage data is read through
    // running pointers one stage ahead of its use (the dependent chain is MMA -> MMA -> shuffle -> rsqrt -> MMA).
    static LMPC_HD double backward_factor(W& w, const FtocpConst& c, const double* c1) {
        const int lane = sweep_lane();
        const LaneMap lm = lane_map(w, lane);
        const int r = lm.r, q = lm.q;
        const double* base = sweep_base(w);
        // constant part of the stage Hessian in D layout: blkdiag(2Q, 2R)
        Frag Hc{0.0, 0.0};
        if (r < 6 && q < 3) Hc = Frag{c.Q2[r * 6 + 2 * q], c.Q2[r * 6 + 2 * q + 1]};
        if (r >= 6 && q == 3) Hc = Frag{c.R2[(r - 6) * 2], c.R2[(r - 6) * 2 + 1]};
        // D layout of Fa', Fa = [Fx 0; 0 Fu; 0 I2]: rows 6,7 select the inputs, their weights Wd[k][6..7] carry the input-rate
        // cost (2 dR2, the last stage 1 dR2) so that the variable part of the stage Hessian is ONE product Fa' diag(Wd_k) Fa
        const Frag FaT = fa_t_frag(c, r, q);
        // lane roles as 0/1 factors (selects on doubles cost two instructions each, a multiply-add one)
        const double m_x = (r < 6) ? 1.0 : 0.0;                               // column r of Y comes from S (else: the -dR2 constant)
        const double y0c = (r == 6) ? -c.dR2[0] : 0.0, y1c = (r == 7) ? -c.dR2[1] : 0.0;
        const double m_keep = (r < 6 && q < 3) ? 1.0 : 0.0;                   // entries of Sxx
        const double m_q01 = (q < 2) ? 1.0 : 0.0, m_q3 = (q == 3) ? 1.0 : 0.0;
        const double m_ru = (lane == 7) ? 0.0 : 1.0;                          // the costate has no input part
        const Frag Id = Frag{(q < 3 && r == 2 * q) ? 1.0 : 0.0, (q < 3 && r == 2 * q + 1) ? 1.0 : 0.0};   // M' for q < 3 (open loop)
        // closed loop: K in the D layout of M (lane (r >= 6, q): K[r-6][2q], K[r-6][2q+1]): column j of W sits in the lanes 4j..4j+3, and
        // the lanes with odd q hand out row 1, those with even q row 0
        const int k_src = 8 * q + (r & 1);

        // terminal cost-to-go
        Frag Pf{0.0, 0.0};
        if (r < 6 && q < 3) {
            Pf.a = c.Qf2[r * 6 + 2 * q] + (LMPC ? w.Wi[(r * 6 + 2 * q) % TMW] : 0.0);
            Pf.b = c.Qf2[r * 6 + 2 * q + 1] + (LMPC ? w.Wi[(r * 6 + 2 * q + 1) % TMW] : 0.0);
        }
        Frag Vf = terminal_vec<true>(w, c1, r, q);      // row vectors of stage k+1: c_N first, then c_{k+1} / (closed loop) h_{k+1}
        bool bad = false;
        // running pointers (stage N-1 first); lanes without a role in a load / store point at the zero constants / a dump slot
        const double* pa = base + lm.at_a + (N - 1) * lm.at_step;
        const double* pb_ = base + lm.at_b + (N - 1) * lm.at_step;
        const double* pw = &w.Wd[N - 1][2 * q];
        const double* pg = (lane < 8) ? &w.gv[N - 1][2 * lane] : &w.cst[4];
        const int g_step = (lane < 8) ? 16 : 0;
        double* pk = &w.Kst[N - 1][r];
        double* psi = &w.Sinv[N - 1][0];
        double* pfs = &w.fst[N - 1][0];
        double* pru = &w.ru[N - 1][0];
        Frag At{*pa, *pb_}, Gn = ld2(pg), Wn = ld2(pw);
        Frag PhT = At;                 // closed loop: D layout of the map of the row vectors, A~'_{N-1} first, then Phi_{k+1}'
LMPC_SWEEP_UNROLL
        for (int k = N - 1; k >= 0; --k) {
            const Frag AtF = At, g = Gn, wd = Wn, PT = PhT;
            {   // prefetch the next stage's operands (k == 0 re-reads stage 0: no branch, nothing out of bounds)
                const int st = (k > 0) ? 1 : 0;
                pa -= st * lm.at_step; pb_ -= st * lm.at_step; pw -= st * 8; pg -= st * g_step;
                At = Frag{*pa, *pb_};
                Gn = ld2(pg);
                Wn = ld2(pw);
            }
            // ---- stage Hessian: constant part + Fa' diag(Wd_k) Fa as one product (independent of the Riccati chain)
            const Frag Hf = prod_add(Frag{FaT.a * wd.a, FaT.b * wd.b}, FaT, Hc);
            // ---- S = A~' P A~ + H
            const Frag Gp = prod(AtF, Pf);                 // A~' P   (P symmetric: its D layout is also its transposed layout)
            const Frag S = prod_add(Gp, AtF, Hf);
            // ---- row vectors: h_k = A~' c + g (= Phi_{k+1}' h_{k+1} + g) (row 0), A~' pi - gst (row 1); rows 2..7 stay 0
            const Frag Tv = prod(Vf, CLOSED ? PT : AtF);
            const Frag Hraw{Tv.a + g.a, Tv.b + g.b};
            if (lane == 7) st2(pru, -Hraw.a, -Hraw.b);      // ru = gst_u - B' pi
            const Frag Hv{Hraw.a * m_ru, Hraw.b * m_ru};
            // ---- eliminate the inputs: Suu^-1 by the adjugate (2 x 2, every lane the same values; no square roots), W = Suu^-1 Y,
            //      K = -W,  P_k = [Sxx 0; 0 0] - Y'W  (Y = [Sux | -dR2]; column r of Sux = S[r][6..7] sits in lane 4r+3)
            double s66 = bcast(S.a, 27);
            const double s76 = bcast(S.a, 31);
            const double s77 = bcast(S.b, 31);
            double y0 = bcast(S.a, lane | 3), y1 = bcast(S.b, lane | 3);
            if (!(s66 > 0.0)) { bad = true; s66 = 1.0; }
            double det = fma(s66, s77, -s76 * s76);
            if (!(det > 0.0)) { bad = true; det = 1.0; }
            const double idet = recip(det);
            const double s00 = s77 * idet, s01 = -s76 * idet, s11 = s66 * idet;
            y0 = fma(m_x, y0, y0c);
            y1 = fma(m_x, y1, y1c);
            const double w0r = fma(s00, y0, s01 * y1);
            const double w1r = fma(s01, y0, s11 * y1);
            const double wq = (q & 1) ? w1r : w0r;
            // ---- feed-forward term f = -Suu^-1 h_u (h_u sits in lane 3)
            if (lane == 3) {
                st2(psi, s00, s01);
                psi[2] = s11;
                st2(pfs, -fma(s00, Hv.a, s01 * Hv.b), -fma(s01, Hv.a, s11 * Hv.b));
            }
            // ---- cost-to-go Hessian of stage k as one MMA (summation index 0,1 used: rows of Y and W)
            dmma(Pf.a, Pf.b, -((q & 1) ? y1 : y0), m_q01 * wq, m_keep * S.a, m_keep * S.b);
            if constexpr (CLOSED) {
                // ---- Phi_k' = A~'_{k-1} M_k' (At holds A~_{k-1}; at k == 0 a product that is never read): only the q == 3
                //      columns (K_k A~_{k-1})' differ from A~'_{k-1}; they are stored for the vector sweeps.  Off the Riccati chain.
                const Frag WA = prod(At, Frag{bcast(wq, k_src), bcast(wq, k_src + 4)});     // W = -K
                const Frag KA{-WA.a, -WA.b};
                if (q == 3) { pk[0] = KA.a; pk[8] = KA.b; }
                PhT = (q == 3) ? KA : At;
                // ---- the row vectors go on in h-form: the costate passes through Phi (its input part is zero, row 1)
                Vf = Hv;
            } else {
                if (q == 0) { pk[0] = -w0r; pk[8] = -w1r; }
                // ---- c_k = M' h (row 0); the costate passes through the identity part (row 1)
                Vf = prod(Hv, Frag{fma(-m_q3, w0r, Id.a), fma(-m_q3, w1r, Id.b)});
            }
            pk -= 16; psi -= 4; pfs -= 2; pru -= 2;
        }
        if (bad && lane == 0) w.flag = ST_NUMERICAL;
        wsync();
        double ru_max = 0.0;
        FOR_LANES(e, N * 2) ru_max = fmax(ru_max, fabs(w.ru[e >> 1][e & 1]));
        return wmax_nn(ru_max);
    }

    // Closed-loop gradient-only backward sweep for a new right-hand side (corrector / recentring): h_{k-1} = Phi_k' h_k + g_{k-1}, f_k.
    static LMPC_HD void backward_rhs_closed(W& w, const FtocpConst& c, const double* c1) {
        const int lane = sweep_lane();
        const LaneMap lm = lane_map(w, lane);
        const int r = lm.r, q = lm.q;
        const double* base = sweep_base(w);
        Frag Hv = terminal_vec<false>(w, c1, r, q);    // c_N, then h_{k+1}
        // Phi_{N-1}', Phi_{N-2}', ..., Phi_1' in turn; the pointer stays at stage 1 once there (no read out of bounds)
        const double* pa = base + lm.pt_a + (N - 2) * lm.pt_step;
        const double* pb_ = base + lm.pt_b + (N - 2) * lm.pt_step;
        const double* pg = (lane < 4) ? &w.gv[N - 1][2 * lane] : &w.cst[4];
        const int g_step = (lane < 4) ? 16 : 0;
        const double* psi = &w.Sinv[N - 1][0];
        double* pfs = &w.fst[N - 1][0];
        Frag Pt{base[lm.at_a + (N - 1) * lm.at_step], base[lm.at_b + (N - 1) * lm.at_step]};   // A~'_{N-1}: c_N enters through A~
        Frag Gn = ld2(pg), Sn = ld2(psi);
        Frag Pt2 = Pt;                 // STREAM: the model comes from L2, so its fragments are fetched two stages ahead
        if constexpr (STREAM) { Pt2 = Frag{*pa, *pb_}; pa -= lm.pt_step; pb_ -= lm.pt_step; }
        double S2n = psi[2];
LMPC_SWEEP_UNROLL
        for (int k = N - 1; k >= 0; --k) {
            const Frag PT = Pt, g = Gn, s0 = Sn;
            const double s11 = S2n;
            {   // prefetch the next stage's operands off the dependent chain (k == 0 re-reads stage 0 / Phi_1')
                const int st = (k > 0) ? 1 : 0;
                pg -= st * g_step; psi -= st * 4;
                if constexpr (STREAM) {
                    Pt = Pt2;
                    Pt2 = Frag{*pa, *pb_};                 // Phi_{k-1}'
                    const int s2 = (k > 2) ? 1 : 0;
                    pa -= s2 * lm.pt_step; pb_ -= s2 * lm.pt_step;
                } else {
                    Pt = Frag{*pa, *pb_};                  // Phi_k'
                    const int s1 = (k > 1) ? 1 : 0;
                    pa -= s1 * lm.pt_step; pb_ -= s1 * lm.pt_step;
                }
                Gn = ld2(pg);
                Sn = ld2(psi);
                S2n = psi[2];
            }
            Hv = prod_add(Hv, PT, g);                      // h_k (row 0; other rows 0)
            if (lane == 3) st2(pfs, -fma(s0.a, Hv.a, s0.b * Hv.b), -fma(s0.b, Hv.a, s11 * Hv.b));
            pfs -= 2;
        }
        wsync();
    }

    // Closed-loop forward sweep on the stage variables: z_0 = (0, f_0), z_k = Phi_k z_{k-1} + (0, f_k), dx_N = [A B]_{N-1} z_{N-1}.
    static LMPC_HD void forward_closed(W& w) {
        const int lane = sweep_lane();
        const LaneMap lm = lane_map(w, lane);
        const double* base = sweep_base(w);
        const double* pp = base + lm.pf;               // Phi_1
        const double* pc = (lane == 3) ? &w.fst[0][0] : &w.cst[4];
        const int c_step = (lane == 3) ? 2 : 0;
        // one store per stage: lanes 0..2 write dx_k, lane 3 writes du_k
        double* po = (lane < 3) ? &w.dx[2 * lane] : &w.du[0];
        const int o_step = (lane < 3) ? 6 : 2;
        Frag Z = ld2(pc);                             // row 0: (dx_0 | du_0) = (0 | f_0)
        pc += c_step;
        Frag Pf = ld2(pp), Cf = ld2(pc);
        Frag Pf2 = Pf;                 // STREAM: two stages ahead (see backward_rhs)
        if constexpr (STREAM) { pp += ((N > 2) ? 1 : 0) * lm.pf_step; Pf2 = ld2(pp); }
LMPC_SWEEP_UNROLL
        for (int k = 1; k < N; ++k) {
            const Frag PF = Pf, CF = Cf;
            {   // prefetch the next stage's operands off the dependent chain (the last stage re-reads itself)
                const int st = (k + 1 < N) ? 1 : 0;
                pc += st * c_step;
                if constexpr (STREAM) {
                    pp += ((k + 2 < N) ? 1 : 0) * lm.pf_step;
                    Pf = Pf2;
                    Pf2 = ld2(pp);
                } else {
                    pp += st * lm.pf_step;
                    Pf = ld2(pp);
                }
                Cf = ld2(pc);
            }
            if (lane < 4) st2(po, Z.a, Z.b);               // z_{k-1}
            po += o_step;
            Z = prod_add(Z, PF, CF);                       // row 0: (dx_k | du_k)
        }
        if (lane < 4) st2(po, Z.a, Z.b);
        const Frag X = prod(Z, ld2(base + lm.af + (N - 1) * lm.af_step));     // row 0: (dx_N | du_{N-1})
        if (lane < 3) st2(&w.dx[N * 6 + 2 * lane], X.a, X.b);
        wsync();
    }

    // Open-loop gradient-only backward sweep for a new right-hand side (corrector / recentring): c_k = M'(A~'c + g_k), f_k.
    static LMPC_HD void backward_rhs_open(W& w, const FtocpConst& c, const double* c1) {
        const int lane = sweep_lane();
        const LaneMap lm = lane_map(w, lane);
        const int r = lm.r, q = lm.q;
        const double* base = sweep_base(w);
        Frag Vf = terminal_vec<false>(w, c1, r, q);
        const double* pa = base + lm.at_a + (N - 1) * lm.at_step;
        const double* pb_ = base + lm.at_b + (N - 1) * lm.at_step;
        const double* ma = base + lm.mt_a + (N - 1) * lm.mt_step;
        const double* mb = base + lm.mt_b + (N - 1) * lm.mt_step;
        const double* pg = (lane < 4) ? &w.gv[N - 1][2 * lane] : &w.cst[4];
        const int g_step = (lane < 4) ? 16 : 0;
        const double* psi = &w.Sinv[N - 1][0];
        double* pfs = &w.fst[N - 1][0];
        Frag At{*pa, *pb_}, Mt{*ma, *mb}, Gn = ld2(pg), Sn = ld2(psi);
        Frag At2 = At;                 // STREAM: the model comes from L2, so its fragments are fetched two stages ahead
        if constexpr (STREAM) { pa -= lm.at_step; pb_ -= lm.at_step; At2 = Frag{*pa, *pb_}; }
        double S2n = psi[2];
LMPC_SWEEP_UNROLL
        for (int k = N - 1; k >= 0; --k) {
            const Frag AtF = At, MT = Mt, g = Gn, s0 = Sn;
            const double s11 = S2n;
            {   // prefetch the next stage's operands off the dependent chain (k == 0 re-reads stage 0)
                const int st = (k > 0) ? 1 : 0;
                ma -= st * lm.mt_step; mb -= st * lm.mt_step;
                pg -= st * g_step; psi -= st * 4;
                if constexpr (STREAM) {
                    const int s2 = (k > 1) ? 1 : 0;
                    pa -= s2 * lm.at_step; pb_ -= s2 * lm.at_step;
                    At = At2;
                    At2 = Frag{*pa, *pb_};
                } else {
                    pa -= st * lm.at_step; pb_ -= st * lm.at_step;
                    At = Frag{*pa, *pb_};
                }
                Mt = Frag{*ma, *mb};
                Gn = ld2(pg);
                Sn = ld2(psi);
                S2n = psi[2];
            }
            const Frag Tv = prod(Vf, AtF);
            const Frag Hv{Tv.a + g.a, Tv.b + g.b};         // rows other than 0: 0 + 0
            if (lane == 3) st2(pfs, -fma(s0.a, Hv.a, s0.b * Hv.b), -fma(s0.b, Hv.a, s11 * Hv.b));
            pfs -= 2;
            Vf = prod(Hv, MT);
        }
        wsync();
    }

    // Open-loop forward sweep: (dx_k, du_k) = M w_k + (0, f_k), w_{k+1} = A~ (dx_k, du_k), from w_0 = 0.
    static LMPC_HD void forward_open(W& w) {
        const int lane = sweep_lane();
        const LaneMap lm = lane_map(w, lane);
        const double* base = sweep_base(w);
        const double* pf = base + lm.af;
        const double* pm = base + lm.mf;
        const double* pc = (lane == 3) ? &w.fst[0][0] : &w.cst[4];
        const int c_step = (lane == 3) ? 2 : 0;
        // one store per stage: lanes 0..2 write dx_k, lane 3 writes du_k
        double* po = (lane < 3) ? &w.dx[2 * lane] : &w.du[0];
        const int o_step = (lane < 3) ? 6 : 2;
        Frag Wf{0.0, 0.0};
        Frag Af = ld2(pf), Mf = ld2(pm), Cf = ld2(pc);
        Frag Af2 = Af;                 // STREAM: two stages ahead (see backward_rhs)
        if constexpr (STREAM) { pf += lm.af_step; Af2 = ld2(pf); }
LMPC_SWEEP_UNROLL
        for (int k = 0; k < N; ++k) {
            const Frag AF = Af, MF = Mf, CF = Cf;
            {   // prefetch the next stage's operands off the dependent chain (the last stage re-reads itself)
                const int st = (k + 1 < N) ? 1 : 0;
                pm += st * lm.mf_step; pc += st * c_step;
                if constexpr (STREAM) {
                    pf += ((k + 2 < N) ? 1 : 0) * lm.af_step;
                    Af = Af2;
                    Af2 = ld2(pf);
                } else {
                    pf += st * lm.af_step;
                    Af = ld2(pf);
                }
                Mf = ld2(pm);
                Cf = ld2(pc);
            }
            const Frag Uf = prod_add(Wf, MF, CF);          // row 0: (dx_k | du_k)
            if (lane < 4) st2(po, Uf.a, Uf.b);
            po += o_step;
            Wf = prod(Uf, AF);                             // row 0: (dx_{k+1} | du_k)
        }
        if (lane < 3) st2(&w.dx[N * 6 + 2 * lane], Wf.a, Wf.b);
        wsync();
    }

    static LMPC_HD void backward_rhs(W& w, const FtocpConst& c, const double* c1) {
        if constexpr (CLOSED) backward_rhs_closed(w, c, c1);
        else backward_rhs_open(w, c, c1);
    }
    static LMPC_HD void forward(W& w) {
        if constexpr (CLOSED) forward_closed(w);
        else forward_open(w);
    }

    // Model roll-out of a starting point with the inputs in w.u: (x_{k+1} | u_k) = A~ (x_k | u_k) + (C_k | 0)
    static LMPC_HD void rollout(W& w, const double* x0) {
        const int lane = sweep_lane();
        const LaneMap lm = lane_map(w, lane);
        const double* base = sweep_base(w);
        const double* pf = base + lm.af;
        const double* pc = base + ((lane < 3) ? (Off)(48 + 2 * lane) : lm.cst + 4);
        const int c_step = (lane < 3) ? stage_step(w) : 0;
        Frag Wf{0.0, 0.0};
#pragma unroll
        for (int h = 0; h < 3; ++h)
            if (lane == h) Wf = Frag{x0[2 * h], x0[2 * h + 1]};
        if (lane < 3) st2(&w.x[2 * lane], Wf.a, Wf.b);
        LMPC_SWEEP_UNROLL
        for (int k = 0; k < N; ++k) {
            if (lane == 3) Wf = ld2(&w.u[k * 2]);
            Wf = prod_add(Wf, ld2(pf), ld2(pc));
            pf += lm.af_step; pc += c_step;
            if (lane < 3) st2(&w.x[(k + 1) * 6 + 2 * lane], Wf.a, Wf.b);
        }
        wsync();
    }
#endif  // LMPC_MMA

    // terminal recovery after a forward sweep: dlam (registers); returns dy1.
    // The 6x6 covariance-form solve loses ~cond(W)*eps in dyT, which the division by a small d4 amplifies in
    // the dlam of active safe-set points.  One step of iterative refinement with the residual of
    //     Tinv dyT + S~ dlam = dx_N - sbar*b1
    // evaluated THROUGH the recovered dlam removes it (oracle/pdip_model.py W_REFINE).
    static LMPC_HD double terminal_recover(W& w, RG& g, const FtocpConst& c, const double* c1, double beta,
                                           double delta, double b1) {
        // the 6 x 6 products run one row per lane; the results travel through shared memory
        double dyT[6];
        wsync();                                   // earlier readers of tv are done
        FOR_LANES(a, 6) {
            double t = 0.0;
#pragma unroll
            for (int b = 0; b < 6; ++b) t += w.Wi[a * 6 + b] * (w.dx[N * 6 + b] + c1[b]);
            w.tv[a] = t;
        }
        wsync();
#pragma unroll
        for (int a = 0; a < 6; ++a) dyT[a] = w.tv[a];
        const double dy1t = -beta * recip(delta);
        double acc[6] = {0, 0, 0, 0, 0, 0};
        FOR_SLOTS(r, row, R4) {
            double t = g.rho[r] - dy1t;
#pragma unroll
            for (int a = 0; a < 6; ++a) t += (w.SS[a * M + row] - w.sbar[a]) * dyT[a];
            t *= w.d4i[row];
            g.dlam[r] = t;
#pragma unroll
            for (int a = 0; a < 6; ++a) acc[a] += (w.SS[a * M + row] - w.sbar[a]) * t;
        }
        wsumv<6>(w, acc);                          // also leaves the sums in w.red
        FOR_LANES(a, 6) {                          // residual of the terminal equality through the recovered dlam (tv is free: dyT is in registers)
            double t = w.dx[N * 6 + a] - w.sbar[a] * b1 - w.red[a];
#pragma unroll
            for (int b = 0; b < 6; ++b) t -= c.Tinv[a * 6 + b] * dyT[b];
            w.tv[a] = t;
        }
        wsync();
        FOR_LANES(a, 6) {                          // (red is free: its sums were consumed above)
            double t = 0.0;
#pragma unroll
            for (int b = 0; b < 6; ++b) t += w.Wi[a * 6 + b] * w.tv[b];
            w.red[a] = t;
        }
        wsync();
        double ddy[6];
        double sdy = 0.0;
#pragma unroll
        for (int a = 0; a < 6; ++a) {
            ddy[a] = w.red[a];
            sdy += w.sbar[a] * (dyT[a] + ddy[a]);
        }
        FOR_SLOTS(r, row, R4) {
            double t = 0.0;
#pragma unroll
            for (int a = 0; a < 6; ++a) t += (w.SS[a * M + row] - w.sbar[a]) * ddy[a];
            g.dlam[r] += t * w.d4i[row];
        }
        return dy1t + sdy;
    }

    // ---------------------------------------------------------------- the solver ---------
    // Preconditions: w.ABC, w.SS, w.Qfun, w.uOld loaded and visible to the warp; x0[6].
    // warm: this controller's warm-start record (WS_SIZE doubles, global memory) or null; warm_valid: in = the record holds a
    // snapshot of the previous solve, out = it holds one of this solve.
    static LMPC_HD void solve(W& w, const FtocpConst& c, const double* x0, SolveInfo& info,
                              double* lam_out /* M or null */, double* slack_out /* R1 or null */,
                              double* warm = nullptr, int* warm_valid = nullptr) {
        RG g;
        if (LMPC_LANE == 0) w.flag = 0;
        wsync();
        bool snapped = (warm == nullptr), warm_started = false, warm_restarted = false;
        // late_it / max_it: iteration limits of the start the solve runs from; a restart moves both by restart_it, so the cold
        // start that replaces a warm one has the budget it would have had without the record
        int late_it = LATE_ACCEPT_IT, max_it = c.max_iter;
        const int restart_it = (c.max_iter < WARM_MAX_ITERS) ? c.max_iter : WARM_MAX_ITERS;
        int age = 0;
        if (warm != nullptr) {
            age = *warm_valid;                            // 0 = no record, else 1 + number of solves it has been carried through
            warm_started = (age >= 1 && age <= WARM_MAX_AGE);
        }
        if (warm_started) warm_point(w, g, c, x0, warm);
        else init_point(w, g, c, x0);
        wsync();
        if (warm != nullptr && LMPC_LANE == 0) *warm_valid = 0;
        const double n_ineq = (double)(2 * R1 + R2 + (LMPC ? M : 0));
        int it = 0, status = ST_MAX_ITER, late = 0;
        double r_prim = 0.0, r_dual = 0.0, mu = 0.0, ru_prev = 0.0, al_prev = 0.0, step_prev = 1e300;
        // the iterate meets eps_res / eps_gap and is only refined further for the eps_step criterion: if that refinement breaks
        // down at rounding level (no positive step, lost pivot, iteration limit), the iterate is the answer, not a failure
        bool res_ok = false;
        const double d4_floor = c.d4_min;

        for (;; ++it) {
            if (warm_started && it == restart_it) {
                // a start from the previous solve's iterate that is still not through: give the QP the cold start it would have
                // had without the record (the same answer at the same tolerances, restart_it iterations later), drop the record
                init_point(w, g, c, x0, false);
                wsync();
                warm_started = false;
                warm_restarted = true;
                late_it = LATE_ACCEPT_IT + restart_it;
                max_it = c.max_iter + restart_it;
                al_prev = 0.0; ru_prev = 0.0; step_prev = 1e300; res_ok = false;
            }
            // ---- lane-local residuals, barrier diagonals, predictor right-hand sides -------
            double comp = 0.0, rd_loc = 0.0;
            FOR_SLOTS(r, row, R1) {
                int k = row / NCX, i = row % NCX;
                double w1 = c.bx[i] - dot6(&c.Fx[i * 6], &w.x[k * 6]) + g.s[r];   // derived slack
                g.w1[r] = w1;
                double rs = c.qs2 * g.s[r] + c.ql - g.nu1[r] - g.nu3[r];
                g.rs[r] = rs;
                rd_loc = fmax(rd_loc, fabs(rs));
                comp += w1 * g.nu1[r] + g.s[r] * g.nu3[r];
                const double iw1 = recip(w1), is = recip(g.s[r]);
                g.iw1[r] = iw1;
                g.is_[r] = is;
                double d1 = g.nu1[r] * iw1, d3 = g.nu3[r] * is;
                const double ihs = recip(c.qs2 + d1 + d3);
                g.d1[r] = d1;
                g.ihs[r] = ihs;
                LMPC_WDT(w, k, i, row) = d1 * (c.qs2 + d3) * ihs;
                // predictor: rc1 = w1 nu1, rc3 = s nu3  ->  e1 = -nu1, rs + rc3/s = rs + nu3
                w.ex[row] = (-g.nu1[r] * (c.qs2 + d3) + d1 * (rs + g.nu3[r])) * ihs;
                w.dx[row] = g.nu1[r];
            }
            FOR_SLOTS(r, row, R2) {
                int k = row / NCU, j = row % NCU;
                double w2 = c.bu[j] - (c.Fu[j * 2] * w.u[k * 2] + c.Fu[j * 2 + 1] * w.u[k * 2 + 1]);
                g.w2[r] = w2;
                comp += w2 * g.nu2[r];
                const double iw2 = recip(w2);
                g.iw2[r] = iw2;
                LMPC_WD2(w, k, j, row) = g.nu2[r] * iw2;
                w.eu[row] = -g.nu2[r];           // predictor: -rc2/w2
                w.dx[N * NCX + row] = g.nu2[r];
            }
            double rone = 0.0, delta = 1.0, beta = 0.0, c1[6] = {0, 0, 0, 0, 0, 0};
            if (LMPC) {
                rone = terminal_state(w, g, c);
                FOR_SLOTS(r, row, R4) {
                    double rl = w.Qfun[row] + g.y1 - g.nu4[r];
#pragma unroll
                    for (int a = 0; a < 6; ++a) rl -= w.SS[a * M + row] * w.yT[a];
                    g.rl[r] = rl;
                    rd_loc = fmax(rd_loc, fabs(rl));
                    comp += g.lam[r] * g.nu4[r];
                    g.ilam[r] = recip(g.lam[r]);
                    g.rho[r] = -rl - g.nu4[r];   // predictor: rc4/lam = nu4
                }
            } else {
                wsync();
            }
            comp = wsum(comp);
            mu = comp * (1.0 / n_ineq);
            if (!snapped && mu <= WARM_SNAP_MU) {                // record this iterate for the controller's next solve
                if (mu >= WARM_MIN_MU) {
                    warm_snapshot(w, g, warm);
                    if (LMPC_LANE == 0) *warm_valid = warm_started ? age + 1 : 1;
                }
                snapped = true;
            }
            rd_loc = wmax_nn(rd_loc);
            r_prim = fabs(rone);
            if (it > 0 && step_prev < 1e299) {      // (not right after a (re)start: there is no previous step to extrapolate from)
                // The input-stationarity residual is linear in the iterate and every variable moved by the same step
                // length, so after a step alpha it is exactly (1 - alpha) times its previous value: convergence can be
                // decided here, before paying for another factorisation.
                r_dual = fmax(rd_loc, (1.0 - al_prev) * ru_prev);
                // Residuals and gap alone do not bound the distance to the optimum: on a QP without strict complementarity the
                // iterate trails the solution by O(sqrt(mu)) (one of the 4096 configs[1] QPs sat 7.5e-6 away at mu = 1e-11 with
                // residuals at rounding level).  The primal step just taken does: the iteration is superlinear, so once a step
                // moved (x, u) by less than eps_step the remaining distance is smaller still.
                res_ok = (r_prim <= c.eps_res && r_dual <= c.eps_res && mu <= c.eps_gap);
                if (res_ok && step_prev <= c.eps_step) { status = ST_SOLVED; break; }
                // Stragglers: on a few LMPC instances (LP-degenerate simplex block) the covariance-form recovery of
                // d(lambda) puts a noise floor of ~1e-7..1e-6 under the dual residual and the tail converges linearly.
                // Once the iterate meets the 1e-6 parity contract, stop after LATE_ACCEPT_IT iterations (and at max_iter).
                if ((it >= late_it || it >= max_it) && r_prim <= 1e-6 && r_dual <= 1e-6 && mu <= 1e-6) {
                    status = ST_SOLVED;
                    late = res_ok ? 0 : 1;
                    break;
                }
                if (it >= max_it) { status = ST_MAX_ITER; break; }
            }
            // ---- factorising backward sweep (also yields the input residual) ------------------
            if (LMPC) {
                delta = terminal_factor(w, g, c, d4_floor);
                terminal_rhs(w, g, -rone, c1, beta);
            }
            stage_gradients(w, c);
#if LMPC_MMA
            terminal_costate(w, c);
            wsync();
            const double ru_max = backward_factor(w, c, c1);
#else
            backward_start<true>(w, c, c1);
            const double ru_max = backward_factor(w, c);
#endif
            ru_prev = ru_max;
            r_dual = fmax(rd_loc, ru_max);
            if (w.flag != 0) { status = res_ok ? ST_SOLVED : w.flag; break; }
            if (r_prim <= c.eps_res && r_dual <= c.eps_res && mu <= c.eps_gap && step_prev <= c.eps_step) { status = ST_SOLVED; break; }
            if (it >= max_it) {
                if (res_ok) { status = ST_SOLVED; }
                else if (r_prim <= 1e-6 && r_dual <= 1e-6 && mu <= 1e-6) { status = ST_SOLVED; late = 1; }
                else { status = ST_MAX_ITER; }
                break;
            }

            // ---- predictor -----------------------------------------------------------------------
            forward(w);
            double dy1 = 0.0;
            if (LMPC) dy1 = terminal_recover(w, g, c, c1, beta, delta, -rone);
            double rn = 0.0, rd = 1.0;
            FOR_SLOTS(r, row, R1) {
                int k = row / NCX, i = row % NCX;
                double fdx = dot6(&c.Fx[i * 6], &w.dx[k * 6]);
                double gs = -g.rs[r] - g.nu1[r] - g.nu3[r];
                double ds = (gs + g.d1[r] * fdx) * g.ihs[r];
                double dw1 = -fdx + ds;
                double dn1 = -g.nu1[r] - g.d1[r] * dw1;
                double dn3 = -g.nu3[r] - (g.nu3[r] * g.is_[r]) * ds;
                ratio_update(g.w1[r], dw1, rn, rd);
                ratio_update(g.s[r], ds, rn, rd);
                ratio_update(g.nu1[r], dn1, rn, rd);
                ratio_update(g.nu3[r], dn3, rn, rd);
                g.p1[r] = dw1 * dn1;
                g.p3[r] = ds * dn3;
            }
            FOR_SLOTS(r, row, R2) {
                int k = row / NCU, j = row % NCU;
                double dw2 = -(c.Fu[j * 2] * w.du[k * 2] + c.Fu[j * 2 + 1] * w.du[k * 2 + 1]);
                double dn2 = -g.nu2[r] - (g.nu2[r] * g.iw2[r]) * dw2;
                ratio_update(g.w2[r], dw2, rn, rd);
                ratio_update(g.nu2[r], dn2, rn, rd);
                g.p2[r] = dw2 * dn2;
            }
            if (LMPC) {
                FOR_SLOTS(r, row, R4) {
                    double dn4 = -g.nu4[r] - (g.nu4[r] * g.ilam[r]) * g.dlam[r];
                    ratio_update(g.lam[r], g.dlam[r], rn, rd);
                    ratio_update(g.nu4[r], dn4, rn, rd);
                    g.p4[r] = g.dlam[r] * dn4;
                }
            }
            const double a_aff = wmin_nn(ratio_bound(rn, rd, 1.0));
            // complementarity after the affine step.  With p = dw*dnu and dw*nu + w*dnu = -w*nu:
            //   (w + a dw)(nu + a dnu) = w nu (1 - a) + a^2 p
            double comp_aff = 0.0;
            FOR_SLOTS(r, row, R1) {
                comp_aff += (g.w1[r] * g.nu1[r] + g.s[r] * g.nu3[r]) * (1.0 - a_aff) + a_aff * a_aff * (g.p1[r] + g.p3[r]);
            }
            FOR_SLOTS(r, row, R2) { comp_aff += g.w2[r] * g.nu2[r] * (1.0 - a_aff) + a_aff * a_aff * g.p2[r]; }
            if (LMPC) {
                FOR_SLOTS(r, row, R4) { comp_aff += g.lam[r] * g.nu4[r] * (1.0 - a_aff) + a_aff * a_aff * g.p4[r]; }
            }
            comp_aff = wsum(comp_aff);
            double sig = comp_aff * recip(comp);
            sig = LMPC_TUNE_SIGMA(sig);
            const double sm = sig * mu;

            // ---- corrector (pass 0), recentring (pass 1, rare) -----------------------------------------
            // Pass 0 is Mehrotra's corrector.  If its step cannot be brought back into the central-path neighbourhood within
            // RECENTRE_AFTER reductions, the iterate sits on the neighbourhood boundary and an aggressive sigma would only allow
            // tiny steps from now on (0.002 % of closed-loop LMPC steps stalled like that): pass 1 re-uses the factorisation
            // for a pure centring direction (sigma = 1, no second-order term) instead.
            double al = 0.0;
            double ds_[NSLOT(R1)], dw1_[NSLOT(R1)], dn1_[NSLOT(R1)], dn3_[NSLOT(R1)], dw2_[NSLOT(R2)], dn2_[NSLOT(R2)], dn4_[NSLOT(R4)];
            bool bad_step = false;
#pragma unroll 1
            for (int pass = 0; pass < 2; ++pass) {
#if defined(LMPC_HOST_COUNT) && !defined(__CUDA_ARCH__)
                g_host_count[pass] += 1;                 // host emulation only: corrector / recentring passes of a sweep run
#endif
                const double tgt = pass ? mu : sm;      // complementarity target
                const double so = pass ? 0.0 : 1.0;     // second-order (dw*dnu) term on/off
                FOR_SLOTS(r, row, R1) {
                    double rc1 = g.w1[r] * g.nu1[r] + so * g.p1[r] - tgt;
                    double rc3 = g.s[r] * g.nu3[r] + so * g.p3[r] - tgt;
                    double d3 = g.nu3[r] * g.is_[r];
                    double e1 = -rc1 * g.iw1[r];
                    w.ex[row] = (e1 * (c.qs2 + d3) + g.d1[r] * (g.rs[r] + rc3 * g.is_[r])) * g.ihs[r];
                    g.p1[r] = rc1;   // keep rc for the final recovery
                    g.p3[r] = rc3;
                }
                FOR_SLOTS(r, row, R2) {
                    double rc2 = g.w2[r] * g.nu2[r] + so * g.p2[r] - tgt;
                    w.eu[row] = -rc2 * g.iw2[r];
                    g.p2[r] = rc2;
                }
                if (LMPC) {
                    FOR_SLOTS(r, row, R4) {
                        double rc4 = g.lam[r] * g.nu4[r] + so * g.p4[r] - tgt;
                        g.rho[r] = -g.rl[r] - rc4 * g.ilam[r];
                        g.p4[r] = rc4;
                    }
                    terminal_rhs(w, g, -rone, c1, beta);
                }
                wsync();
#if LMPC_MMA
                stage_rhs(w, c);
                wsync();
                backward_rhs(w, c, c1);
#else
                backward_start<false>(w, c, c1);
                backward_rhs(w, c);
#endif
                forward(w);
                if (LMPC) dy1 = terminal_recover(w, g, c, c1, beta, delta, -rone);

                // ---- step length ---------------------------------------------------------------------
                rn = 0.0;
                rd = 1.0;
                FOR_SLOTS(r, row, R1) {
                    int k = row / NCX, i = row % NCX;
                    double fdx = dot6(&c.Fx[i * 6], &w.dx[k * 6]);
                    double rc1 = g.p1[r], rc3 = g.p3[r];
                    double gs = -g.rs[r] - rc1 * g.iw1[r] - rc3 * g.is_[r];
                    double ds = (gs + g.d1[r] * fdx) * g.ihs[r];
                    double dw1 = -fdx + ds;
                    double dn1 = (-rc1 - g.nu1[r] * dw1) * g.iw1[r];
                    double dn3 = (-rc3 - g.nu3[r] * ds) * g.is_[r];
                    ratio_update(g.w1[r], dw1, rn, rd);
                    ratio_update(g.s[r], ds, rn, rd);
                    ratio_update(g.nu1[r], dn1, rn, rd);
                    ratio_update(g.nu3[r], dn3, rn, rd);
                    ds_[r] = ds; dw1_[r] = dw1; dn1_[r] = dn1; dn3_[r] = dn3;
                }
                FOR_SLOTS(r, row, R2) {
                    int k = row / NCU, j = row % NCU;
                    double dw2 = -(c.Fu[j * 2] * w.du[k * 2] + c.Fu[j * 2 + 1] * w.du[k * 2 + 1]);
                    double dn2 = (-g.p2[r] - g.nu2[r] * dw2) * g.iw2[r];
                    ratio_update(g.w2[r], dw2, rn, rd);
                    ratio_update(g.nu2[r], dn2, rn, rd);
                    dw2_[r] = dw2; dn2_[r] = dn2;
                }
                if (LMPC) {
                    FOR_SLOTS(r, row, R4) {
                        double dn4 = (-g.p4[r] - g.nu4[r] * g.dlam[r]) * g.ilam[r];
                        ratio_update(g.lam[r], g.dlam[r], rn, rd);
                        ratio_update(g.nu4[r], dn4, rn, rd);
                        dn4_[r] = dn4;
                    }
                }
                const double amax = wmin_nn(ratio_bound(rn, rd, 1e300));
                al = fmin(1.0, LMPC_TUNE_STEP * amax);
                if (!(al > 0.0) || !(al <= 1.0)) { bad_step = true; break; }
                // Stay in a wide neighbourhood of the central path, min_i w_i nu_i >= gamma * mean: without it
                // Mehrotra steps can 2-cycle against a blocking bound (seen on 3 of 4096 workload QPs).
                bool inside = false;
                for (int tries = 0; tries < 12; ++tries) {
                    double pmin = 1e300, psum = 0.0;
                    FOR_SLOTS(r, row, R1) {
                        double a1 = (g.w1[r] + al * dw1_[r]) * (g.nu1[r] + al * dn1_[r]);
                        double a3 = (g.s[r] + al * ds_[r]) * (g.nu3[r] + al * dn3_[r]);
                        pmin = fmin(pmin, fmin(a1, a3));
                        psum += a1 + a3;
                    }
                    FOR_SLOTS(r, row, R2) {
                        double a2 = (g.w2[r] + al * dw2_[r]) * (g.nu2[r] + al * dn2_[r]);
                        pmin = fmin(pmin, a2);
                        psum += a2;
                    }
                    if (LMPC) {
                        FOR_SLOTS(r, row, R4) {
                            double a4 = (g.lam[r] + al * g.dlam[r]) * (g.nu4[r] + al * dn4_[r]);
                            pmin = fmin(pmin, a4);
                            psum += a4;
                        }
                    }
                    pmin = wmin(pmin);
                    psum = wsum(psum);
                    if (pmin >= (LMPC_TUNE_GAMMA / n_ineq) * psum) { inside = true; break; }
                    if (pass == 0 && tries >= RECENTRE_AFTER) break;
#if defined(LMPC_HOST_COUNT) && !defined(__CUDA_ARCH__)
                    g_host_count[2] += 1;                // step reductions
#endif
                    al *= LMPC_TUNE_BACKOFF;
                }
                if (inside) break;
            }
            if (bad_step) { status = res_ok ? ST_SOLVED : ST_NUMERICAL; break; }
#if defined(LMPC_HOST_TRACE) && !defined(__CUDA_ARCH__)
            printf("it %2d rp %.2e rd %.2e mu %.2e a_aff %.4f sig %.2e al %.4e\n", it, r_prim, r_dual, mu, a_aff, sig, al);
#endif
            FOR_SLOTS(r, row, R1) {
                g.s[r] += al * ds_[r];
                g.nu1[r] += al * dn1_[r];
                g.nu3[r] += al * dn3_[r];
            }
            FOR_SLOTS(r, row, R2) { g.nu2[r] += al * dn2_[r]; }
            if (LMPC) {
                FOR_SLOTS(r, row, R4) {
                    g.lam[r] += al * g.dlam[r];
                    g.nu4[r] += al * dn4_[r];
                }
                g.y1 += al * dy1;
            }
            al_prev = al;
            double dmax = 0.0;
            FOR_LANES(e, (N + 1) * 6) { const double d = al * w.dx[e]; w.x[e] += d; dmax = fmax(dmax, fabs(d)); }
            FOR_LANES(e, N * 2) { const double d = al * w.du[e]; w.u[e] += d; dmax = fmax(dmax, fabs(d)); }
            step_prev = wmax_nn(dmax);
            wsync();
        }

        // ---- final residual (adds the dynamics defect, which the iteration keeps at rounding level)
        double rdyn = 0.0;
        FOR_LANES(e, N * 6) {
            int k = e / 6, a = e % 6;
#if LMPC_MMA
            const double* T = sweep_base(w) + (long long)k * stage_step(w);
            double v = T[48 + a] + T[36 + a * 2] * w.u[k * 2] + T[37 + a * 2] * w.u[k * 2 + 1];      // stage record as loaded
#pragma unroll
            for (int b = 0; b < 6; ++b) v += T[a * 6 + b] * w.x[k * 6 + b];
#else
            const double* T = &w.ABC[k][0];
            double v = T[48 + a] + T[36 + a] * w.u[k * 2] + T[42 + a] * w.u[k * 2 + 1];              // transposed in place
#pragma unroll
            for (int b = 0; b < 6; ++b) v += T[b * 6 + a] * w.x[k * 6 + b];
#endif
            rdyn = fmax(rdyn, fabs(w.x[(k + 1) * 6 + a] - v));
        }
        r_prim = fmax(r_prim, wmax_nn(rdyn));
        if (warm != nullptr && (warm_restarted || (warm_started && status != ST_SOLVED)) && LMPC_LANE == 0) *warm_valid = 0;
        info.status = status;
        info.iters = it;
        info.late = late;
        info.r_prim = r_prim;
        info.r_dual = r_dual;
        info.gap = mu;
        if (LMPC && lam_out) {
            FOR_SLOTS(r, row, R4) { lam_out[row] = g.lam[r]; }
        }
        if (slack_out) {
            FOR_SLOTS(r, row, R1) { slack_out[row] = g.s[r]; }
        }
        wsync();
    }
};

}  // namespace lmpc
