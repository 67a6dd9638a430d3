// racinglmpc_b200/csrc/lmpc_b200.cu — kernels + C ABI (include/lmpc_b200.h) for sm_90a (H100).
//
// K3/K4/K5 of SURVEY §2.3 fused in one kernel: one warp (= one 32-thread CTA) per FTOCP instance.
//   load   : stage model (A_k,B_k,C_k) and the selected safe set are staged into shared memory with
//            1-D bulk async copies (cp.async.bulk -> UBLKCP, completion on an mbarrier)
//   solve  : racinglmpc_b200/csrc/ftocp_pdip.cuh (Mehrotra PDIP + Riccati, fp64, all in smem/registers)
//   unpack : xPred/uPred/lambd/slack + zt = Succ_SS lam, zt_u = Succ_uSS lam
//            (PredictiveControllers.py:364-384), coalesced stores
// Tensor cores only through the warp-level fp64 MMA (mma.sync.m8n8k4.f64): the largest contraction is 6x6x8 in fp64 and
// wgmma has no f64 type — see DESIGN.md.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <stdio.h>
#include <stdlib.h>
#include <string>
#include <new>
#include <ctype.h>
#include <errno.h>
#include <unistd.h>
#include <sys/syscall.h>
#include <sys/mman.h>
#include <map>
#include <vector>
#include <mutex>

#include "../../include/lmpc_b200.h"
#include "ftocp_pdip.cuh"
#include "safeset.cuh"
#include "lapbooks.cuh"
#include "probe.cuh"
#include "ftocp_launch.cuh"

using namespace lmpc;

#define LMPC_HOST_SLOTS 4              // buffer sets (batches in flight) of the asynchronous host entry points
#ifndef LMPC_STEP_SPLIT_DEFAULT
#define LMPC_STEP_SPLIT_DEFAULT 1     // instance ranges of the pipelined device-resident step (1 = one launch sequence)
#endif

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static int fail(int code, const std::string& msg) {
    g_err = msg;
    return code;
}
#define CK(call)                                                                                        \
    do {                                                                                                \
        cudaError_t e_ = (call);                                                                        \
        if (e_ != cudaSuccess) return fail(LMPC_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
    } while (0)

// The QP kernel's inputs and outputs for one whole batch: [B,6] x0, [B,2] uOld, [B,N,54] abc, [B,6,M] SS, [B,M] Qfun, [B,6,M]
// SuccSS, [B,2,M] SuccU, [B,N+1,6] xPred, [B,N,2] uPred, [B,N*2] slack, [B,M] lambd, [B,6] slackT, [B,6] zt, [B,2] ztu,
// [B,3] resid, [B] status, [B] iters (M = 1 for handles without a safe set)
struct QpBufs {
    double *x0, *uOld, *abc, *SS, *Qfun, *SuccSS, *SuccU, *xPred, *uPred, *slack, *lambd, *slackT, *zt, *ztu, *resid;
    int *status, *iters;
};

struct lmpc_handle {
    lmpc_params p;
    FtocpConst c;
    int batch, device, N, M;
    cudaStream_t stream;
    cudaStream_t cstream[4 * LMPC_HOST_SLOTS];   // chunk pipelines of the *_host entry points (H2D | kernel | D2H overlap), 4 streams per slot
    int hb_chunks[LMPC_HOST_SLOTS];
    bool hb_pending[LMPC_HOST_SLOTS];            // enqueued and not yet waited for
    bool hb_lone;                                // set by the synchronous entry points: the batch being enqueued runs alone
    // pipelined device-resident step: the batch is cut into step_split instance ranges, each running its kernel sequence on its
    // own stream (cstream[0..3]) between a fork and a join event on `stream`
    int step_split;
    cudaEvent_t ev_fork, ev_join[4];
    bool trace_on;
    cudaEvent_t tev[4][3], t0ev;
    long long launches;
    // QP buffer sets, one per slot of the *_host entry points.  hb[0] is allocated at creation and is also the device-resident
    // step's (K1 writes its abc, K2 its safe set, the QP kernel its outputs; lmpc_device_buffer); hb[1..] on first use.
    QpBufs hb[LMPC_HOST_SLOTS];
    unsigned long long* d_late;
    // warm-start records of the controllers of the device-resident step (lmpc_params.warm_start; allocated with the store)
    double* d_warm;
    int* d_warm_valid;
    long long warm_stride;
    int warm_mode;
    // per-controller parameters (lmpc_set_param_sets): table FtocpConstRec[nsets] and set index [batch]; null = uniform handle
    FtocpConstRec* d_sets;
    int* d_set_idx;
    // lap stores + controller state (lmpc_store_create)
    bool has_store;
    ModelConst mc;
    // tracks (lmpc_set_tracks): table TrackRec[ntrk] and track index [batch]; without sets a one-row table holding the track of
    // lmpc_store_create (store_trk) and a null index.  trk_host / trk_idx_host mirror both for the host-side lap restart.
    TrackRec store_trk;
    TrackRec* d_trk;
    int* d_trk_idx;
    std::vector<TrackRec> trk_host;
    std::vector<int> trk_idx_host;
    bool laps_stored;          // a lap entered either pool: the track table is fixed from now on
    LapPool ss, mdl;
    int *d_used, *d_sel, *d_isprev, *d_prevslot, *d_timeStep, *d_hasPred, *d_flags, *d_minidx, *d_xchg, *d_health, *d_dropped;
    double *d_xLin, *d_uLin, *d_ztState, *d_ztFixed, *d_OldInput, *d_xPredPrev, *d_tmpx, *d_tmpu;
    // device-resident closed loop (lmpc_rollout_create)
    bool has_rollout;
    int Tcl;
    unsigned long long sim_step;
    double *d_rx[2], *d_rg[2], *d_clx, *d_clu, *d_z, *d_zpid, *d_abc_lti;
    int *d_cllen, *d_done, cur;
    // vehicles of the simulator (lmpc_rollout_set_vehicles): table lmpc_vehicle_params[nsets] and vehicle index [batch]; without
    // sets a one-row table holding the reference vehicle and a null index (allocated at creation)
    lmpc_vehicle_params* d_veh;
    int* d_veh_idx;
    // device lap books (lapbooks.cuh): slot tables of both pools, lap history, exchange scratch
    LapBooks bk;
    int *d_bkbuf, *d_poolidx, *d_stats;
    bool has_books;
    // rollout trace of chosen controllers (presentation support, lmpc_rollout_trace_*)
    TraceBufs tr;
    int* d_trinst;
    bool has_trace;
};

static bool inv6(const double* A, double* Ai) {
    double m[6][12];
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) { m[i][j] = A[i * 6 + j]; m[i][6 + j] = (i == j) ? 1.0 : 0.0; }
    for (int col = 0; col < 6; ++col) {
        int piv = col;
        for (int r = col + 1; r < 6; ++r) if (fabs(m[r][col]) > fabs(m[piv][col])) piv = r;
        if (fabs(m[piv][col]) < 1e-300) return false;
        if (piv != col) for (int j = 0; j < 12; ++j) { double t = m[col][j]; m[col][j] = m[piv][j]; m[piv][j] = t; }
        double d = 1.0 / m[col][col];
        for (int j = 0; j < 12; ++j) m[col][j] *= d;
        for (int r = 0; r < 6; ++r)
            if (r != col) { double f = m[r][col]; if (f != 0.0) for (int j = 0; j < 12; ++j) m[r][j] -= f * m[col][j]; }
    }
    for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) Ai[i * 6 + j] = m[i][6 + j];
    return true;
}

static int build_const(const lmpc_params& p, FtocpConst& c) {
    for (int j = 0; j < p.ncu; ++j)
        if (!(p.bu[j] > 0.0)) return fail(LMPC_E_INVALID, "bu must be positive (u = 0 strictly feasible)");
    memset(&c, 0, sizeof(c));
    for (int i = 0; i < 36; ++i) { c.Q2[i] = 2.0 * p.Q[i]; c.Qf2[i] = 2.0 * p.Qf[i]; }
    for (int i = 0; i < 4; ++i) c.R2[i] = 2.0 * p.R[i];
    for (int a = 0; a < 6; ++a) {
        double s = 0, sN = 0;
        for (int b = 0; b < 6; ++b) { s += p.Q[a * 6 + b] * p.xRef[b]; sN += p.Qf[a * 6 + b] * p.xRef[b]; }
        c.qx[a] = -2.0 * s;
        c.qxN[a] = -2.0 * sN;
    }
    c.dR2[0] = 2.0 * p.dR[0];
    c.dR2[1] = 2.0 * p.dR[1];
    c.qs2 = 2.0 * p.Qslack[0];
    c.ql = p.Qslack[1];
    for (int i = 0; i < p.ncx * 6; ++i) c.Fx[i] = p.Fx[i];
    for (int i = 0; i < p.ncx; ++i) c.bx[i] = p.bx[i];
    for (int i = 0; i < p.ncu * 2; ++i) c.Fu[i] = p.Fu[i];
    for (int i = 0; i < p.ncu; ++i) c.bu[i] = p.bu[i];
    if (p.numSS_Points > 0) {
        for (int i = 0; i < 36; ++i) c.T[i] = 2.0 * p.QterminalSlack[i];
        if (!inv6(c.T, c.Tinv)) return fail(LMPC_E_INVALID, "QterminalSlack is singular");
    } else {
        for (int i = 0; i < 6; ++i) c.T[i * 6 + i] = c.Tinv[i * 6 + i] = 1.0;
    }
    c.eps_res = p.eps_res > 0 ? p.eps_res : 1e-9;
    c.eps_gap = p.eps_gap > 0 ? p.eps_gap : 1e-11;
    c.eps_step = p.eps_step > 0 ? p.eps_step : 1e-7;
    c.d4_min = 1e-6;
    c.max_iter = p.max_iter > 0 ? p.max_iter : 40;
    return LMPC_OK;
}

// Per-controller tables (lmpc_set_param_sets, lmpc_rollout_set_vehicles): `nsets` rows and one row index per controller.
// The argument rules both calls share: 0 <= nsets <= batch, nsets == 0 exactly when both arrays are NULL, every index in range.
static int check_set_index(const lmpc_handle* h, const char* who, const void* sets, int nsets, const int* set_of_instance) {
    const std::string w(who);
    if (nsets < 0 || nsets > h->batch) return fail(LMPC_E_INVALID, w + ": nsets must be 0 .. batch");
    if ((nsets == 0) != (sets == nullptr) || (nsets == 0) != (set_of_instance == nullptr))
        return fail(LMPC_E_INVALID, w + ": nsets == 0 goes with NULL sets and set_of_instance, nsets >= 1 with both");
    for (int b = 0; b < (nsets ? h->batch : 0); ++b)
        if (set_of_instance[b] < 0 || set_of_instance[b] >= nsets)
            return fail(LMPC_E_INVALID, w + ": set index of instance " + std::to_string(b) + " out of range");
    return LMPC_OK;
}

// Once the handle's streams are idle, replace the table *tab by rows[nrows] (none when nrows == 0) and the index *idx by
// set_of_instance[batch] (none when it is NULL).  The handle keeps its old table unless every allocation and copy succeeds.
template <typename T>
static int swap_table(lmpc_handle* h, const char* who, const T* rows, int nrows, const int* set_of_instance, T** tab, int** idx) {
    CK(cudaSetDevice(h->device));
    // batches already enqueued (the _async entry points, the device-resident step) finish with the table they were enqueued with
    CK(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < 4 * LMPC_HOST_SLOTS; ++i) CK(cudaStreamSynchronize(h->cstream[i]));
    T* t = nullptr;
    int* ix = nullptr;
    cudaError_t e = cudaSuccess;
    if (nrows > 0) {
        e = cudaMalloc((void**)&t, sizeof(T) * nrows);
        if (e == cudaSuccess) e = cudaMemcpy(t, rows, sizeof(T) * nrows, cudaMemcpyHostToDevice);
    }
    if (e == cudaSuccess && set_of_instance) {
        e = cudaMalloc((void**)&ix, sizeof(int) * h->batch);
        if (e == cudaSuccess) e = cudaMemcpy(ix, set_of_instance, sizeof(int) * h->batch, cudaMemcpyHostToDevice);
    }
    if (e != cudaSuccess) {
        cudaFree(t); cudaFree(ix);
        return fail(LMPC_E_CUDA, std::string(who) + ": " + cudaGetErrorString(e));
    }
    cudaFree(*tab);
    cudaFree(*idx);
    *tab = t;
    *idx = ix;
    return LMPC_OK;
}

// Simulator.dynModel's vehicle (SysModel.py:61-70), D in the reference's operation order
static lmpc_vehicle_params reference_vehicle() {
    lmpc_vehicle_params v;
    v.m = 1.98; v.lf = 0.125; v.lr = 0.125; v.Iz = 0.024;
    v.Df = 0.8 * v.m * 9.81 / 2.0; v.Cf = 1.25; v.Bf = 1.0;
    v.Dr = 0.8 * v.m * 9.81 / 2.0; v.Cr = 1.25; v.Br = 1.0;
    return v;
}

template <int N, int M>
static int configure_t(cudaStream_t) {
    CK(cudaFuncSetAttribute(ftocp_kernel<N, M, 2, 4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)sizeof(KernelSmem<N, M, 2, 4, false>)));
    return LMPC_OK;
}

template <int N, int M>
static int launch_t(lmpc_handle* h, const FtocpArgs& a, cudaStream_t st) {
    if (h->d_sets)     // the handle has per-controller parameters: every instance reads its own row (ftocp_sets.cu)
        CK(ftocp_sets_launch(N, M, h->d_sets, a, st));
    else {
        ftocp_kernel<N, M, 2, 4, false><<<a.batch, 32, sizeof(KernelSmem<N, M, 2, 4, false>), st>>>(h->c, a);
        CK(cudaGetLastError());
    }
    h->launches += 1;
    return LMPC_OK;
}

static int launch(lmpc_handle* h, const FtocpArgs& a, bool lmpc_mode, cudaStream_t st) {
    const int N = h->N, M = lmpc_mode ? h->M : 0;
#define LCASE(n, m) if (N == n && M == m) return launch_t<n, m>(h, a, st);
    LMPC_FOR_EACH_CASE(LCASE)
#undef LCASE
    return fail(LMPC_E_INVALID, "unsupported (N, numSS_Points): built for " LMPC_GRID_TEXT);
}

// Opt the kernels this handle can launch into their shared-memory size on the handle's device (the attribute is per device and
// per function: done once per handle at creation, on its device, so handles on different devices never depend on each other).
static int configure(int N, int M) {
    int hit = 0, rc = LMPC_OK;
#define CCASE(n, m) if (N == n && (m == 0 || m == M)) { ++hit; if (rc == LMPC_OK) rc = configure_t<n, m>(0); }
    LMPC_FOR_EACH_CASE(CCASE)
#undef CCASE
    if (rc != LMPC_OK) return rc;
    const bool have_m = (M == 0) || (hit == 2);
    if (hit == 0 || !have_m)
        return fail(LMPC_E_INVALID, "unsupported (N, numSS_Points): built for " LMPC_GRID_TEXT);
    CK(ftocp_sets_configure(N, M));      // the variant lmpc_set_param_sets switches to
    return LMPC_OK;
}

template <typename T>
static void free_null(T*& p) { if (p) cudaFree(p); p = nullptr; }

static void free_store(lmpc_handle* h) {
    free_null(h->ss.x); free_null(h->ss.u); free_null(h->ss.q); free_null(h->ss.len);
    free_null(h->mdl.x); free_null(h->mdl.u); free_null(h->mdl.len);
    free_null(h->d_used); free_null(h->d_sel); free_null(h->d_isprev); free_null(h->d_prevslot); free_null(h->d_timeStep);
    free_null(h->d_hasPred); free_null(h->d_flags); free_null(h->d_minidx); free_null(h->d_xLin); free_null(h->d_uLin);
    free_null(h->d_ztState); free_null(h->d_ztFixed); free_null(h->d_OldInput); free_null(h->d_xPredPrev); free_null(h->d_tmpx);
    free_null(h->d_tmpu); free_null(h->d_xchg); free_null(h->d_dropped);
    free_null(h->d_bkbuf); free_null(h->d_poolidx); free_null(h->d_stats);
    free_null(h->d_warm); free_null(h->d_warm_valid);
    free_null(h->d_trk); free_null(h->d_trk_idx);
    h->trk_host.clear(); h->trk_idx_host.clear();
    h->laps_stored = false;
    h->has_books = false;
    h->has_store = false;
}

static Tracks tracks(const lmpc_handle* h) { return Tracks{h->d_trk, h->d_trk_idx}; }

static void free_rollout(lmpc_handle* h) {
    for (int i = 0; i < 2; ++i) { free_null(h->d_rx[i]); free_null(h->d_rg[i]); }
    free_null(h->d_clx); free_null(h->d_clu); free_null(h->d_z); free_null(h->d_zpid); free_null(h->d_abc_lti);
    free_null(h->d_cllen); free_null(h->d_done); free_null(h->d_health);
    free_null(h->d_trinst); free_null(h->tr.steps); free_null(h->tr.x); free_null(h->tr.g); free_null(h->tr.u); free_null(h->tr.xPred);
    free_null(h->tr.ss); free_null(h->tr.lap);
    h->has_trace = false;
    h->has_rollout = false;
}

static void free_qp_bufs(QpBufs& q) {
    free_null(q.x0); free_null(q.uOld); free_null(q.abc); free_null(q.SS); free_null(q.Qfun); free_null(q.SuccSS); free_null(q.SuccU);
    free_null(q.xPred); free_null(q.uPred); free_null(q.slack); free_null(q.lambd); free_null(q.slackT); free_null(q.zt); free_null(q.ztu);
    free_null(q.resid); free_null(q.status); free_null(q.iters);
}

// Buffer set `slot` of the handle, allocated on first use (x0 != null: allocated); null (and g_err set) if the allocation failed,
// which leaves nothing behind
static QpBufs* qp_bufs(lmpc_handle* h, int slot) {
    QpBufs& q = h->hb[slot];
    if (!q.x0) {
        const size_t B = h->batch, N = h->N, M = h->M > 0 ? h->M : 1;
        cudaError_t e = cudaSuccess;
        auto alloc = [&](auto*& p, size_t count) { if (e == cudaSuccess) e = cudaMalloc((void**)&p, sizeof(*p) * count); };
        alloc(q.x0, B * 6); alloc(q.uOld, B * 2); alloc(q.abc, B * N * 54);
        alloc(q.SS, B * 6 * M); alloc(q.Qfun, B * M); alloc(q.SuccSS, B * 6 * M); alloc(q.SuccU, B * 2 * M);
        alloc(q.xPred, B * (N + 1) * 6); alloc(q.uPred, B * N * 2); alloc(q.slack, B * N * 2);
        alloc(q.lambd, B * M); alloc(q.slackT, B * 6); alloc(q.zt, B * 6); alloc(q.ztu, B * 2);
        alloc(q.resid, B * 3); alloc(q.status, B); alloc(q.iters, B);
        if (e != cudaSuccess) {
            free_qp_bufs(q);
            fail(LMPC_E_CUDA, std::string("cudaMalloc of QP buffer set ") + std::to_string(slot) + ": " + cudaGetErrorString(e));
            return nullptr;
        }
    }
    return &q;
}

// which of the QP kernel's optional inputs and outputs a caller wants (qp_args); the safe-set ones only count on LMPC-type QPs
enum : unsigned { QP_SUCC_SS = 1, QP_SUCC_U = 2, QP_SLACK = 4, QP_LAMBD = 8, QP_SLACKT = 16, QP_ZT = 32, QP_ZTU = 64, QP_ALL = 127 };

// Kernel arguments for the whole batch held in q (per-instance model, strides (N*54, 54)); what the caller does not want stays null,
// which the kernel skips
static FtocpArgs qp_args(const lmpc_handle* h, const QpBufs& q, bool lm, unsigned want) {
    if (!lm) want &= QP_SLACK;
    FtocpArgs a = {};
    a.batch = h->batch;
    a.x0 = q.x0; a.uOld = q.uOld; a.abc = q.abc;
    a.abc_inst_stride = (long long)h->N * 54; a.abc_stage_stride = 54;
    a.SS = lm ? q.SS : nullptr; a.Qfun = lm ? q.Qfun : nullptr;
    a.SuccSS = (want & QP_SUCC_SS) ? q.SuccSS : nullptr; a.SuccU = (want & QP_SUCC_U) ? q.SuccU : nullptr;
    a.xPred = q.xPred; a.uPred = q.uPred; a.slack = (want & QP_SLACK) ? q.slack : nullptr;
    a.lambd = (want & QP_LAMBD) ? q.lambd : nullptr; a.slackT = (want & QP_SLACKT) ? q.slackT : nullptr;
    a.zt = (want & QP_ZT) ? q.zt : nullptr; a.ztu = (want & QP_ZTU) ? q.ztu : nullptr;
    a.status = q.status; a.iters = q.iters; a.resid = q.resid;
    a.late = h->d_late;
    a.set_idx = h->d_set_idx;
    return a;
}

static int create_device_side(lmpc_handle* h) {
    CK(cudaSetDevice(h->device));
    int rc = configure(h->N, h->M > 0 ? h->M : 0);
    if (rc != LMPC_OK) return rc;
    CK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    for (int i = 0; i < 4 * LMPC_HOST_SLOTS; ++i) CK(cudaStreamCreateWithFlags(&h->cstream[i], cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    for (int i = 0; i < 4; ++i) CK(cudaEventCreateWithFlags(&h->ev_join[i], cudaEventDisableTiming));
    h->step_split = LMPC_STEP_SPLIT_DEFAULT;
    if (const char* e = getenv("LMPC_B200_STEP_SPLIT")) { const int v = atoi(e); if (v >= 1 && v <= 4) h->step_split = v; }   // tuning knob
    if (!qp_bufs(h, 0)) return LMPC_E_CUDA;
    CK(cudaMalloc((void**)&h->d_late, sizeof(unsigned long long)));
    CK(cudaMemset(h->d_late, 0, sizeof(unsigned long long)));
    const lmpc_vehicle_params ref = reference_vehicle();
    return swap_table(h, "lmpc_create", &ref, 1, nullptr, &h->d_veh, &h->d_veh_idx);
}

extern "C" {

const char* lmpc_last_error(void) { return g_err.c_str(); }

int lmpc_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

// ---- pinned host memory for the `_host` entry points ----------------------------------------------------------------------
// The `_host` entry points move 21.5 MB per configs[1] step over PCIe.  lmpc_host_alloc hands out blocks a single DMA stream
// reads at link rate: an anonymous mapping in whole 2 MiB units, placed on the NUMA node the GPU hangs
// off (mbind; raw syscalls, libnuma is not in the image), touched, then pinned with cudaHostRegister.
static int gpu_numa_node(int device) {
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, (int)sizeof(bus), device) != cudaSuccess) return -1;
    for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
    char path[96];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}
int lmpc_host_numa_node(int device) {
    const char* e = getenv("LMPC_B200_NUMA");      // "off" / "-1": no placement (A/B measurements); an integer >= 0 forces that node
    if (e && (!strcmp(e, "off") || !strcmp(e, "-1"))) return -1;
    if (e && isdigit((unsigned char)e[0]) && strcmp(e, "auto")) return atoi(e);
    return gpu_numa_node(device);
}
// Why a registered anonymous mapping rather than cudaHostAlloc: the driver allocates cudaHostAlloc / torch.pin_memory() pages
// itself, ignoring the caller's memory policy, and on some two-socket hosts a single DMA stream reads such buffers well below link
// rate (tools/numa_probe.py measures both allocators on a given host).  The node placement costs nothing and matters on hosts
// with a slow inter-socket link.
static std::mutex g_host_mu;
static std::map<void*, size_t> g_host_blocks;      // base -> mapped bytes
int lmpc_host_alloc(int device, size_t bytes, void** out) {
    if (!out || bytes == 0) return fail(LMPC_E_INVALID, "lmpc_host_alloc: null out or zero size");
    *out = nullptr;
    CK(cudaSetDevice(device));
    const size_t gran = 2u << 20;                                   // whole 2 MiB units (huge-page sized; MADV_HUGEPAGE is not requested)
    const size_t len = (bytes + gran - 1) / gran * gran;
    void* p = mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (p == MAP_FAILED) return fail(LMPC_E_CUDA, "lmpc_host_alloc: mmap failed");
    const int node = lmpc_host_numa_node(device);
#ifdef SYS_mbind
    if (node >= 0 && node < 1024) {
        unsigned long mask[1024 / (8 * sizeof(unsigned long))] = {0};
        mask[node / (8 * sizeof(unsigned long))] = 1UL << (node % (8 * sizeof(unsigned long)));
        // MPOL_PREFERRED (1): fall back to other nodes rather than fail when the node is short of memory; errors (seccomp,
        // cpuset without that node) leave the default policy in place
        (void)syscall(SYS_mbind, p, (unsigned long)len, 1, mask, 1024UL, 0U);
    }
#endif
    memset(p, 0, len);                                              // first touch: the pages exist (on the bound node) before they are pinned
    cudaError_t e = cudaHostRegister(p, len, cudaHostRegisterPortable);
    if (e != cudaSuccess) {
        munmap(p, len);
        return fail(LMPC_E_CUDA, std::string("cudaHostRegister: ") + cudaGetErrorString(e));
    }
    { std::lock_guard<std::mutex> g(g_host_mu); g_host_blocks[p] = len; }
    *out = p;
    return LMPC_OK;
}
int lmpc_host_free(void* p) {
    if (!p) return LMPC_OK;
    size_t len = 0;
    {
        std::lock_guard<std::mutex> g(g_host_mu);
        auto it = g_host_blocks.find(p);
        if (it == g_host_blocks.end()) return fail(LMPC_E_INVALID, "lmpc_host_free: not a block of lmpc_host_alloc");
        len = it->second;
        g_host_blocks.erase(it);
    }
    cudaError_t e = cudaHostUnregister(p);
    munmap(p, len);
    if (e != cudaSuccess) return fail(LMPC_E_CUDA, std::string("cudaHostUnregister: ") + cudaGetErrorString(e));
    return LMPC_OK;
}
/* NUMA node of up to n pages of a host block, sampled evenly (move_pages query): nodes_out[n]; diagnostics for the allocator. */
int lmpc_host_page_nodes(const void* p, size_t bytes, int n, int* nodes_out) {
    if (!p || !nodes_out || n <= 0 || n > 64) return fail(LMPC_E_INVALID, "lmpc_host_page_nodes: bad argument");
#ifdef SYS_move_pages
    void* pages[64];
    const size_t ps = 4096, np = bytes / ps > 0 ? bytes / ps : 1;
    for (int i = 0; i < n; ++i) pages[i] = (void*)(((uintptr_t)p & ~(uintptr_t)(ps - 1)) + (np * i / n) * ps);
    if (syscall(SYS_move_pages, 0, (unsigned long)n, pages, nullptr, nodes_out, 0) != 0) {
        if (errno != EPERM && errno != ENOSYS) return fail(LMPC_E_STATE, "move_pages query failed");
        for (int i = 0; i < n; ++i) nodes_out[i] = -1;             // the host forbids the query (e.g. a container's syscall filter)
    }
    return LMPC_OK;
#else
    return fail(LMPC_E_STATE, "move_pages is not available");
#endif
}

int lmpc_create(const lmpc_params* p, int batch, int device, lmpc_handle** out) {
    if (!p || !out || batch <= 0) return fail(LMPC_E_INVALID, "null argument or batch <= 0");
    if (p->ncx != 2 || p->ncu != 4)
        return fail(LMPC_E_INVALID, "this build supports ncx == 2 lane rows and ncu == 4 input rows (the reference's values)");
    FtocpConst c;
    int rc = build_const(*p, c);
    if (rc != LMPC_OK) return rc;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(LMPC_E_NODEVICE, "no CUDA device");
    if (device < 0 || device >= ndev) return fail(LMPC_E_INVALID, "bad device index");
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return fail(LMPC_E_NODEVICE, "liblmpc_b200 is built for sm_90a (H100) only");
    lmpc_handle* h = new (std::nothrow) lmpc_handle();
    if (!h) return fail(LMPC_E_INVALID, "out of host memory");
    memset(h, 0, sizeof(*h));
    h->p = *p;
    h->batch = batch;
    h->device = device;
    h->N = p->N;
    h->M = p->numSS_Points;
    h->c = c;
    rc = create_device_side(h);
    if (rc != LMPC_OK) {             // nothing of a half-built handle survives (zero-initialised: freeing what was never allocated is safe)
        const std::string msg = g_err;
        lmpc_destroy(h);
        g_err = msg;
        return rc;
    }
    *out = h;
    return LMPC_OK;
}

int lmpc_destroy(lmpc_handle* h) {
    if (!h) return LMPC_OK;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    for (int i = 0; i < 4 * LMPC_HOST_SLOTS; ++i) if (h->cstream[i]) cudaStreamSynchronize(h->cstream[i]);
    // every pointer freed here is either a live allocation or still null (handle memory is zero-initialised)
    free_rollout(h);
    free_store(h);
    for (QpBufs& q : h->hb) free_qp_bufs(q);
    cudaFree(h->d_late);
    cudaFree(h->d_sets);
    cudaFree(h->d_set_idx);
    cudaFree(h->d_veh);
    cudaFree(h->d_veh_idx);
    if (h->stream) cudaStreamDestroy(h->stream);
    for (int i = 0; i < 4 * LMPC_HOST_SLOTS; ++i) if (h->cstream[i]) cudaStreamDestroy(h->cstream[i]);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    for (int i = 0; i < 4; ++i) if (h->ev_join[i]) cudaEventDestroy(h->ev_join[i]);
    delete h;
    return LMPC_OK;
}

int lmpc_sync(lmpc_handle* h) {
    if (!h) return fail(LMPC_E_INVALID, "null handle");
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

void* lmpc_stream(lmpc_handle* h) { return h ? (void*)h->stream : nullptr; }

long long lmpc_late_accepts(lmpc_handle* h) {
    if (!h) return -1;
    if (cudaSetDevice(h->device) != cudaSuccess) return -1;
    unsigned long long v = 0;
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) return -1;
    for (int i = 0; i < 4 * LMPC_HOST_SLOTS; ++i) if (cudaStreamSynchronize(h->cstream[i]) != cudaSuccess) return -1;
    if (cudaMemcpy(&v, h->d_late, sizeof(v), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    return (long long)v;
}
long long lmpc_kernel_launches(lmpc_handle* h) { return h ? h->launches : 0; }

// Per-controller parameters: every set goes through build_const (the conversion lmpc_create uses), then the table replaces the
// previous one once the handle's streams are idle.  Nothing about the handle changes unless every check passes.
int lmpc_set_param_sets(lmpc_handle* h, const lmpc_params* sets, int nsets, const int* set_of_instance) {
    if (!h) return fail(LMPC_E_INVALID, "null handle");
    int rc = check_set_index(h, "lmpc_set_param_sets", sets, nsets, set_of_instance);
    if (rc != LMPC_OK) return rc;
    std::vector<FtocpConstRec> rows(nsets);
    for (int k = 0; k < nsets; ++k) {
        const lmpc_params& s = sets[k];
        if (s.N != h->p.N || s.ncx != h->p.ncx || s.ncu != h->p.ncu || s.numSS_Points != h->p.numSS_Points ||
            s.numSS_it != h->p.numSS_it || s.warm_start != h->p.warm_start)
            return fail(LMPC_E_INVALID, "lmpc_set_param_sets: set " + std::to_string(k) +
                                            " differs from the handle in N, ncx, ncu, numSS_Points, numSS_it or warm_start");
        rc = build_const(s, rows[k].c);
        if (rc != LMPC_OK) return fail(rc, "lmpc_set_param_sets: set " + std::to_string(k) + ": " + g_err);
    }
    if ((rc = swap_table(h, "lmpc_set_param_sets", rows.data(), nsets, set_of_instance, &h->d_sets, &h->d_set_idx)) != LMPC_OK) return rc;
    // a warm-start record belongs to the QP it was taken from
    if (h->d_warm_valid) {
        CK(cudaMemsetAsync(h->d_warm_valid, 0, sizeof(int) * h->batch, h->stream));
        CK(cudaStreamSynchronize(h->stream));
    }
    return LMPC_OK;
}

static int check_align(const void* p, const char* what) {
    if (((uintptr_t)p) & 15) return fail(LMPC_E_INVALID, std::string(what) + " must be 16-byte aligned");
    return LMPC_OK;
}

int lmpc_solve_lmpc_dev(lmpc_handle* h, const double* x0, const double* uOld, const double* abc, long long abc_inst_stride,
                        long long abc_stage_stride, const double* SS_sel, const double* Qfun_sel, const double* Succ_SS,
                        const double* Succ_uSS, double* xPred, double* uPred, double* slack, double* lambd,
                        double* slackTerminal, double* zt, double* zt_u, int* status, int* iters, double* resid) {
    if (!h || !x0 || !uOld || !abc || !xPred || !uPred || !status || !iters || !resid) return fail(LMPC_E_INVALID, "null argument");
    const bool lm = (SS_sel != nullptr);
    if (lm && (h->M <= 0 || !Qfun_sel)) return fail(LMPC_E_INVALID, "handle was created without a safe set (numSS_Points == 0)");
    if ((abc_inst_stride % 2) || (abc_stage_stride % 2)) return fail(LMPC_E_INVALID, "abc strides must be even (16-byte rows)");
    int rc;
    if ((rc = check_align(abc, "abc")) != LMPC_OK) return rc;
    if (lm && ((rc = check_align(SS_sel, "SS_sel")) != LMPC_OK || (rc = check_align(Qfun_sel, "Qfun_sel")) != LMPC_OK)) return rc;
    CK(cudaSetDevice(h->device));
    FtocpArgs a = {};   // no warm-start records: caller-supplied QPs start cold; the controllers of the device-resident step
                        // carry warm-start records (step_range)
    a.batch = h->batch;
    a.x0 = x0; a.uOld = uOld; a.abc = abc;
    a.abc_inst_stride = abc_inst_stride; a.abc_stage_stride = abc_stage_stride;
    a.SS = SS_sel; a.Qfun = Qfun_sel; a.SuccSS = Succ_SS; a.SuccU = Succ_uSS;
    a.xPred = xPred; a.uPred = uPred; a.slack = slack; a.lambd = lambd; a.slackT = slackTerminal;
    a.zt = zt; a.ztu = zt_u; a.status = status; a.iters = iters; a.resid = resid;
    a.late = h->d_late;
    a.set_idx = h->d_set_idx;
    return launch(h, a, lm, h->stream);
}

int lmpc_solve_mpc_dev(lmpc_handle* h, const double* x0, const double* uOld, const double* abc, long long abc_inst_stride,
                       long long abc_stage_stride, double* xPred, double* uPred, double* slack, int* status, int* iters,
                       double* resid) {
    return lmpc_solve_lmpc_dev(h, x0, uOld, abc, abc_inst_stride, abc_stage_stride, nullptr, nullptr, nullptr, nullptr, xPred,
                               uPred, slack, nullptr, nullptr, nullptr, nullptr, status, iters, resid);
}

// Enqueue one host-buffer solve on buffer set / stream group `slot` (0 .. LMPC_HOST_SLOTS - 1) WITHOUT waiting for it.
static int enqueue_host_solve_impl(lmpc_handle* h, int slot, const double* x0, const double* uOld, const double* abc,
                              long long abc_inst_stride, long long abc_stage_stride, const double* SS_sel, const double* Qfun_sel,
                              const double* Succ_SS, const double* Succ_uSS, double* xPred, double* uPred, double* slack,
                              double* lambd, double* slackTerminal, double* zt, double* zt_u, int* status, int* iters,
                              double* resid) {
    if (!h || !x0 || !uOld || !abc || !xPred || !uPred || !status || !iters || !resid) return fail(LMPC_E_INVALID, "null argument");
    const bool lm = (SS_sel != nullptr);
    if (lm && (h->M <= 0 || !Qfun_sel)) return fail(LMPC_E_INVALID, "handle was created without a safe set (numSS_Points == 0)");
    if (slot < 0 || slot >= LMPC_HOST_SLOTS) return fail(LMPC_E_INVALID, "slot must be 0 .. 3");
    CK(cudaSetDevice(h->device));
    const size_t B = h->batch, N = h->N, M = h->M > 0 ? h->M : 1;
    const size_t D = sizeof(double);
    const QpBufs* q = qp_bufs(h, slot);
    if (!q) return LMPC_E_CUDA;
    const QpBufs& hb = *q;
    cudaStream_t* cs = h->cstream + 4 * slot;
    long long dis, dss;
    bool per_inst = false;
    if (abc_inst_stride == 0 && abc_stage_stride == 0) { dis = 0; dss = 0; }                       // one shared LTI model
    else if (abc_inst_stride == (long long)N * 54 && abc_stage_stride == 54) { dis = N * 54; dss = 54; per_inst = true; }
    else if (abc_inst_stride == 0 && abc_stage_stride == 54) { dis = 0; dss = 54; }                // one shared LTV model
    else return fail(LMPC_E_INVALID, "host entry supports abc strides (N*54,54), (0,54) or (0,0)");
    CK(cudaStreamSynchronize(h->stream));    // earlier work of this handle is done before the chunk streams start
    if (!per_inst) {
        CK(cudaMemcpyAsync(hb.abc, abc, (dss ? N * 54 : 54) * D, cudaMemcpyHostToDevice, cs[0]));
        CK(cudaStreamSynchronize(cs[0]));
    }
    // Chunk pipeline: the batch is cut into up to four instance ranges, each on its own stream, so that the H2D copy
    // of range i+1, the solve of range i and the D2H copy of range i-1 overlap (PCIe is full duplex).
    // A batch enqueued through the asynchronous entry points shares the device with the batches of the other buffer sets: that
    // overlap is already there, every further piece is ten more driver calls on the enqueueing thread and one more under-filled
    // last wave.  Measured on configs[1] (4096 QPs, three sets in flight, tools/e2e_probe.py, two hosts): 8.8-9.6 M solves/s uncut,
    // 8.7-9.6 M in two pieces, 8.2-8.6 M in four; a lone synchronous batch: 3.1 M uncut, 3.7 M in two, 3.9 M in four.
    bool others = false;
    for (int sl = 0; sl < LMPC_HOST_SLOTS; ++sl) others |= (sl != slot && h->hb_pending[sl]);
    const bool lone = h->hb_lone && !others;
    int nchunk = B >= 2048 ? (lone ? 4 : (others ? 1 : 2)) : (B >= 512 ? (others ? 1 : 2) : 1);
    if (const char* e = getenv("LMPC_B200_CHUNKS")) { int v = atoi(e); if (v >= 1 && v <= 4 && (size_t)v <= B) nchunk = v; }   // tuning knob
    const bool trace = slot == 0 && getenv("LMPC_B200_TRACE") != nullptr;
    if (trace) {
        cudaEventCreate(&h->t0ev);
        for (int i = 0; i < nchunk; ++i) for (int j = 0; j < 3; ++j) cudaEventCreate(&h->tev[i][j]);
        cudaEventRecord(h->t0ev, cs[0]);
    }
    h->trace_on = trace;
    FtocpArgs all = qp_args(h, hb, lm, (Succ_SS ? QP_SUCC_SS : 0) | (Succ_uSS ? QP_SUCC_U : 0) | (slack ? QP_SLACK : 0) |
                                       (lambd ? QP_LAMBD : 0) | (slackTerminal ? QP_SLACKT : 0) | (zt ? QP_ZT : 0) |
                                       (zt_u ? QP_ZTU : 0));
    all.abc_inst_stride = dis; all.abc_stage_stride = dss;
    for (int ci = 0; ci < nchunk; ++ci) {
        const size_t lo = B * ci / nchunk, hi = B * (ci + 1) / nchunk, nb = hi - lo;
        cudaStream_t s = cs[ci];
        CK(cudaMemcpyAsync(hb.x0 + lo * 6, x0 + lo * 6, nb * 6 * D, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(hb.uOld + lo * 2, uOld + lo * 2, nb * 2 * D, cudaMemcpyHostToDevice, s));
        if (per_inst) CK(cudaMemcpyAsync(hb.abc + lo * N * 54, abc + lo * N * 54, nb * N * 54 * D, cudaMemcpyHostToDevice, s));
        if (lm) {
            CK(cudaMemcpyAsync(hb.SS + lo * 6 * M, SS_sel + lo * 6 * M, nb * 6 * M * D, cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(hb.Qfun + lo * M, Qfun_sel + lo * M, nb * M * D, cudaMemcpyHostToDevice, s));
            if (Succ_SS) CK(cudaMemcpyAsync(hb.SuccSS + lo * 6 * M, Succ_SS + lo * 6 * M, nb * 6 * M * D, cudaMemcpyHostToDevice, s));
            if (Succ_uSS) CK(cudaMemcpyAsync(hb.SuccU + lo * 2 * M, Succ_uSS + lo * 2 * M, nb * 2 * M * D, cudaMemcpyHostToDevice, s));
        }
        if (trace) cudaEventRecord(h->tev[ci][0], s);
        int rc = launch(h, all.range((int)lo, (int)nb, (int)N, h->M), lm, s);
        if (rc != LMPC_OK) return rc;
        if (trace) cudaEventRecord(h->tev[ci][1], s);
        CK(cudaMemcpyAsync(xPred + lo * (N + 1) * 6, hb.xPred + lo * (N + 1) * 6, nb * (N + 1) * 6 * D, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(uPred + lo * N * 2, hb.uPred + lo * N * 2, nb * N * 2 * D, cudaMemcpyDeviceToHost, s));
        if (slack) CK(cudaMemcpyAsync(slack + lo * N * 2, hb.slack + lo * N * 2, nb * N * 2 * D, cudaMemcpyDeviceToHost, s));
        if (lm && lambd) CK(cudaMemcpyAsync(lambd + lo * M, hb.lambd + lo * M, nb * M * D, cudaMemcpyDeviceToHost, s));
        if (lm && slackTerminal) CK(cudaMemcpyAsync(slackTerminal + lo * 6, hb.slackT + lo * 6, nb * 6 * D, cudaMemcpyDeviceToHost, s));
        if (lm && zt && Succ_SS) CK(cudaMemcpyAsync(zt + lo * 6, hb.zt + lo * 6, nb * 6 * D, cudaMemcpyDeviceToHost, s));
        if (lm && zt_u && Succ_uSS) CK(cudaMemcpyAsync(zt_u + lo * 2, hb.ztu + lo * 2, nb * 2 * D, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(status + lo, hb.status + lo, nb * sizeof(int), cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(iters + lo, hb.iters + lo, nb * sizeof(int), cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(resid + lo * 3, hb.resid + lo * 3, nb * 3 * D, cudaMemcpyDeviceToHost, s));
        if (trace) cudaEventRecord(h->tev[ci][2], s);
    }
    h->hb_chunks[slot] = nchunk;
    h->hb_pending[slot] = true;
    return LMPC_OK;
}


// Enqueue one host-buffer solve; on ANY failure part-way through, the chunks already enqueued are still copying into the
// caller's arrays, so their streams are drained before the error is reported.
static int enqueue_host_solve(lmpc_handle* h, int slot, const double* x0, const double* uOld, const double* abc,
                              long long abc_inst_stride, long long abc_stage_stride, const double* SS_sel, const double* Qfun_sel,
                              const double* Succ_SS, const double* Succ_uSS, double* xPred, double* uPred, double* slack,
                              double* lambd, double* slackTerminal, double* zt, double* zt_u, int* status, int* iters,
                              double* resid) {
    const int rc = enqueue_host_solve_impl(h, slot, x0, uOld, abc, abc_inst_stride, abc_stage_stride, SS_sel, Qfun_sel, Succ_SS, Succ_uSS,
                                           xPred, uPred, slack, lambd, slackTerminal, zt, zt_u, status, iters, resid);
    if (rc != LMPC_OK && h && slot >= 0 && slot < LMPC_HOST_SLOTS) {
        const std::string msg = g_err;
        for (int i = 0; i < 4; ++i) cudaStreamSynchronize(h->cstream[4 * slot + i]);
        g_err = msg;
    }
    return rc;
}


/* Instance ranges the most recent enqueue on `slot` was cut into (diagnostics of the chunk policy); -1 on a bad argument. */
int lmpc_host_chunks(lmpc_handle* h, int slot) {
    if (!h || slot < 0 || slot >= LMPC_HOST_SLOTS) return -1;
    return h->hb_chunks[slot];
}

int lmpc_host_wait(lmpc_handle* h, int slot) {
    if (!h || slot < 0 || slot >= LMPC_HOST_SLOTS) return fail(LMPC_E_INVALID, "bad handle or slot");
    CK(cudaSetDevice(h->device));
    const int nchunk = h->hb_chunks[slot] > 0 ? h->hb_chunks[slot] : 4;
    for (int ci = 0; ci < nchunk; ++ci) CK(cudaStreamSynchronize(h->cstream[4 * slot + ci]));
    h->hb_pending[slot] = false;
    if (slot == 0 && h->trace_on) {
        for (int i = 0; i < nchunk; ++i) {
            float a_ = 0, b_ = 0, c_ = 0;
            cudaEventElapsedTime(&a_, h->t0ev, h->tev[i][0]); cudaEventElapsedTime(&b_, h->t0ev, h->tev[i][1]); cudaEventElapsedTime(&c_, h->t0ev, h->tev[i][2]);
            fprintf(stderr, "chunk %d: h2d done %.3f ms, kernel done %.3f, d2h done %.3f\n", i, a_, b_, c_);
            for (int j = 0; j < 3; ++j) cudaEventDestroy(h->tev[i][j]);
        }
        cudaEventDestroy(h->t0ev);
        h->trace_on = false;
    }
    return LMPC_OK;
}

int lmpc_solve_lmpc_host_async(lmpc_handle* h, int slot, const double* x0, const double* uOld, const double* abc, long long abc_inst_stride,
                               long long abc_stage_stride, const double* SS_sel, const double* Qfun_sel, const double* Succ_SS,
                               const double* Succ_uSS, double* xPred, double* uPred, double* slack, double* lambd,
                               double* slackTerminal, double* zt, double* zt_u, int* status, int* iters, double* resid) {
    return enqueue_host_solve(h, slot, x0, uOld, abc, abc_inst_stride, abc_stage_stride, SS_sel, Qfun_sel, Succ_SS, Succ_uSS, xPred, uPred,
                              slack, lambd, slackTerminal, zt, zt_u, status, iters, resid);
}

int lmpc_solve_mpc_host_async(lmpc_handle* h, int slot, const double* x0, const double* uOld, const double* abc, long long abc_inst_stride,
                              long long abc_stage_stride, double* xPred, double* uPred, double* slack, int* status, int* iters,
                              double* resid) {
    return enqueue_host_solve(h, slot, x0, uOld, abc, abc_inst_stride, abc_stage_stride, nullptr, nullptr, nullptr, nullptr, xPred, uPred,
                              slack, nullptr, nullptr, nullptr, nullptr, status, iters, resid);
}

int lmpc_solve_lmpc_host(lmpc_handle* h, const double* x0, const double* uOld, const double* abc, long long abc_inst_stride,
                         long long abc_stage_stride, const double* SS_sel, const double* Qfun_sel, const double* Succ_SS,
                         const double* Succ_uSS, double* xPred, double* uPred, double* slack, double* lambd,
                         double* slackTerminal, double* zt, double* zt_u, int* status, int* iters, double* resid) {
    if (h) h->hb_lone = true;
    int rc = enqueue_host_solve(h, 0, x0, uOld, abc, abc_inst_stride, abc_stage_stride, SS_sel, Qfun_sel, Succ_SS, Succ_uSS, xPred, uPred,
                                slack, lambd, slackTerminal, zt, zt_u, status, iters, resid);
    if (h) h->hb_lone = false;
    if (rc) return rc;
    return lmpc_host_wait(h, 0);
}

int lmpc_solve_mpc_host(lmpc_handle* h, const double* x0, const double* uOld, const double* abc, long long abc_inst_stride,
                        long long abc_stage_stride, double* xPred, double* uPred, double* slack, int* status, int* iters,
                        double* resid) {
    return lmpc_solve_lmpc_host(h, x0, uOld, abc, abc_inst_stride, abc_stage_stride, nullptr, nullptr, nullptr, nullptr, xPred,
                                uPred, slack, nullptr, nullptr, nullptr, nullptr, status, iters, resid);
}

// ================================================================================================
// lap stores, state, K1/K2/K6, fused step
// ================================================================================================
int lmpc_sizeof_params(void) { return (int)sizeof(lmpc_params); }
int lmpc_sizeof_model_params(void) { return (int)sizeof(lmpc_model_params); }
int lmpc_sizeof_vehicle_params(void) { return (int)sizeof(lmpc_vehicle_params); }
int lmpc_sizeof_track_params(void) { return (int)sizeof(lmpc_track_params); }

static int store_create_impl(lmpc_handle* h, const lmpc_model_params* mp, int ss_cap, int model_cap, int Tmax);
int lmpc_store_create(lmpc_handle* h, const lmpc_model_params* mp, int ss_cap, int model_cap, int Tmax) {
    const int rc = store_create_impl(h, mp, ss_cap, model_cap, Tmax);
    if (rc != LMPC_OK && h && !h->has_store) { const std::string msg = g_err; free_store(h); g_err = msg; }   // no partial store
    return rc;
}
}  // extern "C" (the helper below has C++ linkage)
static int store_create_impl(lmpc_handle* h, const lmpc_model_params* mp, int ss_cap, int model_cap, int Tmax) {
    if (!h || !mp || ss_cap < 0 || model_cap <= 0 || Tmax < 16) return fail(LMPC_E_INVALID, "bad store arguments");
    if (Tmax > (32 << K1_JBITS)) return fail(LMPC_E_INVALID, "Tmax above 4096 rows per lap is not supported by the neighbour scan");
    if (h->has_store) return fail(LMPC_E_STATE, "store already created");
    if (mp->trToUse < 1 || mp->trToUse > K1_MAXLAPS || mp->trToUse > model_cap) return fail(LMPC_E_INVALID, "trToUse out of range");
    if (mp->MaxNumPoint < 1 || mp->MaxNumPoint > K1_MAXPTS) return fail(LMPC_E_INVALID, "MaxNumPoint must be <= 7");
    if (mp->nseg < 1 || mp->nseg > 16) return fail(LMPC_E_INVALID, "track table has 1..16 segments");
    if (h->M > 0) {
        if (h->p.numSS_it < 1 || h->p.numSS_it > 8 || h->M % h->p.numSS_it) return fail(LMPC_E_INVALID, "numSS_Points must be a multiple of numSS_it <= 8");
        if (((h->M / h->p.numSS_it) % 2) != 0) return fail(LMPC_E_INVALID, "numSS_Points/numSS_it must be even (PC.py:403,492-495)");
        if (ss_cap < h->p.numSS_it) return fail(LMPC_E_INVALID, "ss_cap < numSS_it");
    }
    CK(cudaSetDevice(h->device));
    CK(cudaFuncSetAttribute(knn_ltv_regress_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    CK(cudaFuncSetAttribute(knn_ltv_regress_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    ModelConst& m = h->mc;
    memset(&m, 0, sizeof(m));
    m.trToUse = mp->trToUse; m.MaxNumPoint = mp->MaxNumPoint; m.h = mp->h; m.lamb = mp->lamb; m.dt = mp->dt;
    for (int i = 0; i < 5; ++i) m.scaling[i] = mp->scaling[i];
    TrackRec& t = h->store_trk;
    memset(&t, 0, sizeof(t));
    t.nseg = mp->nseg;
    for (int i = 0; i < mp->nseg * 3; ++i) t.seg[i] = mp->seg[i];
    t.TrackLength = mp->TrackLength;
    int rc = swap_table(h, "lmpc_store_create", &t, 1, nullptr, &h->d_trk, &h->d_trk_idx);
    if (rc != LMPC_OK) return rc;
    h->trk_host.assign(1, t);
    h->trk_idx_host.clear();
    h->laps_stored = false;
    const size_t B = h->batch, N = h->N;
    h->ss.cap = ss_cap > 0 ? ss_cap : 1; h->ss.Tmax = Tmax;
    h->mdl.cap = model_cap; h->mdl.Tmax = Tmax;
#define DA(ptr, T, count) CK(cudaMalloc((void**)&(ptr), sizeof(T) * (count)))
#define DA2(ptr, T, count) CK(cudaMalloc((void**)&(ptr), sizeof(T) * (count)))
    DA(h->ss.x, double, B * h->ss.cap * Tmax * 6); DA(h->ss.u, double, B * h->ss.cap * Tmax * 2); DA(h->ss.q, double, B * h->ss.cap * Tmax);
    DA(h->ss.len, int, B * h->ss.cap);
    DA(h->mdl.x, double, B * model_cap * Tmax * 6); DA(h->mdl.u, double, B * model_cap * Tmax * 2); h->mdl.q = nullptr;
    DA(h->mdl.len, int, B * model_cap);
    DA(h->d_used, int, B * K1_MAXLAPS); DA(h->d_sel, int, B * 8); DA(h->d_isprev, int, B * 8); DA(h->d_prevslot, int, B);
    DA(h->d_timeStep, int, B); DA(h->d_hasPred, int, B); DA(h->d_flags, int, B); DA(h->d_minidx, int, B * 8);
    DA(h->d_xLin, double, B * (N + 1) * 6); DA(h->d_uLin, double, B * N * 2); DA(h->d_ztState, double, B * 6);
    DA(h->d_ztFixed, double, B * 6); DA(h->d_OldInput, double, B * 2); DA(h->d_xPredPrev, double, B * (N + 1) * 6);
    DA(h->d_tmpx, double, B * 6); DA(h->d_tmpu, double, B * 2); DA(h->d_xchg, int, B * 3); DA(h->d_dropped, int, 1);
#undef DA
    CK(cudaMemsetAsync(h->d_dropped, 0, sizeof(int), h->stream));
    if (h->p.warm_start) {          // SURVEY §8f rank 2: per-controller interior-point snapshot for the next solve
        const size_t Mx = h->M > 0 ? h->M : 0;
        h->warm_stride = (long long)(N * 2 + 4 * N * h->p.ncx + N * h->p.ncu + 2 * Mx + 2);
        DA2(h->d_warm, double, B * (size_t)h->warm_stride);
        DA2(h->d_warm_valid, int, B);
        CK(cudaMemsetAsync(h->d_warm_valid, 0, sizeof(int) * B, h->stream));
        h->warm_mode = -1;
    }
    {   // device lap books: one int buffer carved into the slot tables
        const size_t sc = h->ss.cap, mcp = model_cap;
        const size_t n = B * (2 * sc + 1 + 2 * mcp + 1 + LAP_HIST + 1);
        DA2(h->d_bkbuf, int, n);
        int* p = h->d_bkbuf;
        LapBooks& k = h->bk;
        k.ss_time = p; p += B * sc; k.ss_lap = p; p += B * sc; k.it = p; p += B;
        k.md_time = p; p += B * mcp; k.md_seq = p; p += B * mcp; k.md_cnt = p; p += B;
        k.lap_hist = p; p += B * LAP_HIST; k.lap_n = p; p += B;
        k.sel = h->d_sel; k.isprev = h->d_isprev; k.prevslot = h->d_prevslot; k.used = h->d_used;
        k.ss_cap = (int)sc; k.md_cap = (int)mcp; k.numSS_it = h->p.numSS_it > 0 ? h->p.numSS_it : 1; k.trToUse = mp->trToUse;
        CK(cudaMemsetAsync(h->d_bkbuf, 0xff, sizeof(int) * n, h->stream));          // every slot free (-1)
        CK(cudaMemsetAsync(k.it, 0, sizeof(int) * B, h->stream));
        CK(cudaMemsetAsync(k.md_cnt, 0, sizeof(int) * B, h->stream));
        CK(cudaMemsetAsync(k.lap_n, 0, sizeof(int) * B, h->stream));
        DA2(h->d_poolidx, int, 256);
        DA2(h->d_stats, int, 8);
        h->has_books = true;
    }
    CK(cudaMemsetAsync(h->ss.len, 0, sizeof(int) * B * h->ss.cap, h->stream));
    CK(cudaMemsetAsync(h->mdl.len, 0, sizeof(int) * B * model_cap, h->stream));
    CK(cudaMemsetAsync(h->d_used, 0, sizeof(int) * B * K1_MAXLAPS, h->stream));
    CK(cudaMemsetAsync(h->d_sel, 0, sizeof(int) * B * 8, h->stream));
    CK(cudaMemsetAsync(h->d_isprev, 0, sizeof(int) * B * 8, h->stream));
    CK(cudaMemsetAsync(h->d_prevslot, 0xff, sizeof(int) * B, h->stream));
    CK(cudaMemsetAsync(h->d_timeStep, 0, sizeof(int) * B, h->stream));
    CK(cudaMemsetAsync(h->d_hasPred, 0, sizeof(int) * B, h->stream));
    CK(cudaMemsetAsync(h->d_flags, 0, sizeof(int) * B, h->stream));
    CK(cudaMemsetAsync(h->d_OldInput, 0, sizeof(double) * B * 2, h->stream));
    CK(cudaMemsetAsync(h->d_ztState, 0, sizeof(double) * B * 6, h->stream));
    CK(cudaMemsetAsync(h->d_xPredPrev, 0, sizeof(double) * B * (N + 1) * 6, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    h->has_store = true;
    return LMPC_OK;
}
extern "C" {

static int need_store(lmpc_handle* h) {
    if (!h) return fail(LMPC_E_INVALID, "null handle");
    if (!h->has_store) return fail(LMPC_E_STATE, "call lmpc_store_create first");
    return LMPC_OK;
}

// The pooled exchange hands laps between controllers: only when they all drive one circuit
static int one_track(const lmpc_handle* h, const char* who) {
    if (h->trk_host.size() > 1)
        return fail(LMPC_E_STATE, std::string(who) + ": more than one track installed; a lap of another circuit is not a trajectory of this one");
    return LMPC_OK;
}

// Per-controller tracks: every set is checked the way Track.py:54-133 builds the table (start i = start i-1 + length i-1 and
// TrackLength = start + length of the last row, exactly), then the table replaces the previous one once the handle's streams are
// idle.  Nothing about the handle changes unless every check passes.
int lmpc_set_tracks(lmpc_handle* h, const lmpc_track_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_set_tracks";
    int rc = need_store(h);
    if (rc) return rc;
    if (h->laps_stored) return fail(LMPC_E_STATE, std::string(who) + ": laps are stored already; install tracks before the first lap");
    if ((rc = check_set_index(h, who, sets, nsets, set_of_instance)) != LMPC_OK) return rc;
    for (int k = 0; k < nsets; ++k) {
        const lmpc_track_params& t = sets[k];
        const std::string w = std::string(who) + ": track " + std::to_string(k) + ": ";
        if (t.nseg < 1 || t.nseg > LMPC_MAX_SEG) return fail(LMPC_E_INVALID, w + "nseg must be 1 .. 16");
        bool finite = isfinite(t.TrackLength);
        for (int i = 0; i < t.nseg * 3; ++i) finite = finite && isfinite(t.seg[i]);
        if (!finite) return fail(LMPC_E_INVALID, w + "every value must be finite");
        if (t.seg[0] != 0.0) return fail(LMPC_E_INVALID, w + "the first segment must start at s = 0");
        for (int i = 0; i < t.nseg; ++i) {
            if (t.seg[i * 3 + 1] < 0.0) return fail(LMPC_E_INVALID, w + "segment " + std::to_string(i) + " has a negative length");
            if (i > 0 && t.seg[i * 3] != t.seg[(i - 1) * 3] + t.seg[(i - 1) * 3 + 1])
                return fail(LMPC_E_INVALID, w + "segment " + std::to_string(i) + " does not start where the previous one ends");
        }
        const int l = (t.nseg - 1) * 3;
        if (!(t.TrackLength > 0.0) || t.TrackLength != t.seg[l] + t.seg[l + 1])
            return fail(LMPC_E_INVALID, w + "TrackLength must be positive and equal the end of the last segment");
    }
    std::vector<TrackRec> rows;
    if (nsets == 0) rows.push_back(h->store_trk);
    else rows.assign(sets, sets + nsets);
    if ((rc = swap_table(h, who, rows.data(), (int)rows.size(), set_of_instance, &h->d_trk, &h->d_trk_idx)) != LMPC_OK) return rc;
    h->trk_host = rows;
    if (set_of_instance) h->trk_idx_host.assign(set_of_instance, set_of_instance + h->batch);
    else h->trk_idx_host.clear();
    return LMPC_OK;
}

static int put_lap(lmpc_handle* h, LapPool& pool, int inst, int slot, int T, const double* x, const double* u) {
    if (inst < 0 || inst >= h->batch || slot < 0 || slot >= pool.cap || T < 2 || T > pool.Tmax || !x || !u)
        return fail(LMPC_E_INVALID, "put_lap: bad instance/slot/length");
    CK(cudaSetDevice(h->device));
    h->laps_stored = true;
    const size_t lap = pool.lap_index(inst, slot);
    CK(cudaMemcpyAsync(pool.x + lap * pool.Tmax * 6, x, sizeof(double) * T * 6, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(pool.u + lap * pool.Tmax * 2, u, sizeof(double) * T * 2, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(pool.len + lap, &T, sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));   // T lives on the caller's stack
    return LMPC_OK;
}

int lmpc_model_put_lap(lmpc_handle* h, int inst, int slot, int T, const double* x, const double* u) {
    int rc = need_store(h);
    if (rc) return rc;
    return put_lap(h, h->mdl, inst, slot, T, x, u);
}

int lmpc_model_set_used(lmpc_handle* h, const int* slots) {
    int rc = need_store(h);
    if (rc) return rc;
    if (!slots) return fail(LMPC_E_INVALID, "null slots");
    for (size_t i = 0; i < (size_t)h->batch * h->mc.trToUse; ++i)
        if (slots[i] < 0 || slots[i] >= h->mdl.cap) return fail(LMPC_E_INVALID, "model slot out of range");
    CK(cudaSetDevice(h->device));
    CK(cudaMemcpyAsync(h->d_used, slots, sizeof(int) * h->batch * h->mc.trToUse, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_ss_put_lap(lmpc_handle* h, int inst, int slot, int T, const double* x, const double* u, const double* qfun) {
    int rc = need_store(h);
    if (rc) return rc;
    rc = put_lap(h, h->ss, inst, slot, T, x, u);
    if (rc) return rc;
    const size_t lap = h->ss.lap_index(inst, slot);
    if (qfun) {
        CK(cudaMemcpyAsync(h->ss.q + lap * h->ss.Tmax, qfun, sizeof(double) * T, cudaMemcpyHostToDevice, h->stream));
    } else {
        rollout_cost_kernel<<<1, 256, 0, h->stream>>>(h->ss, inst, slot, tracks(h));
        CK(cudaGetLastError());
        h->launches += 1;
    }
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_ss_set_selection(lmpc_handle* h, const int* slots, const int* is_prev, const int* prev_slot) {
    int rc = need_store(h);
    if (rc) return rc;
    if (!slots || !is_prev || !prev_slot) return fail(LMPC_E_INVALID, "null argument");
    const int nit = h->p.numSS_it;
    for (size_t i = 0; i < (size_t)h->batch * nit; ++i)
        if (slots[i] < 0 || slots[i] >= h->ss.cap) return fail(LMPC_E_INVALID, "safe-set slot out of range");
    for (int b = 0; b < h->batch; ++b)
        if (prev_slot[b] >= h->ss.cap) return fail(LMPC_E_INVALID, "prev_slot out of range");
    CK(cudaSetDevice(h->device));
    CK(cudaMemcpyAsync(h->d_sel, slots, sizeof(int) * h->batch * nit, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_isprev, is_prev, sizeof(int) * h->batch * nit, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_prevslot, prev_slot, sizeof(int) * h->batch, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_ss_add_point(lmpc_handle* h, const double* x, const double* u) {
    int rc = need_store(h);
    if (rc) return rc;
    if (!x || !u) return fail(LMPC_E_INVALID, "null argument");
    CK(cudaSetDevice(h->device));
    CK(cudaMemcpyAsync(h->d_tmpx, x, sizeof(double) * h->batch * 6, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_tmpu, u, sizeof(double) * h->batch * 2, cudaMemcpyHostToDevice, h->stream));
    ss_add_point_kernel<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(h->batch, h->ss, h->d_prevslot, h->d_tmpx, h->d_tmpu, 2,
                                                                        tracks(h), h->d_flags, h->d_dropped, 0);
    CK(cudaGetLastError());
    h->launches += 1;
    int dropped = 0;
    CK(cudaMemcpyAsync(&dropped, h->d_dropped, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (dropped) {      // the reference's lists grow without bound (PC.py:466-476); a full slot must not pass silently
        CK(cudaMemsetAsync(h->d_dropped, 0, sizeof(int), h->stream));
        return fail(LMPC_E_STATE, "addPoint: " + std::to_string(dropped) + " safe-set lap(s) reached Tmax rows; create the store with a larger Tmax");
    }
    return LMPC_OK;
}

int lmpc_ss_get_lap(lmpc_handle* h, int inst, int slot, int* T, double* x, double* u, double* qfun) {
    int rc = need_store(h);
    if (rc) return rc;
    if (inst < 0 || inst >= h->batch || slot < 0 || slot >= h->ss.cap || !T) return fail(LMPC_E_INVALID, "bad instance/slot");
    CK(cudaSetDevice(h->device));
    const size_t lap = h->ss.lap_index(inst, slot);
    CK(cudaMemcpyAsync(T, h->ss.len + lap, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (x) CK(cudaMemcpyAsync(x, h->ss.x + lap * h->ss.Tmax * 6, sizeof(double) * (*T) * 6, cudaMemcpyDeviceToHost, h->stream));
    if (u) CK(cudaMemcpyAsync(u, h->ss.u + lap * h->ss.Tmax * 2, sizeof(double) * (*T) * 2, cudaMemcpyDeviceToHost, h->stream));
    if (qfun) CK(cudaMemcpyAsync(qfun, h->ss.q + lap * h->ss.Tmax, sizeof(double) * (*T), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_ss_patch_row(lmpc_handle* h, int inst, int slot, int row, const double* x6, int also_model_slot) {
    int rc = need_store(h);
    if (rc) return rc;
    if (inst < 0 || inst >= h->batch || slot < 0 || slot >= h->ss.cap || row < 0 || row >= h->ss.Tmax || !x6)
        return fail(LMPC_E_INVALID, "bad patch arguments");
    CK(cudaSetDevice(h->device));
    CK(cudaMemcpyAsync(h->ss.x + (h->ss.lap_index(inst, slot) * h->ss.Tmax + row) * 6, x6, sizeof(double) * 6, cudaMemcpyHostToDevice, h->stream));
    if (also_model_slot >= 0 && also_model_slot < h->mdl.cap)
        CK(cudaMemcpyAsync(h->mdl.x + (h->mdl.lap_index(inst, also_model_slot) * h->mdl.Tmax + row) * 6, x6, sizeof(double) * 6,
                           cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_state_set(lmpc_handle* h, const double* xLin, const double* uLin, const double* zt, const double* OldInput,
                   const int* timeStep, const int* has_pred, const double* xPred) {
    int rc = need_store(h);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    const size_t B = h->batch, N = h->N, D = sizeof(double);
    cudaStream_t s = h->stream;
    if (xLin) CK(cudaMemcpyAsync(h->d_xLin, xLin, B * (N + 1) * 6 * D, cudaMemcpyHostToDevice, s));
    if (uLin) CK(cudaMemcpyAsync(h->d_uLin, uLin, B * N * 2 * D, cudaMemcpyHostToDevice, s));
    if (zt) CK(cudaMemcpyAsync(h->d_ztState, zt, B * 6 * D, cudaMemcpyHostToDevice, s));
    if (OldInput) CK(cudaMemcpyAsync(h->d_OldInput, OldInput, B * 2 * D, cudaMemcpyHostToDevice, s));
    if (timeStep) CK(cudaMemcpyAsync(h->d_timeStep, timeStep, B * sizeof(int), cudaMemcpyHostToDevice, s));
    if (has_pred) CK(cudaMemcpyAsync(h->d_hasPred, has_pred, B * sizeof(int), cudaMemcpyHostToDevice, s));
    if (xPred) CK(cudaMemcpyAsync(h->d_xPredPrev, xPred, B * (N + 1) * 6 * D, cudaMemcpyHostToDevice, s));
    if (h->d_warm_valid) CK(cudaMemsetAsync(h->d_warm_valid, 0, sizeof(int) * B, s));     // a new controller state starts cold
    CK(cudaStreamSynchronize(s));
    return LMPC_OK;
}

int lmpc_state_get(lmpc_handle* h, double* xLin, double* uLin, double* zt, double* OldInput, int* timeStep) {
    int rc = need_store(h);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    const size_t B = h->batch, N = h->N, D = sizeof(double);
    cudaStream_t s = h->stream;
    if (xLin) CK(cudaMemcpyAsync(xLin, h->d_xLin, B * (N + 1) * 6 * D, cudaMemcpyDeviceToHost, s));
    if (uLin) CK(cudaMemcpyAsync(uLin, h->d_uLin, B * N * 2 * D, cudaMemcpyDeviceToHost, s));
    if (zt) CK(cudaMemcpyAsync(zt, h->d_ztState, B * 6 * D, cudaMemcpyDeviceToHost, s));
    if (OldInput) CK(cudaMemcpyAsync(OldInput, h->d_OldInput, B * 2 * D, cudaMemcpyDeviceToHost, s));
    if (timeStep) CK(cudaMemcpyAsync(timeStep, h->d_timeStep, B * sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return LMPC_OK;
}

static int launch_k1(lmpc_handle* h, int b0 = 0, int nb = -1, cudaStream_t st = nullptr) {
    if (nb < 0) nb = h->batch;
    if (!st) st = h->stream;
    K1Args a;
    a.batch = h->batch; a.N = h->N; a.b0 = b0;
    a.wpb = h->N < 12 ? h->N : 12;
    a.pts_stride = k1_pts_stride(h->mc.trToUse);
    a.xLin = h->d_xLin; a.uLin = h->d_uLin; a.pool = h->mdl; a.used = h->d_used; a.abc = h->hb[0].abc; a.status = h->d_flags;
    a.trk = tracks(h);
    dim3 grid(nb, (h->N + a.wpb - 1) / a.wpb);
    size_t smem = sizeof(float) * 5 * K1_TILE + sizeof(double) * (size_t)a.pts_stride * a.wpb;
    knn_ltv_regress_kernel<<<grid, 32 * a.wpb, smem, st>>>(h->mc, a);
    CK(cudaGetLastError());
    h->launches += 1;
    return LMPC_OK;
}

static int launch_k2(lmpc_handle* h, const double* d_x0, int b0 = 0, int nb = -1, cudaStream_t st = nullptr) {
    if (nb < 0) nb = h->batch;
    if (!st) st = h->stream;
    K2Args a;
    a.batch = h->batch; a.N = h->N; a.b0 = b0; a.numSS_it = h->p.numSS_it; a.P = h->M / h->p.numSS_it;
    a.trk = tracks(h);
    a.x0 = d_x0; a.zt = h->d_ztState; a.pool = h->ss; a.sel = h->d_sel; a.is_prev = h->d_isprev;
    a.timeStep = h->d_timeStep; a.has_pred = h->d_hasPred; a.xPred = h->d_xPredPrev;
    a.SS_sel = h->hb[0].SS; a.Qfun_sel = h->hb[0].Qfun; a.Succ_SS = h->hb[0].SuccSS; a.Succ_uSS = h->hb[0].SuccU;
    a.zt_fixed = h->d_ztFixed; a.status = h->d_flags; a.min_index = h->d_minidx;
    ss_select_kernel<<<nb, 32 * a.numSS_it, 0, st>>>(a);
    CK(cudaGetLastError());
    h->launches += 1;
    return LMPC_OK;
}

int lmpc_identify_host(lmpc_handle* h, double* abc_out, int* flags) {
    int rc = need_store(h);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    CK(cudaMemsetAsync(h->d_flags, 0, sizeof(int) * h->batch, h->stream));
    rc = launch_k1(h);
    if (rc) return rc;
    if (abc_out) CK(cudaMemcpyAsync(abc_out, h->hb[0].abc, sizeof(double) * h->batch * h->N * 54, cudaMemcpyDeviceToHost, h->stream));
    if (flags) CK(cudaMemcpyAsync(flags, h->d_flags, sizeof(int) * h->batch, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_select_host(lmpc_handle* h, const double* x0, double* SS_sel, double* Qfun_sel, double* Succ_SS, double* Succ_uSS,
                     int* min_index, int* flags) {
    int rc = need_store(h);
    if (rc) return rc;
    if (h->M <= 0 || !x0) return fail(LMPC_E_INVALID, "handle has no safe set or x0 is null");
    CK(cudaSetDevice(h->device));
    const size_t B = h->batch, M = h->M, D = sizeof(double);
    cudaStream_t s = h->stream;
    CK(cudaMemcpyAsync(h->hb[0].x0, x0, B * 6 * D, cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(h->d_flags, 0, sizeof(int) * B, s));
    rc = launch_k2(h, h->hb[0].x0);
    if (rc) return rc;
    if (SS_sel) CK(cudaMemcpyAsync(SS_sel, h->hb[0].SS, B * 6 * M * D, cudaMemcpyDeviceToHost, s));
    if (Qfun_sel) CK(cudaMemcpyAsync(Qfun_sel, h->hb[0].Qfun, B * M * D, cudaMemcpyDeviceToHost, s));
    if (Succ_SS) CK(cudaMemcpyAsync(Succ_SS, h->hb[0].SuccSS, B * 6 * M * D, cudaMemcpyDeviceToHost, s));
    if (Succ_uSS) CK(cudaMemcpyAsync(Succ_uSS, h->hb[0].SuccU, B * 2 * M * D, cudaMemcpyDeviceToHost, s));
    if (min_index) CK(cudaMemcpyAsync(min_index, h->d_minidx, B * h->p.numSS_it * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (flags) CK(cudaMemcpyAsync(flags, h->d_flags, B * sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return LMPC_OK;
}

struct StepTail;
static int step_dev_impl(lmpc_handle* h, int mode, const double* x0_dev, cudaEvent_t* ev, const StepTail* tail);
int lmpc_step_dev(lmpc_handle* h, int mode, const double* x0_dev) { return step_dev_impl(h, mode, x0_dev, nullptr, nullptr); }

// The same step with CUDA events between its kernels: ms4 = durations of K1 (regression), K2 (selection; 0 for mode 0), the QP
// kernel and the state shift.  Measurement support (bench.py's per-kernel rooflines); synchronises.
int lmpc_step_profile(lmpc_handle* h, int mode, const double* x0_dev, float* ms4) {
    if (!h || !ms4) return fail(LMPC_E_INVALID, "null argument");
    CK(cudaSetDevice(h->device));
    cudaEvent_t ev[5];
    for (int i = 0; i < 5; ++i) CK(cudaEventCreate(&ev[i]));
    int rc = step_dev_impl(h, mode, x0_dev, ev, nullptr);
    if (rc == LMPC_OK && cudaStreamSynchronize(h->stream) != cudaSuccess) rc = fail(LMPC_E_CUDA, "stream synchronisation failed");
    if (rc == LMPC_OK)
        for (int i = 0; i < 4; ++i) cudaEventElapsedTime(&ms4[i], ev[i], ev[i + 1]);
    for (int i = 0; i < 5; ++i) cudaEventDestroy(ev[i]);
    return rc;
}
}  // extern "C"

// K1 -> K2 -> QP -> shift (PC.py:110-137) for the controllers [b0, b0 + nb) on stream st.  `tail` (rollouts) appends what
// Simulator.sim does with the result for the same controllers: addPoint (mode 1) and dynModel.
struct StepTail { const double* xc; SimArgs sim; };
static int step_range(lmpc_handle* h, int mode, const double* x0_dev, cudaEvent_t* ev, int b0, int nb, cudaStream_t st, const StepTail* tail) {
    int rc;
    const bool lm = mode == 1;
    const QpBufs& q = h->hb[0];
    if ((rc = launch_k1(h, b0, nb, st)) != LMPC_OK) return rc;                       // PC.py:117
    if (ev) CK(cudaEventRecord(ev[1], st));
    if (lm && (rc = launch_k2(h, x0_dev, b0, nb, st)) != LMPC_OK) return rc;         // PC.py:121
    if (ev) CK(cudaEventRecord(ev[2], st));
    FtocpArgs a = qp_args(h, q, lm, QP_ALL);                                         // PC.py:124-125
    a.x0 = x0_dev; a.uOld = h->d_OldInput;
    if (h->d_warm) { a.warm = h->d_warm; a.warm_valid = h->d_warm_valid; a.warm_stride = h->warm_stride; }
    if ((rc = launch(h, a.range(b0, nb, h->N, h->M), lm, st)) != LMPC_OK) return rc;
    if (ev) CK(cudaEventRecord(ev[3], st));
    ShiftArgs sa;
    sa.batch = h->batch; sa.N = h->N; sa.lmpc = mode; sa.b0 = b0;
    sa.xPred = q.xPred; sa.uPred = q.uPred; sa.zt_in = q.zt; sa.ztu_in = q.ztu;
    sa.xLin = h->d_xLin; sa.uLin = h->d_uLin; sa.zt = h->d_ztState; sa.OldInput = h->d_OldInput; sa.xPredPrev = h->d_xPredPrev;
    sa.timeStep = h->d_timeStep; sa.has_pred = h->d_hasPred;
    shift_state_kernel<<<nb, 64, 0, st>>>(sa);                                       // PC.py:129-137
    CK(cudaGetLastError());
    h->launches += 1;
    if (ev) CK(cudaEventRecord(ev[4], st));
    if (tail) {
        if (lm) {                                                                    // SysModel.py:38 -> PC.py:466-476
            ss_add_point_kernel<<<(nb + 127) / 128, 128, 0, st>>>(b0 + nb, h->ss, h->d_prevslot, tail->xc, q.uPred, (long long)h->N * 2,
                                                                  tracks(h), h->d_flags, nullptr, b0);
            CK(cudaGetLastError());
            h->launches += 1;
        }
        SimArgs sim = tail->sim;                                                     // SysModel.py:40 (dynModel)
        sim.b0 = b0; sim.b1 = b0 + nb;
        sim_step_kernel<<<(nb + 127) / 128, 128, 0, st>>>(h->mc, sim);
        CK(cudaGetLastError());
        h->launches += 1;
    }
    return LMPC_OK;
}

// The whole batch: one launch sequence on the handle's stream, or -- step_split > 1 -- one per instance range, each on its own
// stream between a fork and a join on the handle's stream.  The controllers are independent (PC.py:317-333), so the ranges only
// share the GPU: the regression scan of one range (issue-bound) runs under the interior-point solves of another (latency-bound)
// and the last waves of one range's solves are filled by the next range's.  Results are bit-identical to the unsplit step.
static int step_dev_impl(lmpc_handle* h, int mode, const double* x0_dev, cudaEvent_t* ev, const StepTail* tail) {
    int rc = need_store(h);
    if (rc) return rc;
    if (!x0_dev || (mode != 0 && mode != 1)) return fail(LMPC_E_INVALID, "bad mode or null x0");
    if (mode == 1 && h->M <= 0) return fail(LMPC_E_INVALID, "LMPC step on a handle without a safe set");
    CK(cudaSetDevice(h->device));
    CK(cudaMemsetAsync(h->d_flags, 0, sizeof(int) * h->batch, h->stream));
    if (h->d_warm && h->warm_mode != mode) {             // records of the other problem type are not comparable
        CK(cudaMemsetAsync(h->d_warm_valid, 0, sizeof(int) * h->batch, h->stream));
        h->warm_mode = mode;
    }
    if (ev) CK(cudaEventRecord(ev[0], h->stream));
    int split = ev ? 1 : h->step_split;                  // the per-kernel timing of lmpc_step_profile needs the kernels back to back
    if (split > h->batch / 256) split = h->batch / 256;  // ranges below a few hundred controllers only add launches
    if (split <= 1) return step_range(h, mode, x0_dev, ev, 0, h->batch, h->stream, tail);
    CK(cudaEventRecord(h->ev_fork, h->stream));
    for (int r = 0; r < split; ++r) {
        const int b0 = (int)((long long)h->batch * r / split), b1 = (int)((long long)h->batch * (r + 1) / split);
        cudaStream_t st = h->cstream[r];
        CK(cudaStreamWaitEvent(st, h->ev_fork, 0));
        if ((rc = step_range(h, mode, x0_dev, nullptr, b0, b1 - b0, st, tail)) != LMPC_OK) break;
        CK(cudaEventRecord(h->ev_join[r], st));
    }
    if (rc != LMPC_OK) {                                  // ranges already enqueued finish before the error is reported
        for (int r = 0; r < split; ++r) cudaStreamSynchronize(h->cstream[r]);
        return rc;
    }
    for (int r = 0; r < split; ++r) CK(cudaStreamWaitEvent(h->stream, h->ev_join[r], 0));
    return LMPC_OK;
}
extern "C" {

int lmpc_step_host(lmpc_handle* h, int mode, const double* x0, double* xPred, double* uPred, double* lambd, double* zt,
                   double* zt_u, double* SS_sel, int* status, int* iters, double* resid, int* flags) {
    int rc = need_store(h);
    if (rc) return rc;
    if (!x0) return fail(LMPC_E_INVALID, "null x0");
    CK(cudaSetDevice(h->device));
    const size_t B = h->batch, N = h->N, M = h->M > 0 ? h->M : 1, D = sizeof(double);
    cudaStream_t s = h->stream;
    CK(cudaMemcpyAsync(h->hb[0].x0, x0, B * 6 * D, cudaMemcpyHostToDevice, s));
    rc = lmpc_step_dev(h, mode, h->hb[0].x0);
    if (rc) return rc;
    if (xPred) CK(cudaMemcpyAsync(xPred, h->hb[0].xPred, B * (N + 1) * 6 * D, cudaMemcpyDeviceToHost, s));
    if (uPred) CK(cudaMemcpyAsync(uPred, h->hb[0].uPred, B * N * 2 * D, cudaMemcpyDeviceToHost, s));
    if (mode == 1) {
        if (lambd) CK(cudaMemcpyAsync(lambd, h->hb[0].lambd, B * M * D, cudaMemcpyDeviceToHost, s));
        if (zt) CK(cudaMemcpyAsync(zt, h->hb[0].zt, B * 6 * D, cudaMemcpyDeviceToHost, s));
        if (zt_u) CK(cudaMemcpyAsync(zt_u, h->hb[0].ztu, B * 2 * D, cudaMemcpyDeviceToHost, s));
        if (SS_sel) CK(cudaMemcpyAsync(SS_sel, h->hb[0].SS, B * 6 * M * D, cudaMemcpyDeviceToHost, s));
    }
    if (status) CK(cudaMemcpyAsync(status, h->hb[0].status, B * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (iters) CK(cudaMemcpyAsync(iters, h->hb[0].iters, B * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (resid) CK(cudaMemcpyAsync(resid, h->hb[0].resid, B * 3 * D, cudaMemcpyDeviceToHost, s));
    if (flags) CK(cudaMemcpyAsync(flags, h->d_flags, B * sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return LMPC_OK;
}

int lmpc_read_buffer(lmpc_handle* h, const char* name, size_t offset_bytes, void* dst, size_t bytes) {
    if (!h || !name || !dst) return fail(LMPC_E_INVALID, "null argument");
    const char* p = (const char*)lmpc_device_buffer(h, name);
    if (!p) return fail(LMPC_E_INVALID, "unknown buffer name");
    CK(cudaSetDevice(h->device));
    CK(cudaMemcpyAsync(dst, p + offset_bytes, bytes, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_step_results(lmpc_handle* h, int* status, int* iters, double* resid, int* flags) {
    int rc = need_store(h);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    const size_t B = h->batch;
    if (status) CK(cudaMemcpyAsync(status, h->hb[0].status, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    if (iters) CK(cudaMemcpyAsync(iters, h->hb[0].iters, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    if (resid) CK(cudaMemcpyAsync(resid, h->hb[0].resid, sizeof(double) * B * 3, cudaMemcpyDeviceToHost, h->stream));
    if (flags) CK(cudaMemcpyAsync(flags, h->d_flags, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

void* lmpc_device_buffer(lmpc_handle* h, const char* name) {
    if (!h || !name) return nullptr;
    const QpBufs& q = h->hb[0];
    struct { const char* n; void* p; } tab[] = {
        {"xPred", q.xPred}, {"uPred", q.uPred}, {"lambd", q.lambd}, {"zt", q.zt}, {"zt_u", q.ztu},
        {"abc", q.abc}, {"SS_sel", q.SS}, {"Qfun_sel", q.Qfun}, {"Succ_SS", q.SuccSS}, {"Succ_uSS", q.SuccU},
        {"status", q.status}, {"iters", q.iters}, {"resid", q.resid}, {"flags", h->d_flags}, {"xLin", h->d_xLin},
        {"uLin", h->d_uLin}, {"x0", q.x0}, {"slack", q.slack}, {"slackT", q.slackT}, {"OldInput", h->d_OldInput}, {"abc_lti", h->has_rollout ? h->d_abc_lti : nullptr}};
    for (auto& e : tab) if (strcmp(e.n, name) == 0) return e.p;
    return nullptr;
}

// ================================================================================================
// device-resident closed loop: Simulator.sim's loop body (SysModel.py:33-48) without host round trips
// ================================================================================================
static int rollout_create_impl(lmpc_handle* h, int Tcl);
int lmpc_rollout_create(lmpc_handle* h, int Tcl) {
    const int rc = rollout_create_impl(h, Tcl);
    if (rc != LMPC_OK && h && !h->has_rollout) { const std::string msg = g_err; free_rollout(h); g_err = msg; }
    return rc;
}
}  // extern "C"
static int rollout_create_impl(lmpc_handle* h, int Tcl) {
    int rc = need_store(h);
    if (rc) return rc;
    if (h->has_rollout) return fail(LMPC_E_STATE, "rollout buffers already created");
    if (Tcl < 16) return fail(LMPC_E_INVALID, "Tcl too small");
    CK(cudaSetDevice(h->device));
    const size_t B = h->batch;
    for (int i = 0; i < 2; ++i) {
        CK(cudaMalloc((void**)&h->d_rx[i], sizeof(double) * B * 6));
        CK(cudaMalloc((void**)&h->d_rg[i], sizeof(double) * B * 6));
    }
    CK(cudaMalloc((void**)&h->d_clx, sizeof(double) * B * Tcl * 6));
    CK(cudaMalloc((void**)&h->d_clu, sizeof(double) * B * Tcl * 2));
    CK(cudaMalloc((void**)&h->d_z, sizeof(double) * B * 3));
    CK(cudaMalloc((void**)&h->d_zpid, sizeof(double) * B * 2));
    CK(cudaMalloc((void**)&h->d_abc_lti, sizeof(double) * B * 54));
    CK(cudaMemsetAsync(h->d_abc_lti, 0, sizeof(double) * B * 54, h->stream));
    CK(cudaMalloc((void**)&h->d_cllen, sizeof(int) * B));
    CK(cudaMalloc((void**)&h->d_done, sizeof(int) * B));
    CK(cudaMalloc((void**)&h->d_health, sizeof(int) * B * 2));
    CK(cudaMemsetAsync(h->d_health, 0, sizeof(int) * B * 2, h->stream));
    CK(cudaMemsetAsync(h->d_cllen, 0, sizeof(int) * B, h->stream));
    CK(cudaMemsetAsync(h->d_done, 0, sizeof(int) * B, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    h->Tcl = Tcl; h->cur = 0; h->sim_step = 0; h->has_rollout = true;
    return LMPC_OK;
}
extern "C" {

static int need_rollout(lmpc_handle* h) {
    int rc = need_store(h);
    if (rc) return rc;
    if (!h->has_rollout) return fail(LMPC_E_STATE, "call lmpc_rollout_create first");
    return LMPC_OK;
}

int lmpc_rollout_set_state(lmpc_handle* h, const double* x, const double* xglob) {
    int rc = need_rollout(h);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    if (x) CK(cudaMemcpyAsync(h->d_rx[h->cur], x, sizeof(double) * h->batch * 6, cudaMemcpyHostToDevice, h->stream));
    if (xglob) CK(cudaMemcpyAsync(h->d_rg[h->cur], xglob, sizeof(double) * h->batch * 6, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_rollout_get_state(lmpc_handle* h, double* x, double* xglob, int* done, int* cl_len) {
    int rc = need_rollout(h);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    const size_t B = h->batch;
    if (x) CK(cudaMemcpyAsync(x, h->d_rx[h->cur], sizeof(double) * B * 6, cudaMemcpyDeviceToHost, h->stream));
    if (xglob) CK(cudaMemcpyAsync(xglob, h->d_rg[h->cur], sizeof(double) * B * 6, cudaMemcpyDeviceToHost, h->stream));
    if (done) CK(cudaMemcpyAsync(done, h->d_done, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    if (cl_len) CK(cudaMemcpyAsync(cl_len, h->d_cllen, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_rollout_get_health(lmpc_handle* h, int* flags_or, int* unsolved_steps) {
    int rc = need_rollout(h);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    const size_t B = h->batch;
    if (flags_or) CK(cudaMemcpyAsync(flags_or, h->d_health, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    if (unsolved_steps) CK(cudaMemcpyAsync(unsolved_steps, h->d_health + B, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

// One closed-loop step for every instance, all on the device (SysModel.py:34-48):
//   Controller.solve(x) -> u = uPred[0] -> Controller.addPoint(x, u) (LMPC) -> x+ = dynModel(x, x_glob, u); done = s+ > TrackLength
int lmpc_rollout_step(lmpc_handle* h, int mode, const double* z_host, unsigned long long seed) {
    int rc = need_rollout(h);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    const QpBufs& q = h->hb[0];
    const double* xc = h->d_rx[h->cur];
    if (z_host) CK(cudaMemcpyAsync(h->d_z, z_host, sizeof(double) * h->batch * 3, cudaMemcpyHostToDevice, h->stream));
    StepTail tail;
    tail.xc = xc;
    SimArgs& sa = tail.sim;
    sa.batch = h->batch; sa.x = xc; sa.xg = h->d_rg[h->cur]; sa.u = q.uPred; sa.u_stride = (long long)h->N * 2;
    sa.z = z_host ? h->d_z : nullptr; sa.seed = seed; sa.step = h->sim_step;
    sa.xn = h->d_rx[h->cur ^ 1]; sa.xgn = h->d_rg[h->cur ^ 1];
    sa.cl_x = h->d_clx; sa.cl_u = h->d_clu; sa.cl_len = h->d_cllen; sa.Tcl = h->Tcl; sa.done = h->d_done; sa.active = nullptr;
    sa.flags = h->d_flags; sa.status = q.status; sa.health = h->d_health;
    sa.veh = h->d_veh; sa.veh_idx = h->d_veh_idx; sa.trk = tracks(h);
    // the trace of the chosen controllers reads the step's results and the state before dynModel: it has to sit between the
    // solve and the simulator, so a traced batch runs the simulator for the whole batch after it
    const bool fused_tail = !h->has_trace && mode != 2;
    if (mode == 2) {
        CK(cudaMemsetAsync(h->d_flags, 0, sizeof(int) * h->batch, h->stream));
        // LTI MPC with the per-instance model identified by lmpc_rollout_sysid (main.py:72-80); like the reference's LTI
        // controller it never refreshes the input-rate reference (OldInput keeps its initial value, PC.py:113-115)
        rc = lmpc_solve_mpc_dev(h, xc, h->d_OldInput, h->d_abc_lti, 54, 0, q.xPred, q.uPred, q.slack, q.status, q.iters, q.resid);
    } else {
        rc = step_dev_impl(h, mode, xc, nullptr, fused_tail ? &tail : nullptr);
    }
    if (rc) return rc;
    if (!fused_tail) {
        if (mode == 1) {
            ss_add_point_kernel<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(h->batch, h->ss, h->d_prevslot, xc, q.uPred,
                                                                                (long long)h->N * 2, tracks(h), h->d_flags, nullptr, 0);
            CK(cudaGetLastError());
            h->launches += 1;
        }
        if (h->has_trace) {
            trace_step_kernel<<<h->tr.n, 128, 0, h->stream>>>(h->tr, xc, h->d_rg[h->cur], q.uPred, (long long)h->N * 2, q.xPred,
                                                            mode == 1 ? q.SS : nullptr, h->has_books ? h->bk.lap_n : nullptr);
            CK(cudaGetLastError());
            h->launches += 1;
        }
        sim_step_kernel<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(h->mc, sa);
        CK(cudaGetLastError());
        h->launches += 1;
    }
    h->cur ^= 1;
    h->sim_step += 1;
    return LMPC_OK;
}

// One closed-loop step with the PID path follower as the controller (main.py:65-66: the lap that seeds everything else).
// z_pid_host[B,2] / z_sim_host[B,3]: the reference's standard-normal draws in its order (PID steer, PID accel | vx, vy, wz);
// NULL = Philox on the device.
int lmpc_rollout_pid_step(lmpc_handle* h, double vt, const double* z_pid_host, const double* z_sim_host, unsigned long long seed) {
    int rc = need_rollout(h);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    const double* xc = h->d_rx[h->cur];
    if (z_pid_host) CK(cudaMemcpyAsync(h->d_zpid, z_pid_host, sizeof(double) * h->batch * 2, cudaMemcpyHostToDevice, h->stream));
    if (z_sim_host) CK(cudaMemcpyAsync(h->d_z, z_sim_host, sizeof(double) * h->batch * 3, cudaMemcpyHostToDevice, h->stream));
    PidArgs pa;
    pa.batch = h->batch; pa.x = xc; pa.vt = vt; pa.z = z_pid_host ? h->d_zpid : nullptr; pa.seed = seed; pa.step = h->sim_step;
    pa.u = h->hb[0].uPred; pa.u_stride = (long long)h->N * 2;
    pid_input_kernel<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(pa);
    SimArgs sa;
    sa.batch = h->batch; sa.x = xc; sa.xg = h->d_rg[h->cur]; sa.u = h->hb[0].uPred; sa.u_stride = (long long)h->N * 2;
    sa.z = z_sim_host ? h->d_z : nullptr; sa.seed = seed; sa.step = h->sim_step;
    sa.xn = h->d_rx[h->cur ^ 1]; sa.xgn = h->d_rg[h->cur ^ 1];
    sa.cl_x = h->d_clx; sa.cl_u = h->d_clu; sa.cl_len = h->d_cllen; sa.Tcl = h->Tcl; sa.done = h->d_done; sa.active = nullptr;
    sa.flags = nullptr; sa.status = nullptr; sa.health = nullptr;
    sa.veh = h->d_veh; sa.veh_idx = h->d_veh_idx; sa.trk = tracks(h);
    sim_step_kernel<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(h->mc, sa);
    CK(cudaGetLastError());
    h->launches += 2;
    h->cur ^= 1;
    h->sim_step += 1;
    if (z_pid_host || z_sim_host) CK(cudaStreamSynchronize(h->stream));   // pageable host arrays of the caller
    return LMPC_OK;
}

// Per-controller vehicles: every set is checked, then the table replaces the previous one once the handle's streams are idle.
// Nothing about the handle changes unless every check passes.
int lmpc_rollout_set_vehicles(lmpc_handle* h, const lmpc_vehicle_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_rollout_set_vehicles";
    if (!h) return fail(LMPC_E_INVALID, "null handle");
    int rc = check_set_index(h, who, sets, nsets, set_of_instance);
    if (rc != LMPC_OK) return rc;
    for (int k = 0; k < nsets; ++k) {
        const lmpc_vehicle_params& v = sets[k];
        const double all[10] = {v.m, v.lf, v.lr, v.Iz, v.Df, v.Cf, v.Bf, v.Dr, v.Cr, v.Br};
        bool ok = v.m > 0 && v.Iz > 0 && v.lf > 0 && v.lr > 0;
        for (double x : all) ok = ok && isfinite(x);
        if (!ok)
            return fail(LMPC_E_INVALID, std::string(who) + ": vehicle " + std::to_string(k) +
                                            ": m, Iz, lf, lr must be positive and all ten values finite");
    }
    if (nsets == 0) {
        const lmpc_vehicle_params ref = reference_vehicle();
        return swap_table(h, who, &ref, 1, nullptr, &h->d_veh, &h->d_veh_idx);
    }
    return swap_table(h, who, sets, nsets, set_of_instance, &h->d_veh, &h->d_veh_idx);
}

// Regression(x, u, lamb) of Utilities.py:5-28 on every instance's closed-loop record: per-instance LTI model in the device
// buffer "abc_lti" ([B][54] = A | B | C = 0, the layout lmpc_solve_mpc_dev takes with strides (54, 0)); abc_host may be NULL.
int lmpc_rollout_sysid(lmpc_handle* h, double lamb, double* abc_host, int* flags_host) {
    int rc = need_rollout(h);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    CK(cudaMemsetAsync(h->d_flags, 0, sizeof(int) * h->batch, h->stream));
    ridge_sysid_kernel<<<h->batch, 32, 0, h->stream>>>(h->batch, h->d_clx, h->d_clu, h->d_cllen, h->Tcl, lamb, h->d_abc_lti, h->d_flags);
    CK(cudaGetLastError());
    h->launches += 1;
    if (abc_host) CK(cudaMemcpyAsync(abc_host, h->d_abc_lti, sizeof(double) * h->batch * 54, cudaMemcpyDeviceToHost, h->stream));
    if (flags_host) CK(cudaMemcpyAsync(flags_host, h->d_flags, sizeof(int) * h->batch, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

// main.py:99-110 on the device: every instance's record becomes `copies` identical laps in safe-set slots ss_slot0.. and
// regression slots model_slot0.., the controller state is initialised from it and the record restarts.
int lmpc_rollout_seed_from_record(lmpc_handle* h, int copies, int ss_slot0, int model_slot0) {
    int rc = need_rollout(h);
    if (rc) return rc;
    if (copies < 1 || ss_slot0 < 0 || model_slot0 < 0 || ss_slot0 + copies > h->ss.cap || model_slot0 + copies > h->mdl.cap)
        return fail(LMPC_E_INVALID, "seed copies do not fit the lap pools");
    CK(cudaSetDevice(h->device));
    h->laps_stored = true;
    if (h->d_warm_valid) CK(cudaMemsetAsync(h->d_warm_valid, 0, sizeof(int) * h->batch, h->stream));
    seed_from_record_kernel<<<h->batch, 256, 0, h->stream>>>(h->batch, h->ss, h->mdl, copies, ss_slot0, model_slot0, h->d_clx, h->d_clu,
                                                             h->d_cllen, h->Tcl, h->N, h->d_xLin, h->d_uLin, h->d_ztState, h->d_OldInput,
                                                             h->d_timeStep, h->d_hasPred, h->d_done, tracks(h));
    CK(cudaGetLastError());
    h->launches += 1;
    return LMPC_OK;
}

int lmpc_rollout_get_lap(lmpc_handle* h, int inst, int* T, double* x, double* u) {
    int rc = need_rollout(h);
    if (rc) return rc;
    if (inst < 0 || inst >= h->batch || !T) return fail(LMPC_E_INVALID, "bad instance");
    CK(cudaSetDevice(h->device));
    CK(cudaMemcpyAsync(T, h->d_cllen + inst, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (x) CK(cudaMemcpyAsync(x, h->d_clx + (size_t)inst * h->Tcl * 6, sizeof(double) * (*T) * 6, cudaMemcpyDeviceToHost, h->stream));
    if (u) CK(cudaMemcpyAsync(u, h->d_clu + (size_t)inst * h->Tcl * 2, sizeof(double) * (*T) * 2, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

// Hand the finished lap of `inst` over to the stores without leaving the device: safe-set slot (computeCost on the
// device) and/or regression slot (either may be -1), then restart the record; the curvilinear state is moved back by one
// track length (SysModel.py:50) and the controller's step counter is reset (PC.py:445).
int lmpc_rollout_commit_lap(lmpc_handle* h, int inst, int ss_slot, int model_slot) {
    int rc = need_rollout(h);
    if (rc) return rc;
    if (inst < 0 || inst >= h->batch || ss_slot >= h->ss.cap || model_slot >= h->mdl.cap) return fail(LMPC_E_INVALID, "bad instance/slot");
    CK(cudaSetDevice(h->device));
    if (ss_slot >= 0 || model_slot >= 0) h->laps_stored = true;
    if (ss_slot >= 0) {
        commit_lap_kernel<<<1, 256, 0, h->stream>>>(h->ss, inst, ss_slot, h->d_clx, h->d_clu, h->d_cllen, h->Tcl);
        rollout_cost_kernel<<<1, 256, 0, h->stream>>>(h->ss, inst, ss_slot, tracks(h));
        h->launches += 2;
    }
    if (model_slot >= 0) {
        commit_lap_kernel<<<1, 256, 0, h->stream>>>(h->mdl, inst, model_slot, h->d_clx, h->d_clu, h->d_cllen, h->Tcl);
        h->launches += 1;
    }
    CK(cudaGetLastError());
    // restart: cl_len = 0, s -= TrackLength, timeStep = 0, done = 0
    double s;
    CK(cudaMemcpyAsync(&s, h->d_rx[h->cur] + (size_t)inst * 6 + 4, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    s -= h->trk_host[h->trk_idx_host.empty() ? 0 : h->trk_idx_host[inst]].TrackLength;
    const int zero = 0;
    CK(cudaMemcpyAsync(h->d_rx[h->cur] + (size_t)inst * 6 + 4, &s, sizeof(double), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_cllen + inst, &zero, sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_done + inst, &zero, sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_timeStep + inst, &zero, sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

// The same hand-over for every instance with fin[b] != 0 in ONE launch (a Monte-Carlo batch finishes hundreds of laps in
// the same step).
int lmpc_rollout_commit_laps(lmpc_handle* h, const int* fin, const int* ss_slots, const int* model_slots) {
    int rc = need_rollout(h);
    if (rc) return rc;
    if (!fin || !ss_slots || !model_slots) return fail(LMPC_E_INVALID, "null argument");
    for (int b = 0; b < h->batch; ++b)
        if (fin[b] && (ss_slots[b] >= h->ss.cap || model_slots[b] >= h->mdl.cap)) return fail(LMPC_E_INVALID, "slot out of range");
    const size_t B = h->batch;
    CK(cudaSetDevice(h->device));
    for (int b = 0; b < h->batch; ++b)
        if (fin[b] && (ss_slots[b] >= 0 || model_slots[b] >= 0)) h->laps_stored = true;
    CK(cudaMemcpyAsync(h->d_xchg, fin, sizeof(int) * B, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_xchg + B, ss_slots, sizeof(int) * B, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_xchg + 2 * B, model_slots, sizeof(int) * B, cudaMemcpyHostToDevice, h->stream));
    commit_laps_kernel<<<h->batch, 256, 0, h->stream>>>(h->batch, h->ss, h->mdl, h->d_xchg, h->d_xchg + B, h->d_xchg + 2 * B, h->d_clx,
                                                        h->d_clu, h->d_cllen, h->Tcl, h->d_rx[h->cur], h->d_timeStep, h->d_done,
                                                        tracks(h));
    CK(cudaGetLastError());
    h->launches += 1;
    CK(cudaStreamSynchronize(h->stream));   // the three host arrays are pageable memory of the caller
    return LMPC_OK;
}

int lmpc_rollout_export_laps_dev(lmpc_handle* h, int Tpad, double* rows_dev, int* lens_dev) {
    int rc = need_rollout(h);
    if (rc) return rc;
    if (!rows_dev || !lens_dev || Tpad < 1) return fail(LMPC_E_INVALID, "bad export arguments");
    CK(cudaSetDevice(h->device));
    export_laps_kernel<<<h->batch, 256, 0, h->stream>>>(h->batch, h->d_clx, h->d_clu, h->d_cllen, h->Tcl, Tpad, rows_dev, lens_dev);
    CK(cudaGetLastError());
    h->launches += 1;
    return LMPC_OK;
}

int lmpc_ss_export_laps_dev(lmpc_handle* h, const int* slots, int Tpad, double* rows_dev, int* lens_dev) {
    int rc = need_store(h);
    if (rc) return rc;
    if (!slots || !rows_dev || !lens_dev || Tpad < 1) return fail(LMPC_E_INVALID, "bad export arguments");
    for (int b = 0; b < h->batch; ++b)
        if (slots[b] >= h->ss.cap) return fail(LMPC_E_INVALID, "safe-set slot out of range");
    CK(cudaSetDevice(h->device));
    CK(cudaMemcpyAsync(h->d_xchg, slots, sizeof(int) * h->batch, cudaMemcpyHostToDevice, h->stream));
    ss_export_laps_kernel<<<h->batch, 256, 0, h->stream>>>(h->batch, h->ss, h->d_xchg, Tpad, rows_dev, lens_dev);
    CK(cudaGetLastError());
    h->launches += 1;
    CK(cudaStreamSynchronize(h->stream));   // `slots` is pageable host memory of the caller
    return LMPC_OK;
}

int lmpc_ss_import_laps_dev(lmpc_handle* h, const int* ss_slots, const int* model_slots, const int* src, int n_src, int Tpad,
                            const double* rows_dev, const int* lens_dev) {
    int rc = need_store(h);
    if (rc) return rc;
    if (!ss_slots || !src || !rows_dev || !lens_dev || Tpad < 1 || n_src < 1) return fail(LMPC_E_INVALID, "bad import arguments");
    if ((rc = one_track(h, "lmpc_ss_import_laps_dev")) != LMPC_OK) return rc;
    for (int b = 0; b < h->batch; ++b) {
        if (ss_slots[b] >= h->ss.cap || (model_slots && model_slots[b] >= h->mdl.cap)) return fail(LMPC_E_INVALID, "slot out of range");
        if (src[b] >= n_src) return fail(LMPC_E_INVALID, "source lap index out of range");
    }
    const size_t B = h->batch;
    CK(cudaSetDevice(h->device));
    for (int b = 0; b < h->batch; ++b)
        if (src[b] >= 0 && (ss_slots[b] >= 0 || (model_slots && model_slots[b] >= 0))) h->laps_stored = true;
    CK(cudaMemcpyAsync(h->d_xchg, ss_slots, sizeof(int) * B, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_xchg + B, src, sizeof(int) * B, cudaMemcpyHostToDevice, h->stream));
    if (model_slots) CK(cudaMemcpyAsync(h->d_xchg + 2 * B, model_slots, sizeof(int) * B, cudaMemcpyHostToDevice, h->stream));
    ss_import_laps_kernel<<<h->batch, 256, 0, h->stream>>>(h->batch, h->ss, h->mdl, h->d_xchg, model_slots ? h->d_xchg + 2 * B : nullptr,
                                                           h->d_xchg + B, Tpad, rows_dev, lens_dev);
    CK(cudaGetLastError());
    h->launches += 1;
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

// ================================================================================================
// fp64 micro-benchmarks (probe.cuh): the measured denominators of the QP kernel's roofline
// ================================================================================================
int lmpc_probe_fp64(int device, double* out8) {
    if (!out8) return fail(LMPC_E_INVALID, "null output");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(LMPC_E_NODEVICE, "no CUDA device");
    if (device < 0 || device >= ndev) return fail(LMPC_E_INVALID, "bad device index");
    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    const int blocks = prop.multiProcessorCount * 8, threads = 256;
    double *d_out = nullptr, *d_lat = nullptr;
    CK(cudaMalloc((void**)&d_out, sizeof(double) * (size_t)blocks * threads));
    CK(cudaMalloc((void**)&d_lat, sizeof(double) * 64));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    float ms = 0.f;
    double best_dfma = 0.0, best_dmma = 0.0;
    const int it_f = 8192, it_m = 2048;
    for (int rep = 0; rep < 5; ++rep) {
        CK(cudaEventRecord(e0));
        probe_dfma_tput<<<blocks, threads>>>(d_out, it_f, 1.0 + rep);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        CK(cudaEventElapsedTime(&ms, e0, e1));
        const double tf = 2.0 * 8.0 * it_f * (double)blocks * threads / (ms * 1e-3) / 1e12;
        if (rep > 0 && tf > best_dfma) best_dfma = tf;
        CK(cudaEventRecord(e0));
        probe_dmma_tput<<<blocks, threads>>>(d_out, it_m, 1.0 + rep);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        CK(cudaEventElapsedTime(&ms, e0, e1));
        const double tm = 2.0 * 256.0 * 4.0 * it_m * (double)blocks * (threads / 32) / (ms * 1e-3) / 1e12;
        if (rep > 0 && tm > best_dmma) best_dmma = tm;
    }
    probe_latency<<<1, 32>>>(d_lat, d_lat + 8, 4096);
    probe_latency<<<1, 32>>>(d_lat, d_lat + 8, 4096);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    double lat[6];
    CK(cudaMemcpy(lat, d_lat, sizeof(lat), cudaMemcpyDeviceToHost));
    out8[0] = best_dfma; out8[1] = best_dmma;
    for (int i = 0; i < 6; ++i) out8[2 + i] = lat[i];
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    cudaFree(d_out); cudaFree(d_lat);
    return LMPC_OK;
}

// ================================================================================================
// device lap books (lapbooks.cuh): the reference's once-per-lap list bookkeeping without the host
// ================================================================================================
static int need_books(lmpc_handle* h) {
    int rc = need_store(h);
    if (rc) return rc;
    if (!h->has_books) return fail(LMPC_E_STATE, "lap books not allocated");
    return LMPC_OK;
}

int lmpc_books_set(lmpc_handle* h, const int* ss_time, const int* ss_lap, const int* it, const int* md_time, const int* md_seq,
                   const int* md_cnt) {
    int rc = need_books(h);
    if (rc) return rc;
    if (!ss_time || !ss_lap || !it || !md_time || !md_seq || !md_cnt) return fail(LMPC_E_INVALID, "null argument");
    CK(cudaSetDevice(h->device));
    const size_t B = h->batch, sc = h->bk.ss_cap, mc = h->bk.md_cap;
    cudaStream_t s = h->stream;
    CK(cudaMemcpyAsync(h->bk.ss_time, ss_time, sizeof(int) * B * sc, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(h->bk.ss_lap, ss_lap, sizeof(int) * B * sc, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(h->bk.it, it, sizeof(int) * B, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(h->bk.md_time, md_time, sizeof(int) * B * mc, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(h->bk.md_seq, md_seq, sizeof(int) * B * mc, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(h->bk.md_cnt, md_cnt, sizeof(int) * B, cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(h->bk.lap_n, 0, sizeof(int) * B, s));
    CK(cudaStreamSynchronize(s));
    return LMPC_OK;
}

int lmpc_books_get(lmpc_handle* h, int* ss_time, int* ss_lap, int* it, int* md_time, int* md_seq, int* md_cnt, int* sel, int* is_prev,
                   int* prev_slot, int* used, int* lap_hist, int* lap_n) {
    int rc = need_books(h);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    const size_t B = h->batch, sc = h->bk.ss_cap, mc = h->bk.md_cap, nit = h->bk.numSS_it, tr = h->bk.trToUse;
    cudaStream_t s = h->stream;
#define GET(dst, src, n) if (dst) CK(cudaMemcpyAsync(dst, src, sizeof(int) * (n), cudaMemcpyDeviceToHost, s))
    GET(ss_time, h->bk.ss_time, B * sc); GET(ss_lap, h->bk.ss_lap, B * sc); GET(it, h->bk.it, B);
    GET(md_time, h->bk.md_time, B * mc); GET(md_seq, h->bk.md_seq, B * mc); GET(md_cnt, h->bk.md_cnt, B);
    GET(sel, h->d_sel, B * nit); GET(is_prev, h->d_isprev, B * nit); GET(prev_slot, h->d_prevslot, B); GET(used, h->d_used, B * tr);
    GET(lap_hist, h->bk.lap_hist, B * LAP_HIST); GET(lap_n, h->bk.lap_n, B);
#undef GET
    CK(cudaStreamSynchronize(s));
    return LMPC_OK;
}

// Lap hand-over of every controller whose lap just ended, bookkeeping on the device; enqueue only.
int lmpc_rollout_commit_laps_dev(lmpc_handle* h) {
    int rc = need_rollout(h);
    if (rc) return rc;
    if ((rc = need_books(h)) != LMPC_OK) return rc;
    CK(cudaSetDevice(h->device));
    h->laps_stored = true;     // enqueue only: which controllers finish a lap is not known here
    commit_laps_books_kernel<<<h->batch, 256, 0, h->stream>>>(h->batch, h->ss, h->mdl, h->bk, h->d_clx, h->d_clu, h->d_cllen, h->Tcl,
                                                              h->d_rx[h->cur], h->d_timeStep, h->d_done, h->d_health, tracks(h),
                                                              h->M > 0 ? 1 : 0);
    CK(cudaGetLastError());
    h->launches += 1;
    return LMPC_OK;
}

int lmpc_rollout_seed_from_record_dev(lmpc_handle* h, int copies) {
    int rc = need_rollout(h);
    if (rc) return rc;
    if ((rc = need_books(h)) != LMPC_OK) return rc;
    if (copies < 1 || (h->M > 0 && copies > h->ss.cap) || copies > h->mdl.cap) return fail(LMPC_E_INVALID, "seed copies do not fit the lap pools");
    CK(cudaSetDevice(h->device));
    h->laps_stored = true;
    if (h->d_warm_valid) CK(cudaMemsetAsync(h->d_warm_valid, 0, sizeof(int) * h->batch, h->stream));
    seed_books_kernel<<<h->batch, 256, 0, h->stream>>>(h->batch, h->ss, h->mdl, h->bk, copies, h->d_clx, h->d_clu, h->d_cllen, h->Tcl, h->N,
                                                       h->d_xLin, h->d_uLin, h->d_ztState, h->d_OldInput, h->d_timeStep, h->d_hasPred,
                                                       h->d_done, tracks(h), h->M > 0 ? 1 : 0);
    CK(cudaGetLastError());
    h->launches += 1;
    return LMPC_OK;
}

int lmpc_rollout_stats(lmpc_handle* h, int* out4) {
    int rc = need_rollout(h);
    if (rc) return rc;
    if ((rc = need_books(h)) != LMPC_OK) return rc;
    if (!out4) return fail(LMPC_E_INVALID, "null output");
    CK(cudaSetDevice(h->device));
    rollout_stats_kernel<<<1, 1024, 0, h->stream>>>(h->batch, h->bk, h->d_cllen, h->d_health, h->d_stats);
    CK(cudaGetLastError());
    h->launches += 1;
    CK(cudaMemcpyAsync(out4, h->d_stats, sizeof(int) * 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

// Send side of the pooled exchange: the kbest fastest latest-own laps of this rank, packed on the device.
int lmpc_pool_export_dev(lmpc_handle* h, int kbest, int Tpad, long long gid_base, double* rows_dev, int* meta_dev) {
    int rc = need_books(h);
    if (rc) return rc;
    if (kbest < 1 || kbest > POOL_MAXK || Tpad < 1 || !rows_dev || !meta_dev) return fail(LMPC_E_INVALID, "bad export arguments");
    if (h->M <= 0) return fail(LMPC_E_STATE, "handle has no safe set");
    if ((rc = one_track(h, "lmpc_pool_export_dev")) != LMPC_OK) return rc;
    CK(cudaSetDevice(h->device));
    pool_local_best_kernel<<<1, 1024, 0, h->stream>>>(h->batch, h->bk, kbest, h->d_poolidx);
    pool_export_kernel<<<kbest, 256, 0, h->stream>>>(h->ss, h->bk, h->d_poolidx, Tpad, gid_base, rows_dev, meta_dev);
    CK(cudaGetLastError());
    h->launches += 2;
    return LMPC_OK;
}

// Receive side: rank the gathered laps, every controller files the `share` fastest it does not own.  took_host (may be NULL)
// receives the number of laps stored; the call then synchronises.
int lmpc_pool_import_dev(lmpc_handle* h, int n_src, int share, int Tpad, long long gid_base, const double* rows_dev, const int* meta_dev,
                         int* took_host) {
    int rc = need_books(h);
    if (rc) return rc;
    if (n_src < 1 || n_src > 64 || share < 1 || Tpad < 1 || !rows_dev || !meta_dev) return fail(LMPC_E_INVALID, "bad import arguments");
    if (h->M <= 0) return fail(LMPC_E_STATE, "handle has no safe set");
    if ((rc = one_track(h, "lmpc_pool_import_dev")) != LMPC_OK) return rc;
    CK(cudaSetDevice(h->device));
    h->laps_stored = true;
    int* order = h->d_poolidx + 64;
    int* took = h->d_poolidx + 200;
    CK(cudaMemsetAsync(took, 0, sizeof(int), h->stream));
    pool_rank_kernel<<<1, 64, 0, h->stream>>>(n_src, meta_dev, order);
    pool_import_kernel<<<h->batch, 256, 0, h->stream>>>(h->batch, h->ss, h->mdl, h->bk, n_src, share, Tpad, rows_dev, meta_dev, order, gid_base,
                                                        took, h->has_rollout ? h->d_health : nullptr);
    CK(cudaGetLastError());
    h->launches += 2;
    if (took_host) {
        CK(cudaMemcpyAsync(took_host, took, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
    }
    return LMPC_OK;
}

// ================================================================================================
// presentation support (SURVEY §8f rank 4): what plot.py reads, for device-resident batches
// ================================================================================================
int lmpc_track_global_position(int device, const double* table6, int nseg, double TrackLength, int n, const double* s, const double* ey,
                               double* xy, int* ok) {
    if (!table6 || nseg < 1 || nseg > 64 || n < 1 || !s || !ey || !xy) return fail(LMPC_E_INVALID, "bad arguments");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(LMPC_E_NODEVICE, "no CUDA device");
    if (device < 0 || device >= ndev) return fail(LMPC_E_INVALID, "bad device index");
    CK(cudaSetDevice(device));
    double *d_t = nullptr, *d_s = nullptr, *d_e = nullptr, *d_xy = nullptr;
    int* d_ok = nullptr;
    int rc = LMPC_OK;
    do {
#define TRY(call) if ((call) != cudaSuccess) { rc = fail(LMPC_E_CUDA, #call " failed"); break; }
        TRY(cudaMalloc((void**)&d_t, sizeof(double) * nseg * 6)); TRY(cudaMalloc((void**)&d_s, sizeof(double) * n));
        TRY(cudaMalloc((void**)&d_e, sizeof(double) * n)); TRY(cudaMalloc((void**)&d_xy, sizeof(double) * n * 2));
        TRY(cudaMalloc((void**)&d_ok, sizeof(int) * n));
        TRY(cudaMemcpy(d_t, table6, sizeof(double) * nseg * 6, cudaMemcpyHostToDevice));
        TRY(cudaMemcpy(d_s, s, sizeof(double) * n, cudaMemcpyHostToDevice));
        TRY(cudaMemcpy(d_e, ey, sizeof(double) * n, cudaMemcpyHostToDevice));
        track_global_position_kernel<<<(n + 127) / 128, 128>>>(d_t, nseg, TrackLength, n, d_s, d_e, d_xy, d_ok);
        TRY(cudaGetLastError());
        TRY(cudaMemcpy(xy, d_xy, sizeof(double) * n * 2, cudaMemcpyDeviceToHost));
        if (ok) TRY(cudaMemcpy(ok, d_ok, sizeof(int) * n, cudaMemcpyDeviceToHost));
#undef TRY
    } while (0);
    cudaFree(d_t); cudaFree(d_s); cudaFree(d_e); cudaFree(d_xy); cudaFree(d_ok);
    return rc;
}

int lmpc_rollout_trace_create(lmpc_handle* h, int n, const int* inst, int cap_steps) {
    int rc = need_rollout(h);
    if (rc) return rc;
    if (h->has_trace) return fail(LMPC_E_STATE, "trace buffers already created");
    if (n < 1 || n > 1024 || !inst || cap_steps < 1) return fail(LMPC_E_INVALID, "bad trace arguments");
    for (int i = 0; i < n; ++i) if (inst[i] < 0 || inst[i] >= h->batch) return fail(LMPC_E_INVALID, "traced controller out of range");
    CK(cudaSetDevice(h->device));
    TraceBufs& t = h->tr;
    t.n = n; t.cap = cap_steps; t.N = h->N; t.M = h->M > 0 ? h->M : 0;
    const size_t rows = (size_t)n * cap_steps, np = (size_t)(h->N + 1) * 6;
    CK(cudaMalloc((void**)&h->d_trinst, sizeof(int) * n));
    CK(cudaMalloc((void**)&t.steps, sizeof(int) * n));
    CK(cudaMalloc((void**)&t.x, sizeof(double) * rows * 6)); CK(cudaMalloc((void**)&t.g, sizeof(double) * rows * 6));
    CK(cudaMalloc((void**)&t.u, sizeof(double) * rows * 2)); CK(cudaMalloc((void**)&t.xPred, sizeof(double) * rows * np));
    CK(cudaMalloc((void**)&t.ss, sizeof(double) * rows * 6 * (t.M > 0 ? t.M : 1)));
    CK(cudaMalloc((void**)&t.lap, sizeof(int) * rows));
    CK(cudaMemcpyAsync(h->d_trinst, inst, sizeof(int) * n, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemsetAsync(t.steps, 0, sizeof(int) * n, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    t.inst = h->d_trinst;
    h->has_trace = true;
    return LMPC_OK;
}

int lmpc_rollout_trace_get(lmpc_handle* h, int tr, int* steps, double* x, double* xglob, double* u, double* xPred, double* SS_sel, int* lap) {
    int rc = need_rollout(h);
    if (rc) return rc;
    if (!h->has_trace || tr < 0 || tr >= h->tr.n || !steps) return fail(LMPC_E_INVALID, "no such trace");
    CK(cudaSetDevice(h->device));
    const TraceBufs& t = h->tr;
    cudaStream_t s = h->stream;
    CK(cudaMemcpyAsync(steps, t.steps + tr, sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    const size_t n = (size_t)*steps, o = (size_t)tr * t.cap, np = (size_t)(t.N + 1) * 6;
    if (n == 0) return LMPC_OK;
    if (x) CK(cudaMemcpyAsync(x, t.x + o * 6, sizeof(double) * n * 6, cudaMemcpyDeviceToHost, s));
    if (xglob) CK(cudaMemcpyAsync(xglob, t.g + o * 6, sizeof(double) * n * 6, cudaMemcpyDeviceToHost, s));
    if (u) CK(cudaMemcpyAsync(u, t.u + o * 2, sizeof(double) * n * 2, cudaMemcpyDeviceToHost, s));
    if (xPred) CK(cudaMemcpyAsync(xPred, t.xPred + o * np, sizeof(double) * n * np, cudaMemcpyDeviceToHost, s));
    if (SS_sel && t.M > 0) CK(cudaMemcpyAsync(SS_sel, t.ss + o * 6 * t.M, sizeof(double) * n * 6 * t.M, cudaMemcpyDeviceToHost, s));
    if (lap) CK(cudaMemcpyAsync(lap, t.lap + o, sizeof(int) * n, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return LMPC_OK;
}

}  // extern "C"
