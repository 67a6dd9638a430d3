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
#include <stddef.h>
#include <string.h>
#include <stdio.h>
#include <stdlib.h>
#include <string>
#include <algorithm>
#include <new>
#include <ctype.h>
#include <errno.h>
#include <unistd.h>
#include <sys/syscall.h>
#include <sys/mman.h>
#include <map>
#include <vector>
#include <mutex>
#include <algorithm>
#include <utility>

#include "../../include/lmpc_b200.h"
#include "ftocp_pdip.cuh"
#include "safeset.cuh"
#include "plant.cuh"
#include "observer.cuh"
#include "lapbooks.cuh"
#include "nominal_model.cuh"
#include "probe.cuh"
#include "ftocp_launch.cuh"
#include "snapshot.cuh"

using namespace lmpc;
static_assert(POOL_MAXG == LMPC_MAX_POOL_GROUPS, "the exchange scratch is sized for LMPC_MAX_POOL_GROUPS groups");

#define LMPC_HOST_SLOTS 4              // buffer sets (batches in flight) of the asynchronous host entry points

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

// The QP kernel's inputs and outputs for one whole batch, either a buffer set of the handle or the caller's arrays (of which the
// inputs are only read); null = not wanted.  QP_FIELDS describes every field.
struct QpIo {
    double *x0, *uOld, *abc, *SS, *Qfun, *SuccSS, *SuccU, *xPred, *uPred, *slack, *lambd, *slackT, *zt, *ztu;
    int *status, *iters;
    double* resid;
};

// One field of QpIo: c1 + cN * N + cM * M elements per instance (M = 1 for handles without a safe set), input or output, and
// whether only LMPC-type QPs (with a safe set) have it.  The table order is the order of the copies of a host solve.
struct QpField {
    size_t off, elem;
    int c1, cN, cM;
    bool in, lmpc_only;
    const char* name;          // lmpc_device_buffer name of buffer set 0, or null
    size_t count(size_t N, size_t M) const { return c1 + cN * N + cM * M; }
    void*& at(QpIo& q) const { return *(void**)((char*)&q + off); }
    void* at(const QpIo& q) const { return *(void* const*)((const char*)&q + off); }
};
#define QF(f, c1, cN, cM, in, lm, name) QpField{offsetof(QpIo, f), sizeof(*QpIo().f), c1, cN, cM, in, lm, name}
static const QpField QP_FIELDS[] = {
    QF(x0, 6, 0, 0, true, false, "x0"), QF(uOld, 2, 0, 0, true, false, nullptr), QF(abc, 0, 54, 0, true, false, "abc"),
    QF(SS, 0, 0, 6, true, true, "SS_sel"), QF(Qfun, 0, 0, 1, true, true, "Qfun_sel"), QF(SuccSS, 0, 0, 6, true, true, "Succ_SS"),
    QF(SuccU, 0, 0, 2, true, true, "Succ_uSS"),
    QF(xPred, 6, 6, 0, false, false, "xPred"), QF(uPred, 0, 2, 0, false, false, "uPred"), QF(slack, 0, 2, 0, false, false, "slack"),
    QF(lambd, 0, 0, 1, false, true, "lambd"), QF(slackT, 6, 0, 0, false, true, "slackT"), QF(zt, 6, 0, 0, false, true, "zt"),
    QF(ztu, 2, 0, 0, false, true, "zt_u"), QF(status, 1, 0, 0, false, false, "status"), QF(iters, 1, 0, 0, false, false, "iters"),
    QF(resid, 3, 0, 0, false, false, "resid")};
#undef QF

// The QP arrays of a public QP entry point's argument list
#define CALLER_QP_IO                                                                                                        \
    QpIo{const_cast<double*>(x0), const_cast<double*>(uOld), const_cast<double*>(abc), const_cast<double*>(SS_sel),        \
         const_cast<double*>(Qfun_sel), const_cast<double*>(Succ_SS), const_cast<double*>(Succ_uSS), xPred, uPred, slack, \
         lambd, slackTerminal, zt, zt_u, status, iters, resid}

// A per-controller table of the handle (DESIGN.md, "Per-controller tables"): device rows tab[rows.size()], or none, and the row
// of every controller idx[batch], or none (row 0 for all), with host copies of both (index empty when idx is null).  The arrays
// without rows (noise streams, lap budgets, pool groups) are the index alone.  swap_table replaces one, free_tables frees it.
template <typename T>
struct HandleTable {
    T* tab = nullptr;
    int* idx = nullptr;
    std::vector<T> rows;
    std::vector<int> index;
    Table<T> view() const { return Table<T>{tab, idx}; }
};
// the row controller b reads from t (which has rows)
template <typename T>
static int table_row(const HandleTable<T>& t, int b) { return t.index.empty() ? 0 : t.index[b]; }

struct lmpc_handle {
    lmpc_params p;
    FtocpConst c;
    int batch, device, N, M;
    cudaStream_t stream;
    cudaStream_t cstream[4 * LMPC_HOST_SLOTS];   // chunk pipelines of the *_host entry points (H2D | kernel | D2H overlap), 4 streams per slot
    int hb_chunks[LMPC_HOST_SLOTS];
    bool hb_pending[LMPC_HOST_SLOTS];            // enqueued and not yet waited for
    bool hb_lone;                                // set by the synchronous entry points: the batch being enqueued runs alone
    long long launches;
    // QP buffer sets, one per slot of the *_host entry points.  hb[0] is allocated at creation and is also the device-resident
    // step's (K1 writes its abc, K2 its safe set, the QP kernel its outputs; lmpc_device_buffer); hb[1..] on first use.
    QpIo hb[LMPC_HOST_SLOTS];
    unsigned long long* d_late;
    // warm-start records of the controllers of the device-resident step (lmpc_params.warm_start; allocated with the store)
    double* d_warm;
    int* d_warm_valid;
    long long warm_stride;
    int warm_mode;
    // per-controller parameters (lmpc_set_param_sets); no table = uniform handle
    HandleTable<FtocpConstRec> sets;
    // lap stores + controller state (lmpc_store_create)
    bool has_store;
    ModelConst mc;
    // tracks (lmpc_set_tracks); without sets the track of lmpc_store_create (store_trk)
    TrackRec store_trk;
    HandleTable<TrackRec> trk;
    bool laps_stored;          // a lap entered either pool: the track table is fixed from now on
    // regression constants (lmpc_set_regression_sets); without sets the constants of lmpc_store_create (store_reg)
    RegressionRec store_reg;
    HandleTable<RegressionRec> reg;
    // per-controller prediction models (lmpc_set_prediction_models), or none: every controller regresses (K1)
    HandleTable<PredictionModelRec> pmod;
    // per-controller shapes (lmpc_set_shapes), or none; shp_order's index is the batch sorted by (N, M), shp_cells the runs of
    // one shape in it (only shapes with controllers), own_c the one-row parameter table of a shaped handle without parameter sets
    HandleTable<ShapeRec> shp;
    HandleTable<int> shp_order;
    struct ShapeCell { int N, M, off, n; };
    std::vector<ShapeCell> shp_cells;
    HandleTable<FtocpConstRec> own_c;
    // per-controller safe-set lap counts (lmpc_set_ss_laps), or none: the handle's numSS_it
    HandleTable<SsLapsRec> ssl;
    // per-controller lap windows (lmpc_set_lap_windows), or none: every window unbounded
    HandleTable<LapWindowRec> lwin;
    // per-controller lane rules (lmpc_set_lane_rules), or none: every lap ranked by its lap time
    HandleTable<LaneRuleRec> lrule;
    // per-controller lane margins (lmpc_set_lane_margins), or none: every controller plans in the lane it is judged against.
    // d_margin [B] the margins m_b, d_plan [B] the planning rows every QP reads through the identity index d_plan_idx [B].
    HandleTable<LaneMarginRec> lmar;
    double* d_margin;
    FtocpConstRec* d_plan;
    int* d_plan_idx;
    LapPool ss, mdl;
    int *d_used, *d_sel, *d_isprev, *d_prevslot, *d_timeStep, *d_hasPred, *d_flags, *d_minidx, *d_xchg, *d_health, *d_dropped;
    double *d_xLin, *d_uLin, *d_ztState, *d_ztFixed, *d_OldInput, *d_xPredPrev, *d_tmpx, *d_tmpu;
    // device-resident closed loop (lmpc_rollout_create)
    bool has_rollout;
    int Tcl;
    unsigned long long sim_step;
    double *d_rx[2], *d_rg[2], *d_clx, *d_clu, *d_z, *d_zpid, *d_abc_lti;
    int *d_cllen, *d_done, cur;
    // vehicles of the simulator (lmpc_rollout_set_vehicles); without sets the reference vehicle (installed at creation)
    HandleTable<lmpc_vehicle_params> veh;
    // noise of the simulator and the PID (lmpc_rollout_set_noise); without sets the reference's constants (installed at
    // creation).  Philox stream of every controller (lmpc_rollout_set_noise_streams), or none for stream b = b.
    HandleTable<lmpc_noise_params> noise;
    HandleTable<int> streams;
    // measurement noise of the controllers (lmpc_rollout_set_measurement_noise), or none: they read the plant state.  d_xmeas is
    // the measured state of the current step (measure_kernel).
    HandleTable<lmpc_measurement_params> meas;
    double* d_xmeas;
    // state observers of the controllers (lmpc_rollout_set_observers), or none: they read the measured or plant state.  d_xest is
    // the state the controllers read in the current step (observe_kernel).
    HandleTable<lmpc_observer_params> obs;
    double* d_xest;
    // where the observers take their prior from (lmpc_rollout_set_observer_priors), or none: their own plan.  d_xprior is the prior
    // formed in the current step (observe_kernel<true>).
    HandleTable<lmpc_observer_prior_params> opri;
    double* d_xprior;
    // the observers' gains (lmpc_rollout_set_observer_gains), or none: every observer row's fixed gains.  d_ojac, d_ocov, d_ogain
    // are A, P and K of the current step's model gains (observer_gain_kernel).
    HandleTable<lmpc_observer_gain_params> ogain;
    double *d_ojac, *d_ocov, *d_ogain;
    // lap budgets (lmpc_rollout_set_lap_budget): laps every controller drives before it retires, or none for no budget
    HandleTable<int> budget;
    // track surfaces of the simulator (lmpc_rollout_set_surfaces), or none: the vehicle's grip all round the lap
    HandleTable<lmpc_surface_params> surf;
    // lap schedules (lmpc_rollout_set_lap_schedule) of the vehicle, noise, measurement and surface tables (LMPC_SCHEDULE_*): rows
    // [B][L] of the table per lap and no index, or none; sched_L[k] = L
    HandleTable<int> sched[4];
    int sched_L[4];
    // device lap books (lapbooks.cuh, allocated with the store): slot tables of both pools, lap history, exchange scratch
    LapBooks bk;
    int *d_poolidx, *d_stats;
    // pool groups of the exchange (lmpc_set_pool_groups): group of every controller; none / 0 = one pool
    HandleTable<int> pool_grp;
    int ngroups;
    int pool_min_over;         // rows a latest lap must have past its finish line to be exported (lmpc_set_pool_min_overrun)
    // rollout trace of chosen controllers (presentation support, lmpc_rollout_trace_*)
    TraceBufs tr;
    int* d_trinst;
    bool has_trace;
    // controller snapshots (snapshot.cuh): header template [SNAP_HDR_WORDS] + check verdict [4], allocated with the store
    int* d_snap;
    // per-lap reports (lmpc_rollout_enable_lap_reports): rows [B][rep_L] and running rows [B], or none (rep_L == 0)
    lmpc_lap_report* d_rep_rows;
    LapRun* d_rep_run;
    int rep_L;
};

// The handle's device buffers outside the QP buffer sets.  A buffer is [rows][B][per] elements (rows == 0: `per` elements for
// the whole handle), B being the batch, or the number of traced controllers for the trace.
enum BufOwner : unsigned {
    OWN_HANDLE = 1, OWN_STORE = 2, OWN_WARM = 4, OWN_ROLLOUT = 8, OWN_TRACE = 16, OWN_QP = 32, OWN_REPORTS = 64, OWN_MARGIN = 128
};
enum BufFill { FILL_NONE, FILL_ZERO, FILL_ONES };      // FILL_ONES: every int -1 (a free slot, no previous lap)
constexpr int SN_SCRATCH = -1;
struct DevBuf {
    void** p;             // the typed handle member it fills
    size_t elem, per;
    int rows;
    BufOwner own;         // what creates and frees it (OWN_WARM: the store, with lmpc_params.warm_start)
    BufFill fill;
    int sect;             // snapshot section of row 0 (row k: sect + k), or SN_SCRATCH
    const char* name;     // lmpc_device_buffer name, or null
    size_t bytes(size_t B) const { return elem * per * (rows ? rows * B : 1); }
};
template <typename T>
static DevBuf dbuf(T*& p, size_t per, BufOwner own, BufFill fill = FILL_NONE, int sect = SN_SCRATCH, const char* name = nullptr,
                   int rows = 1) {
    return DevBuf{(void**)&p, sizeof(T), per, rows, own, fill, sect, name};
}

// Every such buffer, sized from the handle's current dimensions.  Allocation, initial fill, release, the snapshot sections and
// the names of lmpc_device_buffer come from this table, so a new buffer gets a row here and nowhere else; every per-controller
// buffer is a snapshot section or per-step scratch (DESIGN.md, "Controller snapshots").
static std::vector<DevBuf> dev_bufs(lmpc_handle* h) {
    const size_t N = h->N, np = (N + 1) * 6, sc = h->ss.cap, mc = h->mdl.cap, T = h->ss.Tmax, nit = h->bk.numSS_it;
    const size_t Tcl = h->Tcl, cap = h->tr.cap, Mx = h->M > 0 ? h->M : 1;
    const BufOwner S = OWN_STORE, R = OWN_ROLLOUT, X = OWN_TRACE;
    LapBooks& k = h->bk;
    const int cur = h->cur, oth = h->cur ^ 1;
    return {
        dbuf(h->d_late, 1, OWN_HANDLE, FILL_ZERO, SN_SCRATCH, nullptr, 0),
        // lap pools, lap books, controller state
        dbuf(h->ss.x, sc * T * 6, S, FILL_NONE, SN_SS_X), dbuf(h->ss.u, sc * T * 2, S, FILL_NONE, SN_SS_U),
        dbuf(h->ss.q, sc * T, S, FILL_NONE, SN_SS_Q), dbuf(h->ss.len, sc, S, FILL_ZERO, SN_SS_LEN),
        dbuf(h->mdl.x, mc * T * 6, S, FILL_NONE, SN_MD_X), dbuf(h->mdl.u, mc * T * 2, S, FILL_NONE, SN_MD_U),
        dbuf(h->mdl.len, mc, S, FILL_ZERO, SN_MD_LEN),
        dbuf(k.ss_time, sc, S, FILL_ONES, SN_SS_TIME), dbuf(k.ss_lap, sc, S, FILL_ONES, SN_SS_LAP), dbuf(k.it, 1, S, FILL_ZERO, SN_IT),
        dbuf(k.md_time, mc, S, FILL_ONES, SN_MD_TIME), dbuf(k.md_seq, mc, S, FILL_ONES, SN_MD_SEQ),
        dbuf(k.md_cnt, 1, S, FILL_ZERO, SN_MD_CNT), dbuf(k.lap_hist, LAP_HIST, S, FILL_ONES, SN_LAP_HIST),
        dbuf(k.lap_n, 1, S, FILL_ZERO, SN_LAP_N),
        dbuf(h->d_sel, nit, S, FILL_ZERO, SN_SEL), dbuf(h->d_isprev, nit, S, FILL_ZERO, SN_ISPREV),
        dbuf(h->d_prevslot, 1, S, FILL_ONES, SN_PREVSLOT), dbuf(h->d_used, k.trToUse, S, FILL_ZERO, SN_USED),
        dbuf(h->d_xLin, np, S, FILL_NONE, SN_XLIN, "xLin"), dbuf(h->d_uLin, N * 2, S, FILL_NONE, SN_ULIN, "uLin"),
        dbuf(h->d_ztState, 6, S, FILL_ZERO, SN_ZT), dbuf(h->d_OldInput, 2, S, FILL_ZERO, SN_OLDINPUT, "OldInput"),
        dbuf(h->d_xPredPrev, np, S, FILL_ZERO, SN_XPREDPREV, "xPredPrev"), dbuf(h->d_timeStep, 1, S, FILL_ZERO, SN_TIMESTEP),
        dbuf(h->d_hasPred, 1, S, FILL_ZERO, SN_HASPRED, "has_pred"),
        dbuf(h->d_warm, (size_t)h->warm_stride, OWN_WARM, FILL_NONE, SN_WARM, "warm"),
        dbuf(h->d_warm_valid, 1, OWN_WARM, FILL_ZERO, SN_WARM_VALID, "warm_valid"),
        // store scratch: flags (cleared by every step), K2 outputs nothing reads later, staging of host arrays, exchange scratch
        dbuf(h->d_flags, 1, S, FILL_ZERO, SN_SCRATCH, "flags"), dbuf(h->d_minidx, nit, S), dbuf(h->d_ztFixed, 6, S),
        dbuf(h->d_tmpx, 6, S), dbuf(h->d_tmpu, 2, S), dbuf(h->d_xchg, 3, S),
        dbuf(h->d_dropped, 1, S, FILL_ZERO, SN_SCRATCH, nullptr, 0), dbuf(h->d_poolidx, POOL_SCRATCH, S, FILL_NONE, SN_SCRATCH, nullptr, 0),
        dbuf(h->d_stats, POOL_MAXG * 4, S, FILL_NONE, SN_SCRATCH, nullptr, 0),
        dbuf(h->d_snap, SNAP_HDR_WORDS + 4, S, FILL_NONE, SN_SCRATCH, nullptr, 0),
        // closed loop: the simulator's double buffer (the half at cur is the state, the other half is written before it is read)
        dbuf(h->d_rx[cur], 6, R, FILL_NONE, SN_RX), dbuf(h->d_rg[cur], 6, R, FILL_NONE, SN_RG), dbuf(h->d_rx[oth], 6, R),
        dbuf(h->d_rg[oth], 6, R), dbuf(h->d_clx, Tcl * 6, R, FILL_NONE, SN_CLX), dbuf(h->d_clu, Tcl * 2, R, FILL_NONE, SN_CLU),
        dbuf(h->d_cllen, 1, R, FILL_ZERO, SN_CLLEN), dbuf(h->d_done, 1, R, FILL_ZERO, SN_DONE),
        dbuf(h->d_health, 1, R, FILL_ZERO, SN_HEALTH_FLAGS, nullptr, 2),       // [2][B]: flags, then unsolved steps
        dbuf(h->d_abc_lti, 54, R, FILL_ZERO, SN_ABC_LTI, "abc_lti"), dbuf(h->d_z, 3, R), dbuf(h->d_zpid, 2, R),
        dbuf(h->d_xmeas, 6, R, FILL_ZERO, SN_SCRATCH, "x_meas"),     // formed from the plant state and the clock every step
        dbuf(h->d_xest, 6, R, FILL_ZERO, SN_SCRATCH, "x_est"),       // formed from x_meas and xPredPrev every step
        dbuf(h->d_xprior, 6, R, FILL_ZERO, SN_SCRATCH, "x_prior"),   // formed from xPredPrev and OldInput every step (prior table)
        dbuf(h->d_ojac, 36, R, FILL_ZERO, SN_SCRATCH, "obs_jac"),    // formed from xPredPrev, OldInput and the rows every step (gain table)
        dbuf(h->d_ocov, 36, R, FILL_ZERO, SN_SCRATCH, "obs_cov"),
        dbuf(h->d_ogain, 36, R, FILL_ZERO, SN_SCRATCH, "obs_gain"),
        // per-lap reports (lap_reports_reset_kernel gives the running rows their start)
        dbuf(h->d_rep_rows, (size_t)h->rep_L, OWN_REPORTS, FILL_ZERO, SN_LAP_REPORTS), dbuf(h->d_rep_run, 1, OWN_REPORTS, FILL_ZERO, SN_LAP_RUN),
        // lane margins (lmpc_set_lane_margins; lane_margin_rows_kernel fills them)
        dbuf(h->d_margin, 1, OWN_MARGIN, FILL_ZERO, SN_LANE_MARGIN), dbuf(h->d_plan, 1, OWN_MARGIN), dbuf(h->d_plan_idx, 1, OWN_MARGIN),
        // trace of chosen controllers (per traced controller)
        dbuf(h->d_trinst, 1, X), dbuf(h->tr.steps, 1, X, FILL_ZERO), dbuf(h->tr.x, cap * 6, X), dbuf(h->tr.g, cap * 6, X),
        dbuf(h->tr.u, cap * 2, X), dbuf(h->tr.xPred, cap * np, X), dbuf(h->tr.ss, cap * 6 * Mx, X), dbuf(h->tr.lap, cap, X)};
}

template <typename T>
static void free_null(T*& p) { if (p) cudaFree(p); p = nullptr; }

static void free_bufs(const std::vector<DevBuf>& rows, unsigned owners) {
    for (const DevBuf& r : rows) if (r.own & owners) free_null(*r.p);
}

// Free the per-controller tables that belong to `owners`: tracks, regression sets and pool groups go with the store, the others
// with the handle
static void free_tables(lmpc_handle* h, unsigned owners) {
    auto release = [owners](auto& t, BufOwner own) {
        if (!(own & owners)) return;
        free_null(t.tab); free_null(t.idx);
        t.rows.clear(); t.index.clear();
    };
    release(h->sets, OWN_HANDLE); release(h->veh, OWN_HANDLE); release(h->noise, OWN_HANDLE); release(h->streams, OWN_HANDLE);
    release(h->meas, OWN_HANDLE); release(h->obs, OWN_HANDLE); release(h->opri, OWN_HANDLE); release(h->ogain, OWN_HANDLE); release(h->surf, OWN_HANDLE); release(h->budget, OWN_HANDLE); release(h->trk, OWN_STORE); release(h->reg, OWN_STORE); release(h->pool_grp, OWN_STORE);
    for (auto& t : h->sched) release(t, OWN_HANDLE);
    release(h->shp, OWN_STORE); release(h->shp_order, OWN_STORE); release(h->own_c, OWN_HANDLE); release(h->ssl, OWN_STORE);
    release(h->lwin, OWN_STORE); release(h->lrule, OWN_STORE); release(h->lmar, OWN_STORE); release(h->pmod, OWN_STORE);
    if (owners & OWN_STORE) h->shp_cells.clear();
}

// Allocate the buffers of `rows` that belong to `owners` (all null on entry) for nb controllers and give them their initial
// fill.  On a failure every one of them is freed again, so nothing is left allocated and the call can be retried.
static int alloc_bufs(lmpc_handle* h, const std::vector<DevBuf>& rows, unsigned owners, size_t nb, const char* who) {
    cudaError_t e = cudaSuccess;
    bool filled = false;
    for (const DevBuf& r : rows) {
        if (!(r.own & owners) || e != cudaSuccess) continue;
        e = cudaMalloc(r.p, r.bytes(nb));
        if (e == cudaSuccess && r.fill != FILL_NONE) {
            e = cudaMemsetAsync(*r.p, r.fill == FILL_ONES ? 0xff : 0, r.bytes(nb), h->stream);
            filled = true;
        }
    }
    if (e == cudaSuccess && filled) e = cudaStreamSynchronize(h->stream);
    if (e == cudaSuccess) return LMPC_OK;
    free_bufs(rows, owners);
    return fail(LMPC_E_CUDA, std::string(who) + ": device allocation: " + cudaGetErrorString(e));
}

// Whole-buffer copies between handle buffers (rows of dev_bufs, sized by the table) and the caller's arrays, on the handle's
// stream: pairs (handle buffer, caller's array); a null array is skipped
static int copy_bufs(lmpc_handle* h, cudaMemcpyKind kind, std::initializer_list<std::pair<void*, const void*>> pairs) {
    const std::vector<DevBuf> rows = dev_bufs(h);
    for (const auto& pr : pairs) {
        if (!pr.second) continue;
        size_t n = 0;
        for (const DevBuf& r : rows) if (*r.p == pr.first) n = r.bytes(h->batch);
        void* host = const_cast<void*>(pr.second);
        if (kind == cudaMemcpyHostToDevice) CK(cudaMemcpyAsync(pr.first, host, n, kind, h->stream));
        else CK(cudaMemcpyAsync(host, pr.first, n, kind, h->stream));
    }
    return LMPC_OK;
}

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

// The argument rules of the calls that install a per-controller table: 0 <= nsets <= batch, nsets == 0 exactly when both arrays
// are NULL, every index in range.
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

// Once the handle's streams are idle, replace the rows of table t by rows[nrows] (none when nrows == 0) and its index by
// set_of_instance[batch] (none when it is NULL), host copies included.  The handle keeps its old table unless every allocation
// and copy succeeds.
template <typename T>
static int swap_table(lmpc_handle* h, const char* who, HandleTable<T>& t, const T* rows, int nrows, const int* set_of_instance) {
    CK(cudaSetDevice(h->device));
    // batches already enqueued (the _async entry points, the device-resident step) finish with the table they were enqueued with
    CK(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < 4 * LMPC_HOST_SLOTS; ++i) CK(cudaStreamSynchronize(h->cstream[i]));
    T* tab = nullptr;
    int* ix = nullptr;
    cudaError_t e = cudaSuccess;
    if (nrows > 0) {
        e = cudaMalloc((void**)&tab, sizeof(T) * nrows);
        if (e == cudaSuccess) e = cudaMemcpy(tab, rows, sizeof(T) * nrows, cudaMemcpyHostToDevice);
    }
    if (e == cudaSuccess && set_of_instance) {
        e = cudaMalloc((void**)&ix, sizeof(int) * h->batch);
        if (e == cudaSuccess) e = cudaMemcpy(ix, set_of_instance, sizeof(int) * h->batch, cudaMemcpyHostToDevice);
    }
    if (e != cudaSuccess) {
        cudaFree(tab); cudaFree(ix);
        return fail(LMPC_E_CUDA, std::string(who) + ": " + cudaGetErrorString(e));
    }
    cudaFree(t.tab);
    cudaFree(t.idx);
    t.tab = tab;
    t.idx = ix;
    t.rows.assign(rows, rows + nrows);
    if (set_of_instance) t.index.assign(set_of_instance, set_of_instance + h->batch);
    else t.index.clear();
    return LMPC_OK;
}

// The calls that install a table with rows: the index rules, then row(k, rows[k]) checks set k and converts it into its row (an
// error refuses the call), then the swap.  nsets == 0 installs the default row *dflt, or no table when dflt is null.
template <typename T, typename Row>
static int install_table(lmpc_handle* h, const char* who, HandleTable<T>& t, const void* sets, int nsets, const int* set_of_instance,
                         const T* dflt, Row row) {
    int rc = check_set_index(h, who, sets, nsets, set_of_instance);
    if (rc != LMPC_OK) return rc;
    std::vector<T> rows(nsets);
    for (int k = 0; k < nsets; ++k)
        if ((rc = row(k, rows[k])) != LMPC_OK) return rc;
    if (nsets == 0 && dflt) rows.assign(1, *dflt);
    return swap_table(h, who, t, rows.data(), (int)rows.size(), set_of_instance);
}

// Simulator.dynModel's vehicle (SysModel.py:61-70), D in the reference's operation order
static lmpc_vehicle_params reference_vehicle() {
    lmpc_vehicle_params v;
    v.m = 1.98; v.lf = 0.125; v.lr = 0.125; v.Iz = 0.024;
    v.Df = 0.8 * v.m * 9.81 / 2.0; v.Cf = 1.25; v.Bf = 1.0;
    v.Dr = 0.8 * v.m * 9.81 / 2.0; v.Cr = 1.25; v.Br = 1.0;
    return v;
}

// The noise of Simulator.dynModel (SysModel.py:139-145) and of the PID path follower (Utilities.py:42-68)
static lmpc_noise_params reference_noise() {
    return lmpc_noise_params{{0.01, 0.01, 0.005}, {0.05, 0.05, 0.05}, 0.01, {0.25, 0.10}, {0.9, 0.2}};
}

template <int N, int M>
static int configure_t(cudaStream_t) {
    CK(cudaFuncSetAttribute(ftocp_kernel<N, M, 2, 4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)sizeof(KernelSmem<N, M, 2, 4, false>)));
    return LMPC_OK;
}

// The parameter table the QP kernels read: the planning rows of a lane-margin table, else the parameter sets, else none
static const FtocpConstRec* qp_table(const lmpc_handle* h) { return h->lmar.tab ? h->d_plan : h->sets.tab; }

template <int N, int M>
static int launch_t(lmpc_handle* h, const FtocpArgs& a, cudaStream_t st) {
    if (qp_table(h))     // per-controller parameters or margins: every instance reads its own row (ftocp_sets.cu)
        CK(ftocp_sets_launch(N, M, qp_table(h), a, st));
    else {
        ftocp_kernel<N, M, 2, 4, false><<<a.batch, 32, sizeof(KernelSmem<N, M, 2, 4, false>), st>>>(h->c, a);
        CK(cudaGetLastError());
    }
    h->launches += 1;
    return LMPC_OK;
}

// A shaped handle (lmpc_set_shapes): one launch of ftocp_shaped_kernel per run of one shape in the sorted batch, or per run of one
// horizon for the MPC-type QP; parameters from the planning rows of a lane-margin table, the parameter-set table, or the handle's
// own row
static int launch_shaped(lmpc_handle* h, const FtocpArgs& a, bool lmpc_mode, cudaStream_t st) {
    const FtocpConstRec* table = qp_table(h) ? qp_table(h) : h->own_c.tab;
    const auto& cells = h->shp_cells;
    for (size_t k = 0, j; k < cells.size(); k = j) {
        int n = 0;
        for (j = k; j < cells.size() && cells[j].N == cells[k].N && (!lmpc_mode || cells[j].M == cells[k].M); ++j) n += cells[j].n;
        const ShapedLaunch s{h->shp_order.idx + cells[k].off, h->N, h->M};
        CK(ftocp_shaped_launch(cells[k].N, lmpc_mode ? cells[k].M : 0, table, s, n, a, st));
        h->launches += 1;
    }
    return LMPC_OK;
}

static int launch(lmpc_handle* h, const FtocpArgs& a, bool lmpc_mode, cudaStream_t st) {
    if (h->shp.tab) return launch_shaped(h, a, lmpc_mode, st);
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

static void free_store(lmpc_handle* h) {
    free_bufs(dev_bufs(h), OWN_STORE | OWN_WARM | OWN_MARGIN);
    free_tables(h, OWN_STORE);
    h->ngroups = 0;
    h->laps_stored = false;
    h->has_store = false;
}

static Tracks tracks(const lmpc_handle* h) { return h->trk.view(); }

// The lap budgets as the kernels of the device-resident closed loop take them.  Everything else (the host-driven entry points,
// the PID lap, the host-slot hand-over) passes LapBudget{}: nobody is retired there.
static LapBudget lap_budget(const lmpc_handle* h) { return LapBudget{h->budget.idx, h->bk.lap_n}; }

// The lap schedule of table k (LMPC_SCHEDULE_*) as lmpc_rollout_step's kernels take it; the same places that pass LapBudget{} pass
// LapSchedule{} (the table's own index)
static LapSchedule lap_schedule(const lmpc_handle* h, int k) { return LapSchedule{h->sched[k].tab, h->sched_L[k], h->bk.lap_n}; }

// The report buffers and the QP constants the kernels of the closed loop read (all null without reports: the kernels then read
// none of them)
static LapReports reports(const lmpc_handle* h) {
    if (!h->rep_L) return LapReports{};
    return LapReports{h->d_rep_rows, h->d_rep_run, h->rep_L, h->sets.tab ? h->sets.view() : h->own_c.view()};
}

// The lane rules and the QP constants they judge against, as the lap-book kernels take them (read only while a rule table is installed)
static LaneRules lane_rules(const lmpc_handle* h) {
    return LaneRules{h->lrule.view(), h->sets.tab ? h->sets.view() : h->own_c.view()};
}
// A lane rule of mode 1 is installed (a row of the table; rows nobody reads count too)
static bool lane_rules_on(const lmpc_handle* h) {
    for (const LaneRuleRec& r : h->lrule.rows) if (r.mode == 1) return true;
    return false;
}
// Controller b's rule is on: its safe-set keys may carry LMPC_LANE_UNSAFE_KEY
static bool lane_rule_of(const lmpc_handle* h, int b) { return h->lrule.tab && h->lrule.rows[h->lrule.index[b]].mode == 1; }

// The lane margins, their untightened source rows and the planning rows, as the kernels take them (read only while a margin table
// is installed)
static LaneMargins lane_margins(const lmpc_handle* h) {
    return LaneMargins{h->lmar.view(), h->sets.tab ? h->sets.view() : h->own_c.view(), h->d_plan, h->d_margin, h->d_warm_valid};
}
// A lane-margin row of mode 2 is installed (rows nobody reads count too)
static bool lane_margins_adapt(const lmpc_handle* h) {
    for (const LaneMarginRec& r : h->lmar.rows) if (r.mode == 2) return true;
    return false;
}
// The planning rows of every controller from its source row and margin (lane_margin_rows_kernel); reset2: mode 2 margins start
// over at margin0.  Enqueued on the handle's stream; nothing without a table.
static int lane_margin_rows(lmpc_handle* h, bool reset2) {
    if (!h->lmar.tab) return LMPC_OK;
    lane_margin_rows_kernel<<<h->batch, 128, 0, h->stream>>>(h->batch, lane_margins(h), h->d_plan_idx, reset2 ? 1 : 0);
    CK(cudaGetLastError());
    h->launches += 1;
    return LMPC_OK;
}
// Does the margin of row r leave a lane of QP constants c: margin0 (mode 1) or margin_max (mode 2) below min_i bx_i
static bool margin_leaves_lane(const LaneMarginRec& r, const FtocpConst& c) {
    const double m = r.mode == 1 ? r.margin0 : r.mode == 2 ? r.margin_max : -1.0;
    return r.mode == 0 || (m < c.bx[0] && m < c.bx[1]);
}

static void free_rollout(lmpc_handle* h) {
    free_bufs(dev_bufs(h), OWN_ROLLOUT | OWN_TRACE | OWN_REPORTS);
    h->rep_L = 0;
    h->has_trace = false;
    h->has_rollout = false;
}

// The rows of QP buffer set q: every field of QP_FIELDS for the whole batch
static std::vector<DevBuf> qp_rows(const lmpc_handle* h, QpIo& q) {
    std::vector<DevBuf> rows;
    for (const QpField& f : QP_FIELDS)
        rows.push_back(DevBuf{&f.at(q), f.elem, f.count(h->N, h->M > 0 ? h->M : 1), 1, OWN_QP, FILL_NONE, SN_SCRATCH, nullptr});
    return rows;
}

// Buffer set `slot` of the handle, allocated on first use (x0 != null: allocated); null (and g_err set) if the allocation failed,
// which leaves nothing behind
static QpIo* qp_bufs(lmpc_handle* h, int slot) {
    QpIo& q = h->hb[slot];
    if (!q.x0 && alloc_bufs(h, qp_rows(h, q), OWN_QP, h->batch, ("QP buffer set " + std::to_string(slot)).c_str()) != LMPC_OK)
        return nullptr;
    return &q;
}

// Kernel arguments for the whole batch held in q (per-instance model, strides (N*54, 54)); null fields, and the safe-set ones of
// an MPC-type QP, stay null, which the kernel skips
static FtocpArgs qp_args(const lmpc_handle* h, const QpIo& q, bool lm) {
    FtocpArgs a = {};
    a.batch = h->batch;
    a.x0 = q.x0; a.uOld = q.uOld; a.abc = q.abc;
    a.abc_inst_stride = (long long)h->N * 54; a.abc_stage_stride = 54;
    a.xPred = q.xPred; a.uPred = q.uPred; a.slack = q.slack;
    if (lm) {
        a.SS = q.SS; a.Qfun = q.Qfun; a.SuccSS = q.SuccSS; a.SuccU = q.SuccU;
        a.lambd = q.lambd; a.slackT = q.slackT; a.zt = q.zt; a.ztu = q.ztu;
    }
    a.status = q.status; a.iters = q.iters; a.resid = q.resid;
    a.late = h->d_late;
    a.set_idx = h->lmar.tab ? h->d_plan_idx : h->sets.idx;
    return a;
}

// Copy the fields of buffer set 0 that dst names (the safe-set ones only when lm) into the caller's arrays, on the handle's stream
static int copy_out(lmpc_handle* h, const QpIo& dst, bool lm) {
    const size_t B = h->batch, N = h->N, M = h->M > 0 ? h->M : 1;
    for (const QpField& f : QP_FIELDS)
        if (f.at(dst) && (lm || !f.lmpc_only))
            CK(cudaMemcpyAsync(f.at(dst), f.at(h->hb[0]), B * f.count(N, M) * f.elem, cudaMemcpyDeviceToHost, h->stream));
    return LMPC_OK;
}

static int create_device_side(lmpc_handle* h) {
    CK(cudaSetDevice(h->device));
    int rc = configure(h->N, h->M > 0 ? h->M : 0);
    if (rc != LMPC_OK) return rc;
    CK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    for (int i = 0; i < 4 * LMPC_HOST_SLOTS; ++i) CK(cudaStreamCreateWithFlags(&h->cstream[i], cudaStreamNonBlocking));
    if (!qp_bufs(h, 0)) return LMPC_E_CUDA;
    if ((rc = alloc_bufs(h, dev_bufs(h), OWN_HANDLE, 1, "lmpc_create")) != LMPC_OK) return rc;
    FtocpConstRec own;
    own.c = h->c;
    if ((rc = swap_table(h, "lmpc_create", h->own_c, &own, 1, nullptr)) != LMPC_OK) return rc;
    const lmpc_vehicle_params ref = reference_vehicle();
    if ((rc = swap_table(h, "lmpc_create", h->veh, &ref, 1, nullptr)) != LMPC_OK) return rc;
    const lmpc_noise_params noise = reference_noise();
    return swap_table(h, "lmpc_create", h->noise, &noise, 1, nullptr);
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
    free_bufs(dev_bufs(h), OWN_HANDLE);
    free_tables(h, OWN_HANDLE);
    for (QpIo& q : h->hb) free_bufs(qp_rows(h, q), OWN_QP);
    if (h->stream) cudaStreamDestroy(h->stream);
    for (int i = 0; i < 4 * LMPC_HOST_SLOTS; ++i) if (h->cstream[i]) cudaStreamDestroy(h->cstream[i]);
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

// Per-controller parameters: every set goes through build_const (the conversion lmpc_create uses); nsets == 0 returns to the
// uniform kernel (DESIGN.md, "Per-controller tables").
int lmpc_set_param_sets(lmpc_handle* h, const lmpc_params* sets, int nsets, const int* set_of_instance) {
    if (!h) return fail(LMPC_E_INVALID, "null handle");
    // under a lane-margin table every controller's margin must leave a lane of its new row: need[k] is the widest margin a
    // controller of set k plans with (margin0 of mode 1, margin_max of mode 2), held by controller who[k]
    std::vector<double> need;
    std::vector<int> who;
    if (h->lmar.tab) {
        int rc = check_set_index(h, "lmpc_set_param_sets", sets, nsets, set_of_instance);
        if (rc != LMPC_OK) return rc;
        need.assign(nsets, -1.0);
        who.assign(nsets, -1);
        for (int b = 0; b < h->batch; ++b) {
            const LaneMarginRec& r = h->lmar.rows[h->lmar.index[b]];
            if (nsets == 0 && !margin_leaves_lane(r, h->c))
                return fail(LMPC_E_INVALID, "lmpc_set_param_sets: the lane margin of controller " + std::to_string(b) +
                                                " does not leave a lane of the handle's own bx");
            const double m = r.mode == 1 ? r.margin0 : r.mode == 2 ? r.margin_max : -1.0;
            if (nsets > 0 && r.mode != 0 && (who[set_of_instance[b]] < 0 || m > need[set_of_instance[b]])) {
                need[set_of_instance[b]] = m;
                who[set_of_instance[b]] = b;
            }
        }
    }
    int rc = install_table(h, "lmpc_set_param_sets", h->sets, sets, nsets, set_of_instance, (const FtocpConstRec*)nullptr,
                           [&](int k, FtocpConstRec& row) {
        const lmpc_params& s = sets[k];
        if (s.N != h->p.N || s.ncx != h->p.ncx || s.ncu != h->p.ncu || s.numSS_Points != h->p.numSS_Points ||
            s.numSS_it != h->p.numSS_it || s.warm_start != h->p.warm_start)
            return fail(LMPC_E_INVALID, "lmpc_set_param_sets: set " + std::to_string(k) +
                                            " differs from the handle in N, ncx, ncu, numSS_Points, numSS_it or warm_start");
        const int e = build_const(s, row.c);
        if (e != LMPC_OK) return fail(e, "lmpc_set_param_sets: set " + std::to_string(k) + ": " + g_err);
        if (h->lmar.tab && who[k] >= 0 && !margin_leaves_lane(h->lmar.rows[h->lmar.index[who[k]]], row.c))
            return fail(LMPC_E_INVALID, "lmpc_set_param_sets: set " + std::to_string(k) + ": the lane margin of controller " +
                                            std::to_string(who[k]) + " does not leave a lane of its bx");
        return LMPC_OK;
    });
    if (rc != LMPC_OK) return rc;
    if ((rc = lane_margin_rows(h, false)) != LMPC_OK) return rc;     // the planning rows follow the new source rows
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

}  // extern "C" (the helper below has C++ linkage)

// One solve of the device arrays io on the handle's stream; retire: the lap budgets (the closed loop's LTI-MPC step) or none
static int solve_dev(lmpc_handle* h, const QpIo& io, long long abc_inst_stride, long long abc_stage_stride, LapBudget retire) {
    if (!h || !io.x0 || !io.uOld || !io.abc || !io.xPred || !io.uPred || !io.status || !io.iters || !io.resid)
        return fail(LMPC_E_INVALID, "null argument");
    const bool lm = (io.SS != nullptr);
    if (lm && (h->M <= 0 || !io.Qfun)) return fail(LMPC_E_INVALID, "handle was created without a safe set (numSS_Points == 0)");
    if ((abc_inst_stride % 2) || (abc_stage_stride % 2)) return fail(LMPC_E_INVALID, "abc strides must be even (16-byte rows)");
    int rc;
    if ((rc = check_align(io.abc, "abc")) != LMPC_OK) return rc;
    if (lm && ((rc = check_align(io.SS, "SS_sel")) != LMPC_OK || (rc = check_align(io.Qfun, "Qfun_sel")) != LMPC_OK)) return rc;
    CK(cudaSetDevice(h->device));
    // no warm-start records: caller-supplied QPs start cold; the controllers of the device-resident step carry warm-start
    // records (step_dev_impl)
    FtocpArgs a = qp_args(h, io, lm);
    a.abc_inst_stride = abc_inst_stride; a.abc_stage_stride = abc_stage_stride;
    a.retire = retire;
    return launch(h, a, lm, h->stream);
}

extern "C" {

int lmpc_solve_lmpc_dev(lmpc_handle* h, const double* x0, const double* uOld, const double* abc, long long abc_inst_stride,
                        long long abc_stage_stride, const double* SS_sel, const double* Qfun_sel, const double* Succ_SS,
                        const double* Succ_uSS, double* xPred, double* uPred, double* slack, double* lambd,
                        double* slackTerminal, double* zt, double* zt_u, int* status, int* iters, double* resid) {
    if (h && h->shp.tab) return fail(LMPC_E_STATE, "lmpc_solve_*: per-controller shapes are installed; the caller's arrays have no per-controller shape");
    return solve_dev(h, CALLER_QP_IO, abc_inst_stride, abc_stage_stride, LapBudget{});
}

int lmpc_solve_mpc_dev(lmpc_handle* h, const double* x0, const double* uOld, const double* abc, long long abc_inst_stride,
                       long long abc_stage_stride, double* xPred, double* uPred, double* slack, int* status, int* iters,
                       double* resid) {
    return lmpc_solve_lmpc_dev(h, x0, uOld, abc, abc_inst_stride, abc_stage_stride, nullptr, nullptr, nullptr, nullptr, xPred,
                               uPred, slack, nullptr, nullptr, nullptr, nullptr, status, iters, resid);
}

}  // extern "C" (the helpers below have C++ linkage)

// Enqueue one host-buffer solve of the caller's arrays io on buffer set / stream group `slot` (0 .. LMPC_HOST_SLOTS - 1)
// WITHOUT waiting for it.
static int enqueue_host_solve_impl(lmpc_handle* h, int slot, const QpIo& io, long long abc_inst_stride, long long abc_stage_stride) {
    if (!h || !io.x0 || !io.uOld || !io.abc || !io.xPred || !io.uPred || !io.status || !io.iters || !io.resid)
        return fail(LMPC_E_INVALID, "null argument");
    const bool lm = (io.SS != nullptr);
    if (lm && (h->M <= 0 || !io.Qfun)) return fail(LMPC_E_INVALID, "handle was created without a safe set (numSS_Points == 0)");
    if (slot < 0 || slot >= LMPC_HOST_SLOTS) return fail(LMPC_E_INVALID, "slot must be 0 .. 3");
    if (h->shp.tab) return fail(LMPC_E_STATE, "lmpc_solve_*: per-controller shapes are installed; the caller's arrays have no per-controller shape");
    CK(cudaSetDevice(h->device));
    const size_t B = h->batch, N = h->N, M = h->M > 0 ? h->M : 1;
    const size_t D = sizeof(double);
    const QpIo* q = qp_bufs(h, slot);
    if (!q) return LMPC_E_CUDA;
    const QpIo& hb = *q;
    cudaStream_t* cs = h->cstream + 4 * slot;
    long long dis, dss;
    bool per_inst = false;
    if (abc_inst_stride == 0 && abc_stage_stride == 0) { dis = 0; dss = 0; }                       // one shared LTI model
    else if (abc_inst_stride == (long long)N * 54 && abc_stage_stride == 54) { dis = N * 54; dss = 54; per_inst = true; }
    else if (abc_inst_stride == 0 && abc_stage_stride == 54) { dis = 0; dss = 54; }                // one shared LTV model
    else return fail(LMPC_E_INVALID, "host entry supports abc strides (N*54,54), (0,54) or (0,0)");
    CK(cudaStreamSynchronize(h->stream));    // earlier work of this handle is done before the chunk streams start
    if (!per_inst) {
        CK(cudaMemcpyAsync(hb.abc, io.abc, (dss ? N * 54 : 54) * D, cudaMemcpyHostToDevice, cs[0]));
        CK(cudaStreamSynchronize(cs[0]));
    }
    // Chunk pipeline: the batch is cut into up to four instance ranges, each on its own stream, so that the H2D copy
    // of range i+1, the solve of range i and the D2H copy of range i-1 overlap (PCIe is full duplex).
    // A batch enqueued through the asynchronous entry points shares the device with the batches of the other buffer sets: that
    // overlap is already there, every further piece is ten more driver calls on the enqueueing thread and one more under-filled
    // last wave.  Measured on configs[1] (4096 QPs, three sets in flight, two hosts) with tools/e2e_probe.py, which A/B'd the
    // policies through an environment override that has since been removed: 8.8-9.6 M solves/s uncut, 8.7-9.6 M in two pieces,
    // 8.2-8.6 M in four; a lone synchronous batch: 3.1 M uncut, 3.7 M in two, 3.9 M in four.
    bool others = false;
    for (int sl = 0; sl < LMPC_HOST_SLOTS; ++sl) others |= (sl != slot && h->hb_pending[sl]);
    const bool lone = h->hb_lone && !others;
    const int nchunk = B >= 2048 ? (lone ? 4 : (others ? 1 : 2)) : (B >= 512 ? (others ? 1 : 2) : 1);
    // what moves: the fields the caller passes (zt and zt_u are only computed with their successor points) and, per chunk, abc
    // only when every instance has its own model
    QpIo c = io, dev = hb;
    if (!c.SuccSS) c.zt = nullptr;
    if (!c.SuccU) c.ztu = nullptr;
    for (const QpField& f : QP_FIELDS) if (!f.at(c)) f.at(dev) = nullptr;
    FtocpArgs all = qp_args(h, dev, lm);
    all.abc_inst_stride = dis; all.abc_stage_stride = dss;
    if (!per_inst) c.abc = nullptr;
    for (int ci = 0; ci < nchunk; ++ci) {
        const size_t lo = B * ci / nchunk, hi = B * (ci + 1) / nchunk, nb = hi - lo;
        cudaStream_t s = cs[ci];
        for (const QpField& f : QP_FIELDS)
            if (f.in && f.at(c) && (lm || !f.lmpc_only)) {
                const size_t n = f.count(N, M) * f.elem;
                CK(cudaMemcpyAsync((char*)f.at(hb) + lo * n, (const char*)f.at(c) + lo * n, nb * n, cudaMemcpyHostToDevice, s));
            }
        int rc = launch(h, all.range((int)lo, (int)nb, (int)N, h->M), lm, s);
        if (rc != LMPC_OK) return rc;
        for (const QpField& f : QP_FIELDS)
            if (!f.in && f.at(c) && (lm || !f.lmpc_only)) {
                const size_t n = f.count(N, M) * f.elem;
                CK(cudaMemcpyAsync((char*)f.at(c) + lo * n, (const char*)f.at(hb) + lo * n, nb * n, cudaMemcpyDeviceToHost, s));
            }
    }
    h->hb_chunks[slot] = nchunk;
    h->hb_pending[slot] = true;
    return LMPC_OK;
}

// Enqueue one host-buffer solve; on ANY failure part-way through, the chunks already enqueued are still copying into the
// caller's arrays, so their streams are drained before the error is reported.
static int enqueue_host_solve(lmpc_handle* h, int slot, const QpIo& io, long long abc_inst_stride, long long abc_stage_stride) {
    const int rc = enqueue_host_solve_impl(h, slot, io, abc_inst_stride, abc_stage_stride);
    if (rc != LMPC_OK && h && slot >= 0 && slot < LMPC_HOST_SLOTS) {
        const std::string msg = g_err;
        for (int i = 0; i < 4; ++i) cudaStreamSynchronize(h->cstream[4 * slot + i]);
        g_err = msg;
    }
    return rc;
}

extern "C" {

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
    return LMPC_OK;
}

int lmpc_solve_lmpc_host_async(lmpc_handle* h, int slot, const double* x0, const double* uOld, const double* abc, long long abc_inst_stride,
                               long long abc_stage_stride, const double* SS_sel, const double* Qfun_sel, const double* Succ_SS,
                               const double* Succ_uSS, double* xPred, double* uPred, double* slack, double* lambd,
                               double* slackTerminal, double* zt, double* zt_u, int* status, int* iters, double* resid) {
    return enqueue_host_solve(h, slot, CALLER_QP_IO, abc_inst_stride, abc_stage_stride);
}

int lmpc_solve_mpc_host_async(lmpc_handle* h, int slot, const double* x0, const double* uOld, const double* abc, long long abc_inst_stride,
                              long long abc_stage_stride, double* xPred, double* uPred, double* slack, int* status, int* iters,
                              double* resid) {
    return lmpc_solve_lmpc_host_async(h, slot, x0, uOld, abc, abc_inst_stride, abc_stage_stride, nullptr, nullptr, nullptr, nullptr,
                                      xPred, uPred, slack, nullptr, nullptr, nullptr, nullptr, status, iters, resid);
}

int lmpc_solve_lmpc_host(lmpc_handle* h, const double* x0, const double* uOld, const double* abc, long long abc_inst_stride,
                         long long abc_stage_stride, const double* SS_sel, const double* Qfun_sel, const double* Succ_SS,
                         const double* Succ_uSS, double* xPred, double* uPred, double* slack, double* lambd,
                         double* slackTerminal, double* zt, double* zt_u, int* status, int* iters, double* resid) {
    if (h) h->hb_lone = true;
    int rc = enqueue_host_solve(h, 0, CALLER_QP_IO, abc_inst_stride, abc_stage_stride);
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
int lmpc_sizeof_noise_params(void) { return (int)sizeof(lmpc_noise_params); }
int lmpc_sizeof_measurement_params(void) { return (int)sizeof(lmpc_measurement_params); }
int lmpc_sizeof_observer_params(void) { return (int)sizeof(lmpc_observer_params); }
int lmpc_sizeof_observer_prior_params(void) { return (int)sizeof(lmpc_observer_prior_params); }
int lmpc_sizeof_observer_gain_params(void) { return (int)sizeof(lmpc_observer_gain_params); }
int lmpc_sizeof_regression_params(void) { return (int)sizeof(lmpc_regression_params); }
int lmpc_sizeof_shape_params(void) { return (int)sizeof(lmpc_shape_params); }
int lmpc_sizeof_ss_laps_params(void) { return (int)sizeof(lmpc_ss_laps_params); }
int lmpc_sizeof_lap_window_params(void) { return (int)sizeof(lmpc_lap_window_params); }
int lmpc_sizeof_lane_rule_params(void) { return (int)sizeof(lmpc_lane_rule_params); }
int lmpc_sizeof_lane_margin_params(void) { return (int)sizeof(lmpc_lane_margin_params); }
int lmpc_sizeof_prediction_model_params(void) { return (int)sizeof(lmpc_prediction_model_params); }
int lmpc_sizeof_surface_params(void) { return (int)sizeof(lmpc_surface_params); }
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
    // the largest launch: trToUse = K1_MAXLAPS at K1_MAXWPB warps (103360 B, above a flat 100 KiB)
    for (auto k1 : {knn_ltv_regress_kernel<false, false>, knn_ltv_regress_kernel<true, false>, knn_ltv_regress_kernel<false, true>,
                    knn_ltv_regress_kernel<true, true>}) {
        CK(cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k1_smem_bytes(K1_MAXLAPS, K1_MAXWPB)));
        CK(cudaFuncSetAttribute(k1, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    }
    ModelConst& m = h->mc;
    memset(&m, 0, sizeof(m));
    m.trToUse = mp->trToUse; m.dt = mp->dt;
    RegressionRec& r = h->store_reg;
    memset(&r, 0, sizeof(r));
    r.trToUse = mp->trToUse; r.MaxNumPoint = mp->MaxNumPoint; r.h = mp->h; r.lamb = mp->lamb;
    // |(x - q) s| == |(x - q) |s|| bit for bit, and the fp32 scan of K1 needs non-negative partial distances to order its keys
    for (int i = 0; i < 5; ++i) r.scaling[i] = fabs(mp->scaling[i]);
    TrackRec& t = h->store_trk;
    memset(&t, 0, sizeof(t));
    t.nseg = mp->nseg;
    for (int i = 0; i < mp->nseg * 3; ++i) t.seg[i] = mp->seg[i];
    t.TrackLength = mp->TrackLength;
    int rc = swap_table(h, "lmpc_store_create", h->trk, &t, 1, nullptr);
    if (rc != LMPC_OK) return rc;
    if ((rc = swap_table(h, "lmpc_store_create", h->reg, &r, 1, nullptr)) != LMPC_OK) return rc;
    h->laps_stored = false;
    h->ss.cap = ss_cap > 0 ? ss_cap : 1; h->ss.Tmax = Tmax;
    h->mdl.cap = model_cap; h->mdl.Tmax = Tmax; h->mdl.q = nullptr;
    LapBooks& k = h->bk;
    k.ss_cap = h->ss.cap; k.md_cap = model_cap; k.numSS_it = h->p.numSS_it > 0 ? h->p.numSS_it : 1; k.trToUse = mp->trToUse;
    if (h->p.warm_start) {          // SURVEY §8f rank 2: per-controller interior-point snapshot for the next solve
        const long long N = h->N, Mx = h->M > 0 ? h->M : 0;
        h->warm_stride = N * 2 + 4 * N * h->p.ncx + N * h->p.ncu + 2 * Mx + 2;
        h->warm_mode = -1;
    }
    if ((rc = alloc_bufs(h, dev_bufs(h), OWN_STORE | (h->p.warm_start ? OWN_WARM : 0), h->batch, "lmpc_store_create")) != LMPC_OK)
        return rc;
    k.sel = h->d_sel; k.isprev = h->d_isprev; k.prevslot = h->d_prevslot; k.used = h->d_used;
    h->has_store = true;
    return LMPC_OK;
}
extern "C" {

// The preconditions of an entry point, one line each: the handle has a store (need_store) or a store and a rollout
// (need_rollout); both then select the handle's device.  The lap books are part of the store.
static int need_store(lmpc_handle* h) {
    if (!h) return fail(LMPC_E_INVALID, "null handle");
    if (!h->has_store) return fail(LMPC_E_STATE, "call lmpc_store_create first");
    CK(cudaSetDevice(h->device));
    return LMPC_OK;
}

// The host-chosen exchange (lmpc_ss_import_laps_dev) hands laps between any controllers: only when they all drive one circuit
static int one_track(const lmpc_handle* h, const char* who) {
    if (h->trk.rows.size() > 1)
        return fail(LMPC_E_STATE, std::string(who) + ": more than one track installed; a lap of another circuit is not a trajectory of this one");
    return LMPC_OK;
}

// The pooled exchange hands laps only within a pool group: with several tracks installed, every group must drive one circuit
static int one_track_per_group(const lmpc_handle* h, const char* who) {
    if (h->trk.rows.size() <= 1) return LMPC_OK;
    if (h->ngroups == 0)
        return fail(LMPC_E_STATE, std::string(who) + ": more than one track installed and no pool groups; a lap of another circuit is "
                                                     "not a trajectory of this one");
    std::vector<int> trk(h->ngroups, -1);
    for (int b = 0; b < h->batch; ++b) {
        int& t = trk[h->pool_grp.index[b]];
        if (t >= 0 && t != h->trk.index[b])
            return fail(LMPC_E_STATE, std::string(who) + ": pool group " + std::to_string(h->pool_grp.index[b]) + " spans two tracks");
        t = h->trk.index[b];
    }
    return LMPC_OK;
}

// A latest own lap is exported only once it has `rows` rows past its finish line; 0 exports any.
int lmpc_set_pool_min_overrun(lmpc_handle* h, int rows) {
    if (!h) return fail(LMPC_E_INVALID, "null handle");
    if (rows < 0) return fail(LMPC_E_INVALID, "lmpc_set_pool_min_overrun: rows must be >= 0");
    h->pool_min_over = rows;
    return LMPC_OK;
}

// Pool groups: controller b exchanges laps only with the controllers of group group_of_instance[b].  Nothing about the handle
// changes unless every check passes; regrouping affects the exchanges that follow, not the laps already filed.
int lmpc_set_pool_groups(lmpc_handle* h, int ngroups, const int* group_of_instance) {
    static const char* who = "lmpc_set_pool_groups";
    int rc = need_store(h);
    if (rc) return rc;
    if (ngroups > LMPC_MAX_POOL_GROUPS) return fail(LMPC_E_INVALID, std::string(who) + ": ngroups above LMPC_MAX_POOL_GROUPS");
    // the index rules of the per-controller tables; there are no rows, so the index stands in for them
    if ((rc = check_set_index(h, who, ngroups ? group_of_instance : nullptr, ngroups, group_of_instance)) != LMPC_OK) return rc;
    if ((rc = swap_table<int>(h, who, h->pool_grp, nullptr, 0, group_of_instance)) != LMPC_OK) return rc;
    h->ngroups = ngroups;
    return LMPC_OK;
}

// Per-controller tracks: every set is checked the way Track.py:54-133 builds the table (start i = start i-1 + length i-1 and
// TrackLength = start + length of the last row, exactly); nsets == 0 returns to the track of lmpc_store_create.
int lmpc_set_tracks(lmpc_handle* h, const lmpc_track_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_set_tracks";
    int rc = need_store(h);
    if (rc) return rc;
    if (h->laps_stored) return fail(LMPC_E_STATE, std::string(who) + ": laps are stored already; install tracks before the first lap");
    return install_table(h, who, h->trk, sets, nsets, set_of_instance, &h->store_trk, [&](int k, TrackRec& row) {
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
        // canonical row: padding and the entries past nseg are zero, so a record's track row is the circuit alone
        memset(&row, 0, sizeof(TrackRec));
        row.nseg = t.nseg;
        for (int i = 0; i < t.nseg * 3; ++i) row.seg[i] = t.seg[i];
        row.TrackLength = t.TrackLength;
        return LMPC_OK;
    });
}

// Per-controller regression constants: every set checked (the scaling range is the one K1's fp32 pre-filter is certified for:
// safeset.cuh, above its threshold); nsets == 0 returns to the constants of lmpc_store_create.
int lmpc_set_regression_sets(lmpc_handle* h, const lmpc_regression_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_set_regression_sets";
    int rc = need_store(h);
    if (rc) return rc;
    return install_table(h, who, h->reg, sets, nsets, set_of_instance, &h->store_reg, [&](int k, RegressionRec& r) {
        const lmpc_regression_params& s = sets[k];
        const std::string w = std::string(who) + ": set " + std::to_string(k) + ": ";
        if (s.trToUse < 1 || s.trToUse > h->mc.trToUse)
            return fail(LMPC_E_INVALID, w + "trToUse must be 1 .. the store's trToUse (" + std::to_string(h->mc.trToUse) + ")");
        if (s.MaxNumPoint < 1 || s.MaxNumPoint > K1_MAXPTS) return fail(LMPC_E_INVALID, w + "MaxNumPoint must be 1 .. 7");
        if (!(s.h >= 0x1p-1022 && s.h <= 0x1p1022)) return fail(LMPC_E_INVALID, w + "h must be finite and in [2^-1022, 2^1022]");
        if (!(isfinite(s.lamb) && s.lamb >= 0.0)) return fail(LMPC_E_INVALID, w + "lamb must be finite and >= 0");
        memset(&r, 0, sizeof(r));
        r.trToUse = s.trToUse; r.MaxNumPoint = s.MaxNumPoint; r.h = s.h; r.lamb = s.lamb;
        for (int i = 0; i < 5; ++i) {
            const double a = fabs(s.scaling[i]);
            if (!(a == 0.0 || (a >= 0x1p-32 && a <= 0x1p32)))
                return fail(LMPC_E_INVALID, w + "every |scaling| must be 0 or in [2^-32, 2^32]");
            r.scaling[i] = a;
        }
        return LMPC_OK;
    });
}

// Per-controller prediction models: mode 0, 1 or 2, all ten vehicle values finite, and m, lf, lr, Iz positive in a mode 1 row;
// nsets == 0 removes the table.
int lmpc_set_prediction_models(lmpc_handle* h, const lmpc_prediction_model_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_set_prediction_models";
    int rc = need_store(h);
    if (rc) return rc;
    return install_table(h, who, h->pmod, sets, nsets, set_of_instance, (const PredictionModelRec*)nullptr, [&](int k, PredictionModelRec& r) {
        const lmpc_prediction_model_params& s = sets[k];
        const lmpc_vehicle_params& v = s.vehicle;
        const std::string w = std::string(who) + ": row " + std::to_string(k) + ": ";
        if (s.mode < 0 || s.mode > 2) return fail(LMPC_E_INVALID, w + "mode must be 0, 1 or 2");
        const double all[10] = {v.m, v.lf, v.lr, v.Iz, v.Df, v.Cf, v.Bf, v.Dr, v.Cr, v.Br};
        for (double x : all)
            if (!isfinite(x)) return fail(LMPC_E_INVALID, w + "all ten vehicle values must be finite");
        if (s.mode == 1 && !(v.m > 0 && v.lf > 0 && v.lr > 0 && v.Iz > 0))
            return fail(LMPC_E_INVALID, w + "a mode 1 vehicle needs m, lf, lr, Iz > 0");
        memset(&r, 0, sizeof(r));
        r.mode = s.mode;
        r.vehicle = v;
        return LMPC_OK;
    });
}

static bool on_grid(int N, int M) {
#define GCASE(n, m) if (N == n && M == m) return true;
    LMPC_FOR_EACH_CASE(GCASE)
#undef GCASE
    return false;
}

// numSS_it / numSS_Points of controller b: its row of the lap-count / shape table, or the handle's
static int laps_of(const lmpc_handle* h, int b) { return h->ssl.tab ? h->ssl.rows[h->ssl.index[b]].numSS_it : h->p.numSS_it; }
// ss_window of controller b: its row of the lap-window table, or 0 (unbounded)
static int ss_window_of(const lmpc_handle* h, int b) { return h->lwin.tab ? h->lwin.rows[h->lwin.index[b]].ss_window : 0; }
static int points_of(const lmpc_handle* h, int b) { return h->shp.tab ? h->shp.rows[h->shp.index[b]].numSS_Points : h->M; }
// M points split into nit laps of an even number of points each (PC.py:403,492-495)
static bool even_split(int M, int nit) { return M % nit == 0 && (M / nit) % 2 == 0; }

// Per-controller shapes: every set checked against the grid and the handle, the shaped kernels of every set opted into their
// shared-memory size, then the table and the sorted instance list (DESIGN.md, "Per-controller horizons and safe-set sizes");
// nsets == 0 returns to the handle's own shape.
int lmpc_set_shapes(lmpc_handle* h, const lmpc_shape_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_set_shapes";
    int rc = need_store(h);
    if (rc) return rc;
    if (h->laps_stored) return fail(LMPC_E_STATE, std::string(who) + ": laps are stored already; install shapes before the first lap");
    if (h->p.warm_start) return fail(LMPC_E_STATE, std::string(who) + ": the handle was created with warm_start; its records are laid out per (N, M)");
    const int nit = h->p.numSS_it;
    if (h->ssl.tab) {                   // every controller's numSS_Points against its own numSS_it (lmpc_set_ss_laps)
        if ((rc = check_set_index(h, who, sets, nsets, set_of_instance)) != LMPC_OK) return rc;
        for (int b = 0; b < h->batch; ++b) {
            const int m = nsets ? sets[set_of_instance[b]].numSS_Points : h->M;
            if (!even_split(m, laps_of(h, b)))
                return fail(LMPC_E_INVALID, std::string(who) + ": controller " + std::to_string(b) + ": numSS_Points " + std::to_string(m) +
                                                " is not its numSS_it (" + std::to_string(laps_of(h, b)) + ") times an even number of points per lap");
        }
    }
    rc = install_table(h, who, h->shp, sets, nsets, set_of_instance, (const ShapeRec*)nullptr, [&](int k, ShapeRec& row) {
        const lmpc_shape_params& s = sets[k];
        const std::string w = std::string(who) + ": set " + std::to_string(k) + ": ";
        if (!on_grid(s.N, s.numSS_Points)) return fail(LMPC_E_INVALID, w + "(N, numSS_Points) is not instantiated: built for " LMPC_GRID_TEXT);
        if (s.N > h->N || s.numSS_Points > h->M)
            return fail(LMPC_E_INVALID, w + "N and numSS_Points must not exceed the handle's (" + std::to_string(h->N) + ", " +
                                            std::to_string(h->M) + ")");
        if ((s.numSS_Points > 0) != (h->M > 0)) return fail(LMPC_E_INVALID, w + "numSS_Points must be > 0 exactly when the handle's is");
        if (!h->ssl.tab && s.numSS_Points > 0 && !even_split(s.numSS_Points, nit))
            return fail(LMPC_E_INVALID, w + "numSS_Points must be a multiple of numSS_it with an even number of points per lap");
        const cudaError_t e = ftocp_shaped_configure(s.N, s.numSS_Points);
        if (e != cudaSuccess) return fail(LMPC_E_CUDA, w + cudaGetErrorString(e));
        row = s;
        return LMPC_OK;
    });
    if (rc != LMPC_OK) return rc;
    // the batch sorted by (N, M) and the runs of one shape in it
    std::vector<int> order(nsets ? h->batch : 0);
    for (size_t b = 0; b < order.size(); ++b) order[b] = (int)b;
    auto key = [&](int b) { const ShapeRec& r = h->shp.rows[h->shp.index[b]]; return std::make_pair(r.N, r.numSS_Points); };
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return key(x) < key(y); });
    h->shp_cells.clear();
    for (size_t i = 0; i < order.size(); ++i) {
        const auto k = key(order[i]);
        if (i == 0 || k != key(order[i - 1])) h->shp_cells.push_back({k.first, k.second, (int)i, 0});
        h->shp_cells.back().n += 1;
    }
    if ((rc = swap_table<int>(h, who, h->shp_order, nullptr, 0, nsets ? order.data() : nullptr)) != LMPC_OK) {
        const std::string msg = g_err;      // no shapes rather than shapes without their instance list
        swap_table<ShapeRec>(h, who, h->shp, nullptr, 0, nullptr);
        h->shp_cells.clear();
        g_err = msg;
    }
    return rc;
}

// Per-controller safe-set lap counts: every set checked against the handle, every controller's numSS_Points against its value,
// then the table (DESIGN.md, "Per-controller safe-set lap counts"); nsets == 0 returns to the handle's numSS_it.
int lmpc_set_ss_laps(lmpc_handle* h, const lmpc_ss_laps_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_set_ss_laps";
    int rc = need_store(h);
    if (rc) return rc;
    if (h->laps_stored) return fail(LMPC_E_STATE, std::string(who) + ": laps are stored already; install lap counts before the first lap");
    if (h->M <= 0) return fail(LMPC_E_INVALID, std::string(who) + ": the handle has no safe set (numSS_Points == 0)");
    if ((rc = check_set_index(h, who, sets, nsets, set_of_instance)) != LMPC_OK) return rc;
    const int nit = h->p.numSS_it;
    for (int k = 0; k < nsets; ++k)
        if (sets[k].numSS_it < 1 || sets[k].numSS_it > nit)
            return fail(LMPC_E_INVALID, std::string(who) + ": set " + std::to_string(k) + ": numSS_it must be 1 .. the handle's " +
                                            std::to_string(nit));
    for (int b = 0; b < h->batch; ++b) {       // nsets == 0: the handle's numSS_it against the installed shapes and windows
        const int v = nsets ? sets[set_of_instance[b]].numSS_it : nit;
        if (!even_split(points_of(h, b), v))
            return fail(LMPC_E_INVALID, std::string(who) + ": controller " + std::to_string(b) + ": its numSS_Points " +
                                            std::to_string(points_of(h, b)) + " is not numSS_it (" + std::to_string(v) +
                                            ") times an even number of points per lap");
        if (ss_window_of(h, b) > 0 && v > ss_window_of(h, b))
            return fail(LMPC_E_INVALID, std::string(who) + ": controller " + std::to_string(b) + ": numSS_it " + std::to_string(v) +
                                            " exceeds its ss_window (" + std::to_string(ss_window_of(h, b)) + ")");
    }
    return install_table(h, who, h->ssl, sets, nsets, set_of_instance, (const SsLapsRec*)nullptr, [&](int k, SsLapsRec& row) {
        row = sets[k];
        return LMPC_OK;
    });
}

// Per-controller lap windows: every set checked against the store and every controller's numSS_it, then the table (DESIGN.md,
// "Per-controller lap windows"); nsets == 0 removes it.
int lmpc_set_lap_windows(lmpc_handle* h, const lmpc_lap_window_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_set_lap_windows";
    int rc = need_store(h);
    if (rc) return rc;
    if (h->laps_stored) return fail(LMPC_E_STATE, std::string(who) + ": laps are stored already; install lap windows before the first lap");
    if ((rc = check_set_index(h, who, sets, nsets, set_of_instance)) != LMPC_OK) return rc;
    for (int b = 0; b < (nsets ? h->batch : 0); ++b) {    // the safe-set window against the controller's own numSS_it
        const int w = sets[set_of_instance[b]].ss_window;
        if (w > 0 && w < laps_of(h, b))
            return fail(LMPC_E_INVALID, std::string(who) + ": controller " + std::to_string(b) + ": ss_window " + std::to_string(w) +
                                            " is below its numSS_it (" + std::to_string(laps_of(h, b)) + ")");
    }
    return install_table(h, who, h->lwin, sets, nsets, set_of_instance, (const LapWindowRec*)nullptr, [&](int k, LapWindowRec& row) {
        const lmpc_lap_window_params& s = sets[k];
        const std::string w = std::string(who) + ": set " + std::to_string(k) + ": ";
        if (s.ss_window != 0 && h->M <= 0) return fail(LMPC_E_INVALID, w + "ss_window must be 0: the handle has no safe set (numSS_Points == 0)");
        if (s.ss_window < 0 || s.ss_window > h->ss.cap)
            return fail(LMPC_E_INVALID, w + "ss_window must be 0 or numSS_it .. ss_cap (" + std::to_string(h->ss.cap) + ")");
        if (s.model_window != 0 && (s.model_window < h->mc.trToUse || s.model_window > h->mdl.cap))
            return fail(LMPC_E_INVALID, w + "model_window must be 0 or trToUse (" + std::to_string(h->mc.trToUse) + ") .. model_cap (" +
                                            std::to_string(h->mdl.cap) + ")");
        row = s;
        return LMPC_OK;
    });
}

// Per-controller lane rules: every set checked, then the table (DESIGN.md, "Lane-safe safe sets"); nsets == 0 removes it.
int lmpc_set_lane_rules(lmpc_handle* h, const lmpc_lane_rule_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_set_lane_rules";
    int rc = need_store(h);
    if (rc) return rc;
    if (h->M <= 0) return fail(LMPC_E_STATE, std::string(who) + ": the handle has no safe set (numSS_Points == 0)");
    if (h->laps_stored) return fail(LMPC_E_STATE, std::string(who) + ": laps are stored already; install lane rules before the first lap");
    return install_table(h, who, h->lrule, sets, nsets, set_of_instance, (const LaneRuleRec*)nullptr, [&](int k, LaneRuleRec& row) {
        const lmpc_lane_rule_params& s = sets[k];
        const std::string w = std::string(who) + ": set " + std::to_string(k) + ": ";
        if (s.mode != 0 && s.mode != 1) return fail(LMPC_E_INVALID, w + "mode must be 0 or 1");
        if (!isfinite(s.lane_tol) || s.lane_tol < 0.0) return fail(LMPC_E_INVALID, w + "lane_tol must be finite and >= 0");
        if (s.mode == 1 && h->has_rollout && h->Tcl >= LMPC_LANE_UNSAFE_KEY)
            return fail(LMPC_E_INVALID, w + "the rollout's Tcl is not below LMPC_LANE_UNSAFE_KEY");
        row = s;
        row.pad = 0;
        return LMPC_OK;
    });
}

// Per-controller lane margins: every set checked, every controller's margin against the QP row it reads, then the margin buffers
// (allocated with the first table), the table and the planning rows (DESIGN.md, "Lane margins"); nsets == 0 removes them.
int lmpc_set_lane_margins(lmpc_handle* h, const lmpc_lane_margin_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_set_lane_margins";
    int rc = need_store(h);
    if (rc) return rc;
    if ((rc = check_set_index(h, who, sets, nsets, set_of_instance)) != LMPC_OK) return rc;
    for (int b = 0; b < (nsets ? h->batch : 0); ++b) {
        const int k = set_of_instance[b];
        const FtocpConst& c = h->sets.tab ? h->sets.rows[h->sets.index[b]].c : h->c;
        const lmpc_lane_margin_params& r = sets[k];
        if ((r.mode == 1 || r.mode == 2) && isfinite(r.margin0) && isfinite(r.margin_max) && !margin_leaves_lane(r, c))
            return fail(LMPC_E_INVALID, std::string(who) + ": set " + std::to_string(k) + ": the margin of controller " +
                                            std::to_string(b) + " does not leave a lane (" + (r.mode == 1 ? "margin0" : "margin_max") +
                                            " must be below min_i bx_i of its QP row)");
    }
    const bool fresh = nsets > 0 && !h->d_margin;
    if (fresh && (rc = alloc_bufs(h, dev_bufs(h), OWN_MARGIN, h->batch, who)) != LMPC_OK) return rc;
    rc = install_table(h, who, h->lmar, sets, nsets, set_of_instance, (const LaneMarginRec*)nullptr, [&](int k, LaneMarginRec& row) {
        const lmpc_lane_margin_params& s = sets[k];
        const std::string w = std::string(who) + ": set " + std::to_string(k) + ": ";
        if (s.mode < 0 || s.mode > 2) return fail(LMPC_E_INVALID, w + "mode must be 0, 1 or 2");
        for (double v : {s.margin0, s.margin_max, s.step_up, s.step_down})
            if (!isfinite(v) || v < 0.0) return fail(LMPC_E_INVALID, w + "margin0, margin_max, step_up and step_down must be finite and >= 0");
        if (s.margin0 > s.margin_max) return fail(LMPC_E_INVALID, w + "margin0 must not exceed margin_max");
        row = s;
        row.pad = 0;
        return LMPC_OK;
    });
    if (rc != LMPC_OK) {
        if (fresh) free_bufs(dev_bufs(h), OWN_MARGIN);
        return rc;
    }
    if (nsets == 0) free_bufs(dev_bufs(h), OWN_MARGIN);     // swap_table left the streams idle
    if ((rc = lane_margin_rows(h, true)) != LMPC_OK) return rc;
    // a warm-start record belongs to the QP it was taken from
    if (h->d_warm_valid) CK(cudaMemsetAsync(h->d_warm_valid, 0, sizeof(int) * h->batch, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_get_lane_margins(lmpc_handle* h, double* m) {
    if (int rc = need_store(h)) return rc;
    if (!h->lmar.tab) return fail(LMPC_E_STATE, "lmpc_get_lane_margins: no lane-margin table is installed");
    if (!m) return fail(LMPC_E_INVALID, "null output");
    CK(cudaMemcpyAsync(m, h->d_margin, sizeof(double) * h->batch, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

static int put_lap(lmpc_handle* h, LapPool& pool, int inst, int slot, int T, const double* x, const double* u) {
    if (inst < 0 || inst >= h->batch || slot < 0 || slot >= pool.cap || T < 2 || T > pool.Tmax || !x || !u)
        return fail(LMPC_E_INVALID, "put_lap: bad instance/slot/length");
    h->laps_stored = true;
    const size_t lap = pool.lap_index(inst, slot);
    CK(cudaMemcpyAsync(pool.x + lap * pool.Tmax * 6, x, sizeof(double) * T * 6, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(pool.u + lap * pool.Tmax * 2, u, sizeof(double) * T * 2, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(pool.len + lap, &T, sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));   // T lives on the caller's stack
    return LMPC_OK;
}

int lmpc_model_put_lap(lmpc_handle* h, int inst, int slot, int T, const double* x, const double* u) {
    if (int rc = need_store(h)) return rc;
    return put_lap(h, h->mdl, inst, slot, T, x, u);
}

int lmpc_model_set_used(lmpc_handle* h, const int* slots) {
    if (int rc = need_store(h)) return rc;
    if (!slots) return fail(LMPC_E_INVALID, "null slots");
    for (size_t i = 0; i < (size_t)h->batch * h->mc.trToUse; ++i)
        if (slots[i] < 0 || slots[i] >= h->mdl.cap) return fail(LMPC_E_INVALID, "model slot out of range");
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
    if (int rc = need_store(h)) return rc;
    if (!slots || !is_prev || !prev_slot) return fail(LMPC_E_INVALID, "null argument");
    const int nit = h->p.numSS_it;
    for (size_t i = 0; i < (size_t)h->batch * nit; ++i)
        if (slots[i] < 0 || slots[i] >= h->ss.cap) return fail(LMPC_E_INVALID, "safe-set slot out of range");
    for (int b = 0; b < h->batch; ++b)
        if (prev_slot[b] >= h->ss.cap) return fail(LMPC_E_INVALID, "prev_slot out of range");
    CK(cudaMemcpyAsync(h->d_sel, slots, sizeof(int) * h->batch * nit, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_isprev, is_prev, sizeof(int) * h->batch * nit, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_prevslot, prev_slot, sizeof(int) * h->batch, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_ss_add_point(lmpc_handle* h, const double* x, const double* u) {
    if (int rc = need_store(h)) return rc;
    if (!x || !u) return fail(LMPC_E_INVALID, "null argument");
    for (int b = 0; b < h->batch; ++b)       // the kernel would skip such a point and flag 512; the host caller hears of it here
        for (int j = 0; j < 6; ++j)
            if (!isfinite(x[(size_t)b * 6 + j]) || (j < 2 && !isfinite(u[(size_t)b * 2 + j])))
                return fail(LMPC_E_INVALID, "addPoint: non-finite x or u of instance " + std::to_string(b));
    CK(cudaMemcpyAsync(h->d_tmpx, x, sizeof(double) * h->batch * 6, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_tmpu, u, sizeof(double) * h->batch * 2, cudaMemcpyHostToDevice, h->stream));
    ss_add_point_kernel<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(h->batch, h->ss, h->d_prevslot, h->d_tmpx, h->d_tmpu, 2,
                                                                        tracks(h), h->d_flags, h->d_dropped, LapBudget{});
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
    if (int rc = need_store(h)) return rc;
    if (inst < 0 || inst >= h->batch || slot < 0 || slot >= h->ss.cap || !T) return fail(LMPC_E_INVALID, "bad instance/slot");
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
    if (int rc = need_store(h)) return rc;
    if (inst < 0 || inst >= h->batch || slot < 0 || slot >= h->ss.cap || row < 0 || row >= h->ss.Tmax || !x6)
        return fail(LMPC_E_INVALID, "bad patch arguments");
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
    if ((rc = copy_bufs(h, cudaMemcpyHostToDevice, {{h->d_xLin, xLin}, {h->d_uLin, uLin}, {h->d_ztState, zt}, {h->d_OldInput, OldInput},
                                                   {h->d_timeStep, timeStep}, {h->d_hasPred, has_pred}, {h->d_xPredPrev, xPred}})))
        return rc;
    if (h->d_warm_valid) CK(cudaMemsetAsync(h->d_warm_valid, 0, sizeof(int) * h->batch, h->stream));     // a new state starts cold
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_state_get(lmpc_handle* h, double* xLin, double* uLin, double* zt, double* OldInput, int* timeStep) {
    int rc = need_store(h);
    if (rc) return rc;
    if ((rc = copy_bufs(h, cudaMemcpyDeviceToHost, {{h->d_xLin, xLin}, {h->d_uLin, uLin}, {h->d_ztState, zt}, {h->d_OldInput, OldInput},
                                                   {h->d_timeStep, timeStep}})))
        return rc;
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

// K1 for the whole batch, and with a prediction-model table the nominal model after it (nominal_model.cuh).  vsched, ssched: the
// vehicle and surface lap schedules a mode 2 controller follows (lmpc_rollout_step), or none: its vehicle- and surface-table rows.
static int launch_k1(lmpc_handle* h, LapBudget retire = {}, LapSchedule vsched = {}, LapSchedule ssched = {}) {
    K1Args a;
    a.batch = h->batch; a.N = h->N;
    a.wpb = h->N < K1_MAXWPB ? h->N : K1_MAXWPB;
    a.pts_stride = k1_pts_stride(h->mc.trToUse);
    a.xLin = h->d_xLin; a.uLin = h->d_uLin; a.pool = h->mdl; a.used = h->d_used; a.abc = h->hb[0].abc; a.status = h->d_flags;
    a.trk = tracks(h);
    a.reg = h->reg.view();
    a.retire = retire;
    a.shp = h->shp.view();
    a.pm = h->pmod.view();
    dim3 grid(h->batch, (h->N + a.wpb - 1) / a.wpb);
    const size_t smem = k1_smem_bytes(h->mc.trToUse, a.wpb);
    if (!h->pmod.tab) {
        (h->shp.tab ? knn_ltv_regress_kernel<true, false> : knn_ltv_regress_kernel<false, false>)<<<grid, 32 * a.wpb, smem, h->stream>>>(h->mc, a);
    } else {
        (h->shp.tab ? knn_ltv_regress_kernel<true, true> : knn_ltv_regress_kernel<false, true>)<<<grid, 32 * a.wpb, smem, h->stream>>>(h->mc, a);
    }
    CK(cudaGetLastError());
    h->launches += 1;
    if (!h->pmod.tab) return LMPC_OK;
    NominalArgs na;
    na.batch = h->batch; na.N = h->N; na.dt = h->mc.dt; na.xLin = h->d_xLin; na.uLin = h->d_uLin;
    na.pm = h->pmod.view(); na.veh = h->veh.view(); na.veh_s = vsched; na.trk = tracks(h); na.retire = retire; na.shp = h->shp.view();
    na.abc = h->hb[0].abc; na.status = h->d_flags;
    na.surf = h->surf.view(); na.surf_s = ssched;
    const long long nthr = (long long)h->batch * h->N;
    (h->surf.tab ? nominal_model_kernel<true> : nominal_model_kernel<false>)<<<(unsigned)((nthr + 127) / 128), 128, 0, h->stream>>>(na);
    CK(cudaGetLastError());
    h->launches += 1;
    return LMPC_OK;
}

static int launch_k2(lmpc_handle* h, const double* d_x0, LapBudget retire = {}) {
    K2Args a;
    a.batch = h->batch; a.N = h->N; a.numSS_it = h->p.numSS_it; a.P = h->M / h->p.numSS_it;
    a.trk = tracks(h);
    a.x0 = d_x0; a.zt = h->d_ztState; a.pool = h->ss; a.sel = h->d_sel; a.is_prev = h->d_isprev;
    a.timeStep = h->d_timeStep; a.has_pred = h->d_hasPred; a.xPred = h->d_xPredPrev;
    a.SS_sel = h->hb[0].SS; a.Qfun_sel = h->hb[0].Qfun; a.Succ_SS = h->hb[0].SuccSS; a.Succ_uSS = h->hb[0].SuccU;
    a.zt_fixed = h->d_ztFixed; a.status = h->d_flags; a.min_index = h->d_minidx;
    a.retire = retire;
    a.shp = h->shp.view();
    a.laps = h->ssl.view();
    (h->shp.tab || h->ssl.tab ? ss_select_kernel<true> : ss_select_kernel<false>)<<<h->batch, 32 * a.numSS_it, 0, h->stream>>>(a);
    CK(cudaGetLastError());
    h->launches += 1;
    return LMPC_OK;
}

int lmpc_identify_host(lmpc_handle* h, double* abc_out, int* flags) {
    int rc = need_store(h);
    if (rc) return rc;
    CK(cudaMemsetAsync(h->d_flags, 0, sizeof(int) * h->batch, h->stream));
    rc = launch_k1(h);
    if (rc) return rc;
    QpIo out = {};
    out.abc = abc_out;
    if ((rc = copy_out(h, out, false)) != LMPC_OK) return rc;
    if (flags) CK(cudaMemcpyAsync(flags, h->d_flags, sizeof(int) * h->batch, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_select_host(lmpc_handle* h, const double* x0, double* SS_sel, double* Qfun_sel, double* Succ_SS, double* Succ_uSS,
                     int* min_index, int* flags) {
    int rc = need_store(h);
    if (rc) return rc;
    if (h->M <= 0 || !x0) return fail(LMPC_E_INVALID, "handle has no safe set or x0 is null");
    const size_t B = h->batch;
    cudaStream_t s = h->stream;
    CK(cudaMemcpyAsync(h->hb[0].x0, x0, B * 6 * sizeof(double), cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(h->d_flags, 0, sizeof(int) * B, s));
    rc = launch_k2(h, h->hb[0].x0);
    if (rc) return rc;
    QpIo out = {};
    out.SS = SS_sel; out.Qfun = Qfun_sel; out.SuccSS = Succ_SS; out.SuccU = Succ_uSS;
    if ((rc = copy_out(h, out, true)) != LMPC_OK) return rc;
    if (min_index) CK(cudaMemcpyAsync(min_index, h->d_minidx, B * h->p.numSS_it * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (flags) CK(cudaMemcpyAsync(flags, h->d_flags, B * sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return LMPC_OK;
}

}  // extern "C"

// One device-resident step for the whole batch on the handle's stream: K1 -> K2 -> QP -> shift (PC.py:110-137).  ev (five events
// or null) brackets the four kernels for lmpc_step_profile.  retire: the lap budgets (the closed loop) or none; vsched, ssched: the
// vehicle and surface lap schedules a mode 2 prediction model follows (the closed loop) or none.
// flags_cleared: the caller cleared the step flags before a kernel of its own set some (the state observer), so they stay.
static int step_dev_impl(lmpc_handle* h, int mode, const double* x0_dev, cudaEvent_t* ev, LapBudget retire = {},
                         LapSchedule vsched = {}, LapSchedule ssched = {}, bool flags_cleared = false) {
    int rc = need_store(h);
    if (rc) return rc;
    if (!x0_dev || (mode != 0 && mode != 1)) return fail(LMPC_E_INVALID, "bad mode or null x0");
    if (mode == 1 && h->M <= 0) return fail(LMPC_E_INVALID, "LMPC step on a handle without a safe set");
    cudaStream_t st = h->stream;
    if (!flags_cleared) CK(cudaMemsetAsync(h->d_flags, 0, sizeof(int) * h->batch, st));
    if (h->d_warm && h->warm_mode != mode) {             // records of the other problem type are not comparable
        CK(cudaMemsetAsync(h->d_warm_valid, 0, sizeof(int) * h->batch, st));
        h->warm_mode = mode;
    }
    const bool lm = mode == 1;
    const QpIo& q = h->hb[0];
    if (ev) CK(cudaEventRecord(ev[0], st));
    if ((rc = launch_k1(h, retire, vsched, ssched)) != LMPC_OK) return rc;                   // PC.py:117
    if (ev) CK(cudaEventRecord(ev[1], st));
    if (lm && (rc = launch_k2(h, x0_dev, retire)) != LMPC_OK) return rc;             // PC.py:121
    if (ev) CK(cudaEventRecord(ev[2], st));
    FtocpArgs a = qp_args(h, q, lm);                                         // PC.py:124-125
    a.x0 = x0_dev; a.uOld = h->d_OldInput;
    if (h->d_warm) { a.warm = h->d_warm; a.warm_valid = h->d_warm_valid; a.warm_stride = h->warm_stride; }
    a.retire = retire;
    if ((rc = launch(h, a, lm, st)) != LMPC_OK) return rc;
    if (ev) CK(cudaEventRecord(ev[3], st));
    ShiftArgs sa;
    sa.batch = h->batch; sa.N = h->N; sa.lmpc = mode;
    sa.xPred = q.xPred; sa.uPred = q.uPred; sa.zt_in = q.zt; sa.ztu_in = q.ztu;
    sa.xLin = h->d_xLin; sa.uLin = h->d_uLin; sa.zt = h->d_ztState; sa.OldInput = h->d_OldInput; sa.xPredPrev = h->d_xPredPrev;
    sa.timeStep = h->d_timeStep; sa.has_pred = h->d_hasPred;
    sa.retire = retire;
    sa.shp = h->shp.view();
    (h->shp.tab ? shift_state_kernel<true> : shift_state_kernel<false>)<<<h->batch, 64, 0, st>>>(sa);   // PC.py:129-137
    CK(cudaGetLastError());
    h->launches += 1;
    if (ev) CK(cudaEventRecord(ev[4], st));
    return LMPC_OK;
}

extern "C" {

int lmpc_step_dev(lmpc_handle* h, int mode, const double* x0_dev) { return step_dev_impl(h, mode, x0_dev, nullptr); }

// The same step with CUDA events between its kernels: ms4 = durations of K1 (regression), K2 (selection; 0 for mode 0), the QP
// kernel and the state shift.  Measurement support (bench.py's per-kernel rooflines); synchronises.
int lmpc_step_profile(lmpc_handle* h, int mode, const double* x0_dev, float* ms4) {
    if (!h || !ms4) return fail(LMPC_E_INVALID, "null argument");
    CK(cudaSetDevice(h->device));
    cudaEvent_t ev[5];
    for (int i = 0; i < 5; ++i) CK(cudaEventCreate(&ev[i]));
    int rc = step_dev_impl(h, mode, x0_dev, ev);
    if (rc == LMPC_OK && cudaStreamSynchronize(h->stream) != cudaSuccess) rc = fail(LMPC_E_CUDA, "stream synchronisation failed");
    if (rc == LMPC_OK)
        for (int i = 0; i < 4; ++i) cudaEventElapsedTime(&ms4[i], ev[i], ev[i + 1]);
    for (int i = 0; i < 5; ++i) cudaEventDestroy(ev[i]);
    return rc;
}

int lmpc_step_host(lmpc_handle* h, int mode, const double* x0, double* xPred, double* uPred, double* lambd, double* zt,
                   double* zt_u, double* SS_sel, int* status, int* iters, double* resid, int* flags) {
    int rc = need_store(h);
    if (rc) return rc;
    if (!x0) return fail(LMPC_E_INVALID, "null x0");
    const size_t B = h->batch;
    cudaStream_t s = h->stream;
    CK(cudaMemcpyAsync(h->hb[0].x0, x0, B * 6 * sizeof(double), cudaMemcpyHostToDevice, s));
    rc = lmpc_step_dev(h, mode, h->hb[0].x0);
    if (rc) return rc;
    QpIo out = {};
    out.xPred = xPred; out.uPred = uPred; out.lambd = lambd; out.zt = zt; out.ztu = zt_u; out.SS = SS_sel;
    out.status = status; out.iters = iters; out.resid = resid;
    if ((rc = copy_out(h, out, mode == 1)) != LMPC_OK) return rc;
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
    QpIo out = {};
    out.status = status; out.iters = iters; out.resid = resid;
    if ((rc = copy_out(h, out, false)) != LMPC_OK) return rc;
    if (flags) CK(cudaMemcpyAsync(flags, h->d_flags, sizeof(int) * h->batch, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

void* lmpc_device_buffer(lmpc_handle* h, const char* name) {
    if (!h || !name) return nullptr;
    for (const QpField& f : QP_FIELDS) if (f.name && !strcmp(f.name, name)) return f.at(h->hb[0]);
    for (const DevBuf& r : dev_bufs(h)) if (r.name && !strcmp(r.name, name)) return *r.p;
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
    if (Tcl >= LMPC_LANE_UNSAFE_KEY && lane_rules_on(h))
        return fail(LMPC_E_INVALID, "lmpc_rollout_create: a lane rule is installed: a lap time must stay below LMPC_LANE_UNSAFE_KEY");
    h->Tcl = Tcl; h->cur = 0; h->sim_step = 0;
    if ((rc = alloc_bufs(h, dev_bufs(h), OWN_ROLLOUT, h->batch, "lmpc_rollout_create")) != LMPC_OK) return rc;
    h->has_rollout = true;
    return LMPC_OK;
}
extern "C" {

static int need_rollout(lmpc_handle* h) {
    if (h && h->has_store && !h->has_rollout) return fail(LMPC_E_STATE, "call lmpc_rollout_create first");
    return need_store(h);
}

int lmpc_rollout_set_state(lmpc_handle* h, const double* x, const double* xglob) {
    if (int rc = need_rollout(h)) return rc;
    if (int rc = copy_bufs(h, cudaMemcpyHostToDevice, {{h->d_rx[h->cur], x}, {h->d_rg[h->cur], xglob}})) return rc;
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_rollout_get_state(lmpc_handle* h, double* x, double* xglob, int* done, int* cl_len) {
    if (int rc = need_rollout(h)) return rc;
    if (int rc = copy_bufs(h, cudaMemcpyDeviceToHost, {{h->d_rx[h->cur], x}, {h->d_rg[h->cur], xglob}, {h->d_done, done},
                                                     {h->d_cllen, cl_len}}))
        return rc;
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_rollout_get_health(lmpc_handle* h, int* flags_or, int* unsolved_steps) {
    if (int rc = need_rollout(h)) return rc;
    const size_t B = h->batch;
    if (flags_or) CK(cudaMemcpyAsync(flags_or, h->d_health, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    if (unsolved_steps) CK(cudaMemcpyAsync(unsolved_steps, h->d_health + B, sizeof(int) * B, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

// The simulator's arguments for one closed-loop step of the whole batch: state cur -> cur ^ 1 under the input uPred[b][0], noise z
// ([B][3] standard-normal draws) or, when null, Philox.  The health inputs (flags, status, health) stay null; the caller sets them.
static SimArgs sim_args(const lmpc_handle* h, const double* z, unsigned long long seed) {
    SimArgs sa = {};
    sa.batch = h->batch; sa.x = h->d_rx[h->cur]; sa.xg = h->d_rg[h->cur]; sa.u = h->hb[0].uPred; sa.u_stride = (long long)h->N * 2;
    sa.z = z; sa.seed = seed; sa.step = h->sim_step;
    sa.xn = h->d_rx[h->cur ^ 1]; sa.xgn = h->d_rg[h->cur ^ 1];
    sa.cl_x = h->d_clx; sa.cl_u = h->d_clu; sa.cl_len = h->d_cllen; sa.Tcl = h->Tcl; sa.done = h->d_done;
    sa.veh = h->veh.view(); sa.trk = tracks(h); sa.noise = h->noise.view(); sa.streams = h->streams.idx;
    return sa;
}

// The state the controllers see this step (DESIGN.md, "Per-controller measurement noise"): with a measurement table, *y is the
// measured state measure_kernel forms from the plant state and the clock; without one, *y is the plant state and nothing runs.
static int measure(lmpc_handle* h, unsigned long long seed, LapBudget retire, LapSchedule sched, const double** y) {
    *y = h->d_rx[h->cur];
    if (!h->meas.tab) return LMPC_OK;
    MeasArgs ma;
    ma.batch = h->batch; ma.x = h->d_rx[h->cur]; ma.y = h->d_xmeas; ma.seed = seed; ma.step = h->sim_step;
    ma.meas = h->meas.view(); ma.streams = h->streams.idx; ma.retire = retire;
    measure_kernel<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(ma, sched);
    CK(cudaGetLastError());
    h->launches += 1;
    *y = h->d_xmeas;
    return LMPC_OK;
}

// The state the controllers read this step (DESIGN.md, "Per-controller state observers"): with an observer table, *y becomes
// x_hat, which observe_kernel forms from *y and the controllers' previous predictions; without one, *y stays and nothing runs.
// blend: a step of mode 0 or 1 (the step flags are cleared before the launch, so a reset flag survives); else a PID or LTI step.
// With a prior table (DESIGN.md, "Observer priors") the MODEL instantiation runs: vsched, ssched are the plant's vehicle and
// surface lap schedules.  With a gain table as well (DESIGN.md, "Observer gains") observer_gain_kernel forms the model gains first
// in a step of mode 0 or 1, and the GAIN instantiation blends with them.
static int observe(lmpc_handle* h, bool blend, LapBudget retire, const double** y, LapSchedule vsched = {}, LapSchedule ssched = {}) {
    if (!h->obs.tab) return LMPC_OK;
    if (blend) CK(cudaMemsetAsync(h->d_flags, 0, sizeof(int) * h->batch, h->stream));
    ObserveArgs oa;
    oa.batch = h->batch; oa.N = h->N; oa.blend = blend ? 1 : 0; oa.y = *y; oa.xPredPrev = h->d_xPredPrev; oa.has_pred = h->d_hasPred;
    oa.x_est = h->d_xest; oa.flags = h->d_flags; oa.obs = h->obs.view(); oa.trk = tracks(h); oa.retire = retire;
    ObservePrior op;
    op.pri = h->opri.view(); op.dt = h->mc.dt; op.OldInput = h->d_OldInput; op.x_prior = h->d_xprior;
    op.veh = h->veh.view(); op.veh_s = vsched; op.surf = h->surf.view(); op.surf_s = ssched;
    ObserveGain og;
    og.gains = h->ogain.view(); og.jac = h->d_ojac; og.cov = h->d_ocov; og.gain = h->d_ogain;
    if (h->ogain.tab && blend) {
        constexpr int per_block = OBS_GAIN_WARPS * OBS_GAIN_PER_WARP;
        observer_gain_kernel<<<(h->batch + per_block - 1) / per_block, 32 * OBS_GAIN_WARPS, 0, h->stream>>>(oa, op, og);
        CK(cudaGetLastError());
        h->launches += 1;
    }
    auto kern = !h->opri.tab ? observe_kernel<false, false> : h->ogain.tab ? observe_kernel<true, true> : observe_kernel<true, false>;
    kern<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(oa, op, og);
    CK(cudaGetLastError());
    h->launches += 1;
    *y = h->d_xest;
    return LMPC_OK;
}

// One closed-loop step for every instance, all on the device (SysModel.py:34-48):
//   Controller.solve(x) -> u = uPred[0] -> Controller.addPoint(x, u) (LMPC) -> x+ = dynModel(x, x_glob, u); done = s+ > TrackLength
// The controller's x (solve, addPoint, the record) is the measured state y when a measurement table is installed, and the
// observer's x_hat formed from it when an observer table is installed.
int lmpc_rollout_step(lmpc_handle* h, int mode, const double* z_host, unsigned long long seed) {
    int rc = need_rollout(h);
    if (rc) return rc;
    const QpIo& q = h->hb[0];
    const double* xc = h->d_rx[h->cur];
    const LapBudget retire = lap_budget(h);
    const double* y = nullptr;
    if ((rc = measure(h, seed, retire, lap_schedule(h, LMPC_SCHEDULE_MEASUREMENT), &y)) != LMPC_OK) return rc;
    if ((rc = observe(h, mode != 2, retire, &y, lap_schedule(h, LMPC_SCHEDULE_VEHICLE), lap_schedule(h, LMPC_SCHEDULE_SURFACE))) != LMPC_OK)
        return rc;
    if (z_host) CK(cudaMemcpyAsync(h->d_z, z_host, sizeof(double) * h->batch * 3, cudaMemcpyHostToDevice, h->stream));
    if (mode == 2) {
        CK(cudaMemsetAsync(h->d_flags, 0, sizeof(int) * h->batch, h->stream));
        // LTI MPC with the per-instance model identified by lmpc_rollout_sysid (main.py:72-80); like the reference's LTI
        // controller it never refreshes the input-rate reference (OldInput keeps its initial value, PC.py:113-115)
        QpIo io = {};
        io.x0 = const_cast<double*>(y); io.uOld = h->d_OldInput; io.abc = h->d_abc_lti;
        io.xPred = q.xPred; io.uPred = q.uPred; io.slack = q.slack; io.status = q.status; io.iters = q.iters; io.resid = q.resid;
        rc = solve_dev(h, io, 54, 0, retire);
    } else {
        rc = step_dev_impl(h, mode, y, nullptr, retire, lap_schedule(h, LMPC_SCHEDULE_VEHICLE), lap_schedule(h, LMPC_SCHEDULE_SURFACE),
                           h->obs.tab != nullptr);
    }
    if (rc) return rc;
    if (mode == 1) {                                                                 // SysModel.py:38 -> PC.py:466-476
        ss_add_point_kernel<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(h->batch, h->ss, h->d_prevslot, y, q.uPred,
                                                                            (long long)h->N * 2, tracks(h), h->d_flags, nullptr, retire);
        CK(cudaGetLastError());
        h->launches += 1;
    }
    // the trace of the chosen controllers reads the step's results and the plant state before dynModel
    if (h->has_trace) {
        trace_step_kernel<<<h->tr.n, 128, 0, h->stream>>>(h->tr, xc, h->d_rg[h->cur], q.uPred, (long long)h->N * 2, q.xPred,
                                                        mode == 1 ? q.SS : nullptr, h->bk.lap_n, retire);
        CK(cudaGetLastError());
        h->launches += 1;
    }
    SimArgs sa = sim_args(h, z_host ? h->d_z : nullptr, seed);                       // SysModel.py:40 (dynModel)
    sa.flags = h->d_flags; sa.status = q.status; sa.health = h->d_health; sa.retire = retire;
    if (h->meas.tab || h->obs.tab) sa.rec_x = y;
    (h->surf.tab ? sim_step_kernel<true> : sim_step_kernel<false>)<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(
        h->mc, sa, reports(h), q.iters, lap_schedule(h, LMPC_SCHEDULE_VEHICLE), lap_schedule(h, LMPC_SCHEDULE_NOISE), h->surf.view(),
        lap_schedule(h, LMPC_SCHEDULE_SURFACE));
    CK(cudaGetLastError());
    h->launches += 1;
    h->cur ^= 1;
    h->sim_step += 1;
    return LMPC_OK;
}

// One closed-loop step with the PID path follower as the controller (main.py:65-66: the lap that seeds everything else).
// z_pid_host[B,2] / z_sim_host[B,3]: the reference's standard-normal draws in its order (PID steer, PID accel | vx, vy, wz);
// NULL = Philox on the device.
int lmpc_rollout_pid_step(lmpc_handle* h, double vt, const double* z_pid_host, const double* z_sim_host, unsigned long long seed) {
    if (int rc = need_rollout(h)) return rc;
    const double* y = nullptr;                   // the PID's input and the record's state rows (measure, observe)
    if (int rc = measure(h, seed, LapBudget{}, LapSchedule{}, &y)) return rc;
    if (int rc = observe(h, false, LapBudget{}, &y)) return rc;
    if (z_pid_host) CK(cudaMemcpyAsync(h->d_zpid, z_pid_host, sizeof(double) * h->batch * 2, cudaMemcpyHostToDevice, h->stream));
    if (z_sim_host) CK(cudaMemcpyAsync(h->d_z, z_sim_host, sizeof(double) * h->batch * 3, cudaMemcpyHostToDevice, h->stream));
    PidArgs pa;
    pa.batch = h->batch; pa.x = y; pa.vt = vt; pa.z = z_pid_host ? h->d_zpid : nullptr; pa.seed = seed; pa.step = h->sim_step;
    pa.u = h->hb[0].uPred; pa.u_stride = (long long)h->N * 2;
    pa.noise = h->noise.view(); pa.streams = h->streams.idx;
    pid_input_kernel<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(pa);
    SimArgs sa = sim_args(h, z_sim_host ? h->d_z : nullptr, seed);
    sa.health = h->d_health;          // no step flags or QP status here: only the simulator's own bits
    if (h->meas.tab || h->obs.tab) sa.rec_x = y;
    (h->surf.tab ? sim_step_kernel<true> : sim_step_kernel<false>)<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(
        h->mc, sa, reports(h), nullptr, LapSchedule{}, LapSchedule{}, h->surf.view(), LapSchedule{});
    CK(cudaGetLastError());
    h->launches += 2;
    h->cur ^= 1;
    h->sim_step += 1;
    if (z_pid_host || z_sim_host) CK(cudaStreamSynchronize(h->stream));   // pageable host arrays of the caller
    return LMPC_OK;
}

// Both install orders of a lap schedule: while schedule k indexes a table, a new table of nrows rows must cover its largest entry
static int check_schedule_cover(const lmpc_handle* h, const char* who, int k, int nrows) {
    const std::vector<int>& r = h->sched[k].rows;
    if (r.empty()) return LMPC_OK;
    const int top = *std::max_element(r.begin(), r.end());
    if (top < nrows) return LMPC_OK;
    return fail(LMPC_E_INVALID, std::string(who) + ": the installed lap schedule names row " + std::to_string(top) + ", the new table has " +
                                    std::to_string(nrows) + " row(s); install a covering schedule first or remove it");
}

// Per-controller vehicles: m, Iz, lf, lr positive and all ten values finite; nsets == 0 returns to the reference vehicle.
int lmpc_rollout_set_vehicles(lmpc_handle* h, const lmpc_vehicle_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_rollout_set_vehicles";
    if (!h) return fail(LMPC_E_INVALID, "null handle");
    if (int rc = check_schedule_cover(h, who, LMPC_SCHEDULE_VEHICLE, nsets > 0 ? nsets : 1)) return rc;
    const lmpc_vehicle_params ref = reference_vehicle();
    return install_table(h, who, h->veh, sets, nsets, set_of_instance, &ref, [&](int k, lmpc_vehicle_params& row) {
        const lmpc_vehicle_params& v = sets[k];
        const double all[10] = {v.m, v.lf, v.lr, v.Iz, v.Df, v.Cf, v.Bf, v.Dr, v.Cr, v.Br};
        bool ok = v.m > 0 && v.Iz > 0 && v.lf > 0 && v.lr > 0;
        for (double x : all) ok = ok && isfinite(x);
        if (!ok)
            return fail(LMPC_E_INVALID, std::string(who) + ": vehicle " + std::to_string(k) +
                                            ": m, Iz, lf, lr must be positive and all ten values finite");
        row = v;
        return LMPC_OK;
    });
}

// Per-controller track surfaces: per row 0 <= nzone <= LMPC_MAX_ZONES, every zone's values finite, 0 <= s_start < s_end, mu_f and
// mu_r >= 0, zones ascending without overlap; nsets == 0 removes the table (refused while a surface schedule names a row).
int lmpc_rollout_set_surfaces(lmpc_handle* h, const lmpc_surface_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_rollout_set_surfaces";
    if (!h) return fail(LMPC_E_INVALID, "null handle");
    if (int rc = check_schedule_cover(h, who, LMPC_SCHEDULE_SURFACE, nsets)) return rc;
    return install_table(h, who, h->surf, sets, nsets, set_of_instance, (const lmpc_surface_params*)nullptr,
                         [&](int k, lmpc_surface_params& row) {
        const lmpc_surface_params& r = sets[k];
        const std::string w = std::string(who) + ": surface " + std::to_string(k);
        if (r.nzone < 0 || r.nzone > LMPC_MAX_ZONES)
            return fail(LMPC_E_INVALID, w + ": nzone must be 0 .. " + std::to_string(LMPC_MAX_ZONES));
        for (int z = 0; z < r.nzone; ++z) {
            const double* v = r.zone + 4 * z;
            const std::string wz = w + ", zone " + std::to_string(z);
            if (!(isfinite(v[0]) && isfinite(v[1]) && isfinite(v[2]) && isfinite(v[3])))
                return fail(LMPC_E_INVALID, wz + ": s_start, s_end, mu_f and mu_r must be finite");
            if (!(v[0] >= 0.0 && v[0] < v[1]))
                return fail(LMPC_E_INVALID, wz + ": needs 0 <= s_start < s_end");
            if (!(v[2] >= 0.0 && v[3] >= 0.0)) return fail(LMPC_E_INVALID, wz + ": mu_f and mu_r must be >= 0");
            if (z > 0 && !(r.zone[4 * (z - 1) + 1] <= v[0]))
                return fail(LMPC_E_INVALID, wz + ": zones must ascend without overlap (s_end of the previous zone <= s_start)");
        }
        row = r;
        return LMPC_OK;
    });
}

// Per-controller noise: every value finite and >= 0; nsets == 0 returns to the reference's constants.
static_assert(sizeof(lmpc_noise_params) == 11 * sizeof(double), "lmpc_noise_params is checked as an array of its 11 doubles");
int lmpc_rollout_set_noise(lmpc_handle* h, const lmpc_noise_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_rollout_set_noise";
    if (!h) return fail(LMPC_E_INVALID, "null handle");
    if (int rc = check_schedule_cover(h, who, LMPC_SCHEDULE_NOISE, nsets > 0 ? nsets : 1)) return rc;
    const lmpc_noise_params ref = reference_noise();
    return install_table(h, who, h->noise, sets, nsets, set_of_instance, &ref, [&](int k, lmpc_noise_params& row) {
        const double* v = (const double*)&sets[k];
        for (size_t j = 0; j < sizeof(lmpc_noise_params) / sizeof(double); ++j)
            if (!(isfinite(v[j]) && v[j] >= 0.0))
                return fail(LMPC_E_INVALID, std::string(who) + ": noise set " + std::to_string(k) +
                                                ": every sigma, clip and the gain must be finite and >= 0");
        row = sets[k];
        return LMPC_OK;
    });
}

// Noise streams: every stream number >= 0 (repeats allowed); NULL returns to stream b = b.  An array without rows.
int lmpc_rollout_set_noise_streams(lmpc_handle* h, const int* stream_of_instance) {
    static const char* who = "lmpc_rollout_set_noise_streams";
    if (!h) return fail(LMPC_E_INVALID, "null handle");
    for (int b = 0; b < (stream_of_instance ? h->batch : 0); ++b)
        if (stream_of_instance[b] < 0)
            return fail(LMPC_E_INVALID, std::string(who) + ": stream of instance " + std::to_string(b) + " is negative");
    return swap_table<int>(h, who, h->streams, nullptr, 0, stream_of_instance);
}

// Per-controller measurement noise: every value finite and >= 0; nsets == 0 removes the table (the controllers read the plant
// state, no kernel runs), the precedent of the parameter sets.
static_assert(sizeof(lmpc_measurement_params) == 12 * sizeof(double), "lmpc_measurement_params is checked as an array of its 12 doubles");
int lmpc_rollout_set_measurement_noise(lmpc_handle* h, const lmpc_measurement_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_rollout_set_measurement_noise";
    if (int rc = need_rollout(h)) return rc;
    if (int rc = check_schedule_cover(h, who, LMPC_SCHEDULE_MEASUREMENT, nsets)) return rc;
    return install_table(h, who, h->meas, sets, nsets, set_of_instance, (const lmpc_measurement_params*)nullptr,
                         [&](int k, lmpc_measurement_params& row) {
        const double* v = (const double*)&sets[k];
        for (size_t j = 0; j < sizeof(lmpc_measurement_params) / sizeof(double); ++j)
            if (!(isfinite(v[j]) && v[j] >= 0.0))
                return fail(LMPC_E_INVALID, std::string(who) + ": measurement set " + std::to_string(k) +
                                                ": every sigma and clip must be finite and >= 0");
        row = sets[k];
        return LMPC_OK;
    });
}

// Per-controller state observers: mode 0 or 1, every gain finite and in [0, 1]; nsets == 0 removes the table (the controllers
// read the measured or plant state, no kernel runs).
int lmpc_rollout_set_observers(lmpc_handle* h, const lmpc_observer_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_rollout_set_observers";
    if (int rc = need_rollout(h)) return rc;
    return install_table(h, who, h->obs, sets, nsets, set_of_instance, (const lmpc_observer_params*)nullptr,
                         [&](int k, lmpc_observer_params& row) {
        const lmpc_observer_params& o = sets[k];
        const std::string w = std::string(who) + ": observer " + std::to_string(k);
        if (o.mode != 0 && o.mode != 1) return fail(LMPC_E_INVALID, w + ": mode must be 0 or 1");
        for (double l : o.gain)
            if (!(isfinite(l) && l >= 0.0 && l <= 1.0)) return fail(LMPC_E_INVALID, w + ": every gain must be finite and in [0, 1]");
        row = o;
        row.pad = 0;
        return LMPC_OK;
    });
}

// Per-controller observer priors: source 0, 1 or 2; under source 1 all ten vehicle values finite and m, lf, lr, Iz > 0 (the
// rule of a mode 1 prediction model); nsets == 0 removes the table (every observer takes its own plan, observe_kernel<false>).
int lmpc_rollout_set_observer_priors(lmpc_handle* h, const lmpc_observer_prior_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_rollout_set_observer_priors";
    if (int rc = need_rollout(h)) return rc;
    if (h->ogain.tab) {        // a mode 1 gain row needs a model prior: the table, or its removal, must not take it away
        if (int rc = check_set_index(h, who, sets, nsets, set_of_instance)) return rc;
        for (int b = 0; b < h->batch; ++b) {
            if (h->ogain.rows[table_row(h->ogain, b)].mode != 1) continue;
            if (nsets == 0 || sets[set_of_instance[b]].source == 0)
                return fail(LMPC_E_INVALID, std::string(who) + ": controller " + std::to_string(b) +
                                                " has a mode 1 observer gain row (lmpc_rollout_set_observer_gains), which needs source 1 or 2");
        }
    }
    return install_table(h, who, h->opri, sets, nsets, set_of_instance, (const lmpc_observer_prior_params*)nullptr,
                         [&](int k, lmpc_observer_prior_params& r) {
        const lmpc_observer_prior_params& s = sets[k];
        const lmpc_vehicle_params& v = s.vehicle;
        const std::string w = std::string(who) + ": row " + std::to_string(k) + ": ";
        if (s.source < 0 || s.source > 2) return fail(LMPC_E_INVALID, w + "source must be 0, 1 or 2");
        memset(&r, 0, sizeof(r));
        r.source = s.source;
        if (s.source == 1) {
            const double all[10] = {v.m, v.lf, v.lr, v.Iz, v.Df, v.Cf, v.Bf, v.Dr, v.Cr, v.Br};
            for (double x : all)
                if (!isfinite(x)) return fail(LMPC_E_INVALID, w + "all ten vehicle values must be finite");
            if (!(v.m > 0 && v.lf > 0 && v.lr > 0 && v.Iz > 0)) return fail(LMPC_E_INVALID, w + "a source 1 vehicle needs m, lf, lr, Iz > 0");
            r.vehicle = v;
        }
        return LMPC_OK;
    });
}

// Per-controller observer gains: mode 0 or 1; under mode 1 every q_j and r_j finite and > 0, and the controller's observer prior
// row source 1 or 2 (check_gain_priors); nsets == 0 removes the table (every observer blends with its row's fixed gains).
int lmpc_rollout_set_observer_gains(lmpc_handle* h, const lmpc_observer_gain_params* sets, int nsets, const int* set_of_instance) {
    static const char* who = "lmpc_rollout_set_observer_gains";
    if (int rc = need_rollout(h)) return rc;
    if (int rc = check_set_index(h, who, sets, nsets, set_of_instance)) return rc;
    for (int b = 0; b < (nsets > 0 ? h->batch : 0); ++b) {
        if (sets[set_of_instance[b]].mode != 1) continue;
        if (!h->opri.tab || h->opri.rows[table_row(h->opri, b)].source == 0)
            return fail(LMPC_E_INVALID, std::string(who) + ": controller " + std::to_string(b) +
                                            ": a mode 1 row needs an observer prior of source 1 or 2 (lmpc_rollout_set_observer_priors)");
    }
    return install_table(h, who, h->ogain, sets, nsets, set_of_instance, (const lmpc_observer_gain_params*)nullptr,
                         [&](int k, lmpc_observer_gain_params& r) {
        const lmpc_observer_gain_params& s = sets[k];
        const std::string w = std::string(who) + ": row " + std::to_string(k) + ": ";
        if (s.mode != 0 && s.mode != 1) return fail(LMPC_E_INVALID, w + "mode must be 0 or 1");
        memset(&r, 0, sizeof(r));
        r.mode = s.mode;
        if (s.mode == 1) {
            for (int j = 0; j < 6; ++j)
                if (!(isfinite(s.q[j]) && s.q[j] > 0.0 && isfinite(s.r[j]) && s.r[j] > 0.0))
                    return fail(LMPC_E_INVALID, w + "every q and r must be finite and > 0");
            for (int j = 0; j < 6; ++j) { r.q[j] = s.q[j]; r.r[j] = s.r[j]; }
        }
        return LMPC_OK;
    });
}

// Lap budgets: every budget >= 1; NULL removes the budgets.  An array without rows, like the noise streams.
int lmpc_rollout_set_lap_budget(lmpc_handle* h, const int* budget_of_instance) {
    static const char* who = "lmpc_rollout_set_lap_budget";
    if (int rc = need_rollout(h)) return rc;
    for (int b = 0; b < (budget_of_instance ? h->batch : 0); ++b)
        if (budget_of_instance[b] < 1)
            return fail(LMPC_E_INVALID, std::string(who) + ": budget of instance " + std::to_string(b) + " is below 1");
    return swap_table<int>(h, who, h->budget, nullptr, 0, budget_of_instance);
}

// Lap schedules: row_of_lap[B][nlaps] of table `table`, every entry a row of the table as installed; nlaps 0 + NULL removes it.
// Stored as a table whose rows are the schedule and which has no index (swap_table), so a failed allocation changes nothing.
int lmpc_rollout_set_lap_schedule(lmpc_handle* h, int table, int nlaps, const int* row_of_lap) {
    static const char* who = "lmpc_rollout_set_lap_schedule";
    if (int rc = need_rollout(h)) return rc;
    const std::string w(who);
    if (table < LMPC_SCHEDULE_VEHICLE || table > LMPC_SCHEDULE_SURFACE)
        return fail(LMPC_E_INVALID, w + ": table must be LMPC_SCHEDULE_VEHICLE, _NOISE, _MEASUREMENT or _SURFACE");
    const size_t nrows = table == LMPC_SCHEDULE_VEHICLE ? h->veh.rows.size()
                       : table == LMPC_SCHEDULE_NOISE   ? h->noise.rows.size()
                       : table == LMPC_SCHEDULE_MEASUREMENT ? h->meas.rows.size() : h->surf.rows.size();
    if (table == LMPC_SCHEDULE_MEASUREMENT && !h->meas.tab && row_of_lap)
        return fail(LMPC_E_STATE, w + ": a measurement schedule needs a measurement table (lmpc_rollout_set_measurement_noise)");
    if (table == LMPC_SCHEDULE_SURFACE && !h->surf.tab && row_of_lap)     // every entry names a row of an absent table
        return fail(LMPC_E_INVALID, w + ": a surface schedule needs a surface table (lmpc_rollout_set_surfaces)");
    if ((nlaps == 0) != (row_of_lap == nullptr))
        return fail(LMPC_E_INVALID, w + ": nlaps == 0 goes with a NULL row_of_lap, nlaps >= 1 with an array");
    if (nlaps < 0 || nlaps > 1024) return fail(LMPC_E_INVALID, w + ": nlaps must be 0 .. 1024");
    const size_t n = (size_t)h->batch * nlaps;
    for (size_t i = 0; i < n; ++i)
        if (row_of_lap[i] < 0 || (size_t)row_of_lap[i] >= nrows)
            return fail(LMPC_E_INVALID, w + ": entry " + std::to_string(i % nlaps) + " of controller " + std::to_string(i / nlaps) +
                                            " is outside the table's " + std::to_string(nrows) + " row(s)");
    if (int rc = swap_table<int>(h, who, h->sched[table], row_of_lap, (int)n, nullptr)) return rc;
    h->sched_L[table] = nlaps;
    return LMPC_OK;
}

// Per-lap reports: 1 <= max_laps <= 1024 allocates an empty table (refused while a record holds rows), 0 frees it.  New buffers are
// allocated before the old ones go, so a failed allocation leaves the handle as it was.
int lmpc_rollout_enable_lap_reports(lmpc_handle* h, int max_laps) {
    static const char* who = "lmpc_rollout_enable_lap_reports";
    if (int rc = need_rollout(h)) return rc;
    if (max_laps < 0 || max_laps > 1024) return fail(LMPC_E_INVALID, std::string(who) + ": max_laps must be 0 .. 1024");
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    if (max_laps > 0) {
        std::vector<int> cl(h->batch);
        CK(cudaMemcpy(cl.data(), h->d_cllen, sizeof(int) * h->batch, cudaMemcpyDeviceToHost));
        for (int b = 0; b < h->batch; ++b)
            if (cl[b] > 0)
                return fail(LMPC_E_STATE, std::string(who) + ": the closed-loop record of controller " + std::to_string(b) +
                                              " holds rows; enable reports before the PID lap or right after a hand-over or seeding");
    }
    lmpc_lap_report* old_rows = h->d_rep_rows;
    LapRun* old_run = h->d_rep_run;
    const int old_L = h->rep_L;
    h->d_rep_rows = nullptr; h->d_rep_run = nullptr; h->rep_L = max_laps;
    if (max_laps > 0) {
        int rc = alloc_bufs(h, dev_bufs(h), OWN_REPORTS, h->batch, who);
        if (rc == LMPC_OK) {
            lap_reports_reset_kernel<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(h->batch, reports(h));
            cudaError_t e = cudaGetLastError();
            if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
            if (e != cudaSuccess) {
                free_bufs(dev_bufs(h), OWN_REPORTS);
                rc = fail(LMPC_E_CUDA, std::string(who) + ": " + cudaGetErrorString(e));
            }
        }
        if (rc != LMPC_OK) {
            h->d_rep_rows = old_rows; h->d_rep_run = old_run; h->rep_L = old_L;
            return rc;
        }
        h->launches += 1;
    }
    if (old_rows) cudaFree(old_rows);
    if (old_run) cudaFree(old_run);
    return LMPC_OK;
}

int lmpc_rollout_get_lap_reports(lmpc_handle* h, lmpc_lap_report* rows, int* n) {
    if (int rc = need_rollout(h)) return rc;
    if (!h->rep_L) return fail(LMPC_E_STATE, "lmpc_rollout_get_lap_reports: lap reports are not enabled");
    if (rows) CK(cudaMemcpyAsync(rows, h->d_rep_rows, sizeof(lmpc_lap_report) * h->batch * h->rep_L, cudaMemcpyDeviceToHost, h->stream));
    if (n) CK(cudaMemcpy2DAsync(n, sizeof(int), &h->d_rep_run->n, sizeof(LapRun), sizeof(int), h->batch, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_sizeof_lap_report(void) { return (int)sizeof(lmpc_lap_report); }

// Regression(x, u, lamb) of Utilities.py:5-28 on every instance's closed-loop record: per-instance LTI model in the device
// buffer "abc_lti" ([B][54] = A | B | C = 0, the layout lmpc_solve_mpc_dev takes with strides (54, 0)); abc_host may be NULL.
int lmpc_rollout_sysid(lmpc_handle* h, double lamb, double* abc_host, int* flags_host) {
    if (int rc = need_rollout(h)) return rc;
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
    if (int rc = need_rollout(h)) return rc;
    if (lane_rules_on(h)) return fail(LMPC_E_STATE, "lmpc_rollout_seed_from_record: lane rules need the device books (_dev)");
    if (copies < 1 || ss_slot0 < 0 || model_slot0 < 0 || ss_slot0 + copies > h->ss.cap || model_slot0 + copies > h->mdl.cap)
        return fail(LMPC_E_INVALID, "seed copies do not fit the lap pools");
    h->laps_stored = true;
    if (h->d_warm_valid) CK(cudaMemsetAsync(h->d_warm_valid, 0, sizeof(int) * h->batch, h->stream));
    seed_from_record_kernel<<<h->batch, 256, 0, h->stream>>>(
        h->batch, h->ss, h->mdl, copies, ss_slot0, model_slot0, h->d_clx, h->d_clu, h->d_cllen, h->Tcl, h->N, h->d_xLin, h->d_uLin,
        h->d_ztState, h->d_OldInput, h->d_timeStep, h->d_hasPred, h->d_done, tracks(h), h->shp.view(), reports(h));
    CK(cudaGetLastError());
    h->launches += 1;
    return lane_margin_rows(h, true);       // adaptive margins start over with the seeded stores
}

int lmpc_rollout_get_lap(lmpc_handle* h, int inst, int* T, double* x, double* u) {
    if (int rc = need_rollout(h)) return rc;
    if (inst < 0 || inst >= h->batch || !T) return fail(LMPC_E_INVALID, "bad instance");
    CK(cudaMemcpyAsync(T, h->d_cllen + inst, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (x) CK(cudaMemcpyAsync(x, h->d_clx + (size_t)inst * h->Tcl * 6, sizeof(double) * (*T) * 6, cudaMemcpyDeviceToHost, h->stream));
    if (u) CK(cudaMemcpyAsync(u, h->d_clu + (size_t)inst * h->Tcl * 2, sizeof(double) * (*T) * 2, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

// Hand the finished laps over to the stores without leaving the device, for every instance with fin[b] != 0 in ONE launch (a
// Monte-Carlo batch finishes hundreds of laps in the same step): safe-set slot (computeCost on the device) and/or regression slot
// (either may be -1), then restart the record; the curvilinear state is moved back by one track length (SysModel.py:50) and the
// controller's step counter is reset (PC.py:445).
int lmpc_rollout_commit_laps(lmpc_handle* h, const int* fin, const int* ss_slots, const int* model_slots) {
    if (int rc = need_rollout(h)) return rc;
    if (lane_rules_on(h)) return fail(LMPC_E_STATE, "lmpc_rollout_commit_laps: lane rules need the device books (_dev)");
    if (lane_margins_adapt(h)) return fail(LMPC_E_STATE, "lmpc_rollout_commit_laps: adaptive lane margins need the device hand-over (_dev)");
    if (!fin || !ss_slots || !model_slots) return fail(LMPC_E_INVALID, "null argument");
    for (int b = 0; b < h->batch; ++b)
        if (fin[b] && (ss_slots[b] >= h->ss.cap || model_slots[b] >= h->mdl.cap)) return fail(LMPC_E_INVALID, "slot out of range");
    const size_t B = h->batch;
    for (int b = 0; b < h->batch; ++b)
        if (fin[b] && (ss_slots[b] >= 0 || model_slots[b] >= 0)) h->laps_stored = true;
    CK(cudaMemcpyAsync(h->d_xchg, fin, sizeof(int) * B, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_xchg + B, ss_slots, sizeof(int) * B, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_xchg + 2 * B, model_slots, sizeof(int) * B, cudaMemcpyHostToDevice, h->stream));
    commit_laps_kernel<<<h->batch, 256, 0, h->stream>>>(
        h->batch, h->ss, h->mdl, h->d_xchg, h->d_xchg + B, h->d_xchg + 2 * B, h->d_clx, h->d_clu, h->d_cllen, h->Tcl, h->d_rx[h->cur],
        h->d_timeStep, h->d_done, tracks(h), reports(h));
    CK(cudaGetLastError());
    h->launches += 1;
    CK(cudaStreamSynchronize(h->stream));   // the three host arrays are pageable memory of the caller
    return LMPC_OK;
}

int lmpc_ss_export_laps_dev(lmpc_handle* h, const int* slots, int Tpad, double* rows_dev, int* lens_dev) {
    if (int rc = need_store(h)) return rc;
    if (!slots || !rows_dev || !lens_dev || Tpad < 1) return fail(LMPC_E_INVALID, "bad export arguments");
    for (int b = 0; b < h->batch; ++b)
        if (slots[b] >= h->ss.cap) return fail(LMPC_E_INVALID, "safe-set slot out of range");
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
int lmpc_books_set(lmpc_handle* h, const int* ss_time, const int* ss_lap, const int* it, const int* md_time, const int* md_seq,
                   const int* md_cnt) {
    int rc = need_store(h);
    if (rc) return rc;
    if (!ss_time || !ss_lap || !it || !md_time || !md_seq || !md_cnt) return fail(LMPC_E_INVALID, "null argument");
    const LapBooks& k = h->bk;
    for (int b = 0; b < h->batch; ++b)     // a lane-unsafe key belongs to a controller whose lane rule is on
        for (int s = 0; s < k.ss_cap && !lane_rule_of(h, b); ++s)
            if (ss_lap[(size_t)b * k.ss_cap + s] >= 0 && ss_time[(size_t)b * k.ss_cap + s] >= LMPC_LANE_UNSAFE_KEY)
                return fail(LMPC_E_INVALID, "lmpc_books_set: controller " + std::to_string(b) + ", slot " + std::to_string(s) +
                                                ": a lane-unsafe key (>= LMPC_LANE_UNSAFE_KEY) without a lane rule");
    if ((rc = copy_bufs(h, cudaMemcpyHostToDevice, {{k.ss_time, ss_time}, {k.ss_lap, ss_lap}, {k.it, it}, {k.md_time, md_time},
                                                   {k.md_seq, md_seq}, {k.md_cnt, md_cnt}})))
        return rc;
    CK(cudaMemsetAsync(k.lap_n, 0, sizeof(int) * h->batch, h->stream));
    // sel, is_prev, prev_slot, used of these tables
    books_refresh_kernel<<<(h->batch + 127) / 128, 128, 0, h->stream>>>(h->batch, k, h->ssl.view(), h->lwin.view());
    CK(cudaGetLastError());
    h->launches += 1;
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_books_get(lmpc_handle* h, int* ss_time, int* ss_lap, int* it, int* md_time, int* md_seq, int* md_cnt, int* sel, int* is_prev,
                   int* prev_slot, int* used, int* lap_hist, int* lap_n) {
    int rc = need_store(h);
    if (rc) return rc;
    const LapBooks& k = h->bk;
    if ((rc = copy_bufs(h, cudaMemcpyDeviceToHost, {{k.ss_time, ss_time}, {k.ss_lap, ss_lap}, {k.it, it}, {k.md_time, md_time},
                                                   {k.md_seq, md_seq}, {k.md_cnt, md_cnt}, {k.sel, sel}, {k.isprev, is_prev},
                                                   {k.prevslot, prev_slot}, {k.used, used}, {k.lap_hist, lap_hist}, {k.lap_n, lap_n}})))
        return rc;
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

// Lap hand-over of every controller whose lap just ended, bookkeeping on the device; enqueue only.
int lmpc_rollout_commit_laps_dev(lmpc_handle* h) {
    if (int rc = need_rollout(h)) return rc;
    h->laps_stored = true;     // enqueue only: which controllers finish a lap is not known here
    commit_laps_books_kernel<<<h->batch, 256, 0, h->stream>>>(
        h->batch, h->ss, h->mdl, h->bk, h->d_clx, h->d_clu, h->d_cllen, h->Tcl, h->d_rx[h->cur], h->d_timeStep, h->d_done, h->d_health,
        tracks(h), h->M > 0 ? 1 : 0, lap_budget(h), h->ssl.view(), reports(h), h->lwin.view(), lane_rules(h), lane_margins(h));
    CK(cudaGetLastError());
    h->launches += 1;
    return LMPC_OK;
}

int lmpc_rollout_seed_from_record_dev(lmpc_handle* h, int copies) {
    if (int rc = need_rollout(h)) return rc;
    if (copies < 1 || (h->M > 0 && copies > h->ss.cap) || copies > h->mdl.cap) return fail(LMPC_E_INVALID, "seed copies do not fit the lap pools");
    h->laps_stored = true;
    if (h->d_warm_valid) CK(cudaMemsetAsync(h->d_warm_valid, 0, sizeof(int) * h->batch, h->stream));
    seed_books_kernel<<<h->batch, 256, 0, h->stream>>>(
        h->batch, h->ss, h->mdl, h->bk, copies, h->d_clx, h->d_clu, h->d_cllen, h->Tcl, h->N, h->d_xLin, h->d_uLin, h->d_ztState,
        h->d_OldInput, h->d_timeStep, h->d_hasPred, h->d_done, tracks(h), h->M > 0 ? 1 : 0, h->shp.view(), h->ssl.view(), reports(h),
        h->lwin.view(), lane_rules(h));
    CK(cudaGetLastError());
    h->launches += 1;
    return lane_margin_rows(h, true);       // adaptive margins start over with the seeded books
}

int lmpc_rollout_stats(lmpc_handle* h, int* out4) {
    if (int rc = need_rollout(h)) return rc;
    if (!out4) return fail(LMPC_E_INVALID, "null output");
    rollout_stats_kernel<<<1, 1024, 0, h->stream>>>(h->batch, h->bk, h->d_cllen, h->d_health, nullptr, 1, h->d_stats, lap_budget(h));
    CK(cudaGetLastError());
    h->launches += 1;
    CK(cudaMemcpyAsync(out4, h->d_stats, sizeof(int) * 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

int lmpc_rollout_group_stats(lmpc_handle* h, int* out) {
    if (int rc = need_rollout(h)) return rc;
    if (!out) return fail(LMPC_E_INVALID, "null output");
    const int G = h->ngroups > 0 ? h->ngroups : 1;
    rollout_stats_kernel<<<1, 1024, 0, h->stream>>>(h->batch, h->bk, h->d_cllen, h->d_health, h->pool_grp.idx, G, h->d_stats, lap_budget(h));
    CK(cudaGetLastError());
    h->launches += 1;
    CK(cudaMemcpyAsync(out, h->d_stats, sizeof(int) * 4 * G, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return LMPC_OK;
}

// Send side of the pooled exchange: per pool group, the kbest fastest latest-own laps of this rank, packed on the device.
// ship_host (null: every group) is a checked 0/1 mask [G]; a masked-out group ships rows with global id -1.
static int pool_export(lmpc_handle* h, const char* who, int kbest, int Tpad, long long gid_base, const int* ship_host, double* rows_dev,
                       int* meta_dev) {
    int rc = need_store(h);
    if (rc) return rc;
    if (kbest < 1 || kbest > POOL_MAXK || Tpad < 1 || !rows_dev || !meta_dev) return fail(LMPC_E_INVALID, "bad export arguments");
    if (h->M <= 0) return fail(LMPC_E_STATE, "handle has no safe set");
    if ((rc = one_track_per_group(h, who)) != LMPC_OK) return rc;
    const int G = h->ngroups > 0 ? h->ngroups : 1;
    int* ship = nullptr;
    if (ship_host) {     // staged from pageable stack memory, so the caller's array may change once the call returns
        int mask[POOL_MAXG];
        for (int g = 0; g < G; ++g) mask[g] = ship_host[g];
        ship = h->d_poolidx + POOL_SHIP;
        CK(cudaMemcpyAsync(ship, mask, sizeof(int) * G, cudaMemcpyHostToDevice, h->stream));
    }
    pool_local_best_kernel<<<G, 1024, 0, h->stream>>>(h->batch, h->ss, h->bk, kbest, Tpad, h->pool_min_over, h->pool_grp.idx, ship,
                                                      h->d_poolidx, h->lrule.tab);
    pool_export_kernel<<<G * kbest, 256, 0, h->stream>>>(h->ss, h->bk, h->d_poolidx, kbest, Tpad, gid_base, rows_dev, meta_dev, h->lrule.tab);
    CK(cudaGetLastError());
    h->launches += 2;
    return LMPC_OK;
}

int lmpc_pool_export_dev(lmpc_handle* h, int kbest, int Tpad, long long gid_base, double* rows_dev, int* meta_dev) {
    return pool_export(h, "lmpc_pool_export_dev", kbest, Tpad, gid_base, nullptr, rows_dev, meta_dev);
}

int lmpc_pool_export_groups_dev(lmpc_handle* h, int kbest, int Tpad, long long gid_base, const int* ship_host, double* rows_dev,
                                int* meta_dev) {
    static const char* who = "lmpc_pool_export_groups_dev";
    if (int rc = need_store(h)) return rc;
    if (!ship_host) return fail(LMPC_E_INVALID, std::string(who) + ": null ship mask");
    const int G = h->ngroups > 0 ? h->ngroups : 1;
    for (int g = 0; g < G; ++g)
        if (ship_host[g] != 0 && ship_host[g] != 1)
            return fail(LMPC_E_INVALID, std::string(who) + ": ship mask entry " + std::to_string(g) + " is neither 0 nor 1");
    return pool_export(h, who, kbest, Tpad, gid_base, ship_host, rows_dev, meta_dev);
}

// Receive side: rank the gathered laps per pool group, every controller files the `share` fastest of its group it does not own.
// took_host (may be NULL) receives the number of laps stored; the call then synchronises.
int lmpc_pool_import_dev(lmpc_handle* h, int n_src, int share, int Tpad, long long gid_base, const double* rows_dev, const int* meta_dev,
                         int* took_host) {
    int rc = need_store(h);
    if (rc) return rc;
    const int G = h->ngroups > 0 ? h->ngroups : 1;
    if (n_src < 1 || n_src > POOL_MAXSRC * G || share < 1 || Tpad < 1 || !rows_dev || !meta_dev)
        return fail(LMPC_E_INVALID, "bad import arguments");
    if (h->M <= 0) return fail(LMPC_E_STATE, "handle has no safe set");
    if ((rc = one_track_per_group(h, "lmpc_pool_import_dev")) != LMPC_OK) return rc;
    h->laps_stored = true;
    int* order = h->d_poolidx + POOL_ORDER;
    int* cnt = h->d_poolidx + POOL_COUNT;
    int* took = h->d_poolidx + POOL_TOOK;
    CK(cudaMemsetAsync(took, 0, sizeof(int), h->stream));
    pool_rank_kernel<<<G, 64, 0, h->stream>>>(n_src, meta_dev, order, cnt);
    pool_import_kernel<<<h->batch, 256, 0, h->stream>>>(
        h->batch, h->ss, h->mdl, h->bk, share, Tpad, rows_dev, meta_dev, h->pool_grp.idx, order, cnt, gid_base, took,
        h->has_rollout ? h->d_health : nullptr, h->ssl.view(), h->lwin.view(), lane_rules(h));
    CK(cudaGetLastError());
    h->launches += 2;
    if (took_host) {
        CK(cudaMemcpyAsync(took_host, took, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
    }
    return LMPC_OK;
}

// ================================================================================================
// controller snapshots (snapshot.cuh): one byte record per controller
// ================================================================================================
}  // extern "C" (the helpers below have C++ linkage)

static const char* snap_field_name(int f) {
    static const char* names[SF_NFIELD] = {
        "magic", "version", "record bytes", "N", "numSS_Points", "ncx", "ncu", "numSS_it", "trToUse", "ss_cap", "model_cap", "Tmax",
        "Tcl", "warm_start", "warm_mode", "nsect", "section table", "track row", "safe-set lap length", "model lap length", "it",
        "safe-set lap number", "md_cnt", "model arrival number", "lap_n", "sel", "is_prev", "prev_slot", "used", "timeStep",
        "has_pred", "warm_valid", "cl_len", "done", "lap report layout", "lap report count", "lane key", "lane margin layout", "lane margin"};
    return f >= 0 && f < SF_NFIELD ? names[f] : "?";
}

// The record layout of this handle: copy table t (handle buffers, record offsets, word sizes, chunks) and header hd (layout ints,
// section offsets; the track row and warm_mode are per pack).  The sections are the allocated rows of dev_bufs that name one.
static void snap_layout(lmpc_handle* h, SnapTable& t, lmpc_snapshot_header& hd) {
    memset(&t, 0, sizeof(t));
    memset(&hd, 0, sizeof(hd));
    for (const DevBuf& r : dev_bufs(h))
        for (int k = 0; r.sect != SN_SCRATCH && *r.p && k < r.rows; ++k) {     // row k of a [rows][B][per] buffer
            SnapSect& e = t.s[r.sect + k];
            e.stride = e.bytes = (int)(r.elem * r.per);
            e.base = (char*)*r.p + k * r.bytes(h->batch) / r.rows;
        }
    auto up16 = [](long long v) { return (v + 15) / 16 * 16; };
    long long off = up16(sizeof(lmpc_snapshot_header));
    for (int s = 0; s < SN_COUNT; ++s) {
        if (!t.s[s].bytes) continue;
        t.s[s].rec_off = (int)off;
        hd.sect_off[s] = (int)off;
        hd.sect_bytes[s] = t.s[s].bytes;
        off += up16(t.s[s].bytes);
    }
    t.s[SN_HEADER].base = (char*)h->d_snap;                       // the handle's header template
    t.s[SN_HEADER].bytes = SNAP_HDR_WORDS * 4;
    t.s[SN_HEADER].pack_only = 1;
    t.s[SN_TRACK].base = (char*)h->trk.tab;
    t.s[SN_TRACK].idx = h->trk.idx;
    t.s[SN_TRACK].stride = h->trk.idx ? sizeof(TrackRec) : 0;
    t.s[SN_TRACK].bytes = sizeof(TrackRec);
    t.s[SN_TRACK].rec_off = SNAP_HDR_WORDS * 4;
    t.s[SN_TRACK].pack_only = 1;
    for (int s = 0; s < SN_TABLE; ++s) {
        SnapSect& e = t.s[s];
        // every address a thread touches is base + k * stride + rec_off-relative offset: the word must divide all four (the
        // second row of a [2][B] buffer, for one, is only 4-byte aligned under an odd batch)
        const long long all = e.bytes | e.stride | e.rec_off | (long long)(uintptr_t)e.base;
        e.word = (all % 16 == 0) ? 16 : (all % 8 == 0) ? 8 : 4;
    }
    t.chunk_bytes = 16 << 10;
    for (;;) {
        int n = 0;
        for (int s = 0; s < SN_TABLE; ++s) n += (t.s[s].bytes + t.chunk_bytes - 1) / t.chunk_bytes;
        if (n <= SNAP_MAXCHUNK) break;
        t.chunk_bytes *= 2;
    }
    for (int s = 0; s < SN_TABLE; ++s)
        for (int c = 0; c * (long long)t.chunk_bytes < t.s[s].bytes; ++c) {
            t.chunk_sect[t.nchunk] = (unsigned short)s;
            t.chunk_no[t.nchunk] = (unsigned short)c;
            ++t.nchunk;
        }
    hd.magic = LMPC_SNAPSHOT_MAGIC; hd.version = LMPC_SNAPSHOT_VERSION; hd.bytes = (int)off;
    hd.N = h->N; hd.M = h->M; hd.ncx = h->p.ncx; hd.ncu = h->p.ncu; hd.numSS_it = h->bk.numSS_it; hd.trToUse = h->bk.trToUse;
    hd.ss_cap = h->ss.cap; hd.model_cap = h->mdl.cap; hd.Tmax = h->ss.Tmax; hd.Tcl = h->has_rollout ? h->Tcl : 0;
    hd.warm_start = h->d_warm ? 1 : 0;
    hd.warm_mode = h->d_warm ? h->warm_mode : -1;
    hd.nsect = LMPC_SNAPSHOT_SECTIONS;
}

// Release the index scratch of a pack / unpack when e is an error, or always (`always`); report e, else the release's error
static int snap_release(lmpc_handle* h, int* d_idx, cudaError_t e, bool always) {
    if (e == cudaSuccess && !always) return LMPC_OK;
    const cudaError_t f = cudaFreeAsync(d_idx, h->stream);
    if (e == cudaSuccess) e = f;
    if (e != cudaSuccess) return fail(LMPC_E_CUDA, std::string("snapshot index scratch: ") + cudaGetErrorString(e));
    return LMPC_OK;
}

// Upload the controller indices (and record indices) of one pack / unpack to stream-ordered scratch of their own
static int snap_indices(lmpc_handle* h, const std::vector<int>& idx, int** d_idx) {
    CK(cudaMallocAsync((void**)d_idx, sizeof(int) * idx.size(), h->stream));
    return snap_release(h, *d_idx, cudaMemcpyAsync(*d_idx, idx.data(), sizeof(int) * idx.size(), cudaMemcpyHostToDevice, h->stream),
                        false);
}

extern "C" {

int lmpc_sizeof_snapshot_header(void) { return (int)sizeof(lmpc_snapshot_header); }

int lmpc_snapshot_bytes(lmpc_handle* h, size_t* bytes) {
    if (int rc = need_store(h)) return rc;
    if (!bytes) return fail(LMPC_E_INVALID, "null output");
    SnapTable t;
    lmpc_snapshot_header hd;
    snap_layout(h, t, hd);
    *bytes = (size_t)hd.bytes;
    return LMPC_OK;
}

int lmpc_snapshot_pack_dev(lmpc_handle* h, int n, const int* inst_host, void* rec_dev) {
    static const char* who = "lmpc_snapshot_pack_dev";
    int rc = need_store(h);
    if (rc) return rc;
    if (!rec_dev || n < 1) return fail(LMPC_E_INVALID, std::string(who) + ": null records or n < 1");
    if (!inst_host && n != h->batch) return fail(LMPC_E_INVALID, std::string(who) + ": NULL controllers means every controller (n == batch)");
    if ((rc = check_align(rec_dev, "the record buffer")) != LMPC_OK) return rc;
    std::vector<int> idx(n);
    for (int i = 0; i < n; ++i) {
        idx[i] = inst_host ? inst_host[i] : i;
        if (idx[i] < 0 || idx[i] >= h->batch)
            return fail(LMPC_E_INVALID, std::string(who) + ": controller index " + std::to_string(i) + " out of range");
    }
    SnapTable t;
    lmpc_snapshot_header hd;
    snap_layout(h, t, hd);
    // the header template, staged from the stack (pageable memory: the copy has left it when the call returns)
    CK(cudaMemcpyAsync(h->d_snap, &hd, SNAP_HDR_WORDS * 4, cudaMemcpyHostToDevice, h->stream));
    int* d_idx = nullptr;
    if ((rc = snap_indices(h, idx, &d_idx)) != LMPC_OK) return rc;
    snapshot_copy_kernel<<<dim3(n, t.nchunk), 256, 0, h->stream>>>(t, 0, d_idx, nullptr, (char*)rec_dev, hd.bytes);
    if ((rc = snap_release(h, d_idx, cudaGetLastError(), true)) != LMPC_OK) return rc;
    h->launches += 1;
    return LMPC_OK;
}

int lmpc_snapshot_unpack_dev(lmpc_handle* h, const void* rec_dev, int nrec, int n, const int* dst_host, const int* rec_of_dst_host) {
    static const char* who = "lmpc_snapshot_unpack_dev";
    int rc = need_store(h);
    if (rc) return rc;
    const std::string w = std::string(who) + ": ";
    if (!rec_dev || !dst_host || nrec < 1 || n < 1 || n > h->batch)
        return fail(LMPC_E_INVALID, w + "null records or destinations, nrec < 1, or n not in 1 .. batch");
    if ((rc = check_align(rec_dev, "the record buffer")) != LMPC_OK) return rc;
    std::vector<int> idx(2 * (size_t)n);               // destinations [n] | records [n]
    std::vector<char> seen(h->batch, 0);
    for (int i = 0; i < n; ++i) {
        const int d = dst_host[i], r = rec_of_dst_host ? rec_of_dst_host[i] : i;
        if (d < 0 || d >= h->batch) return fail(LMPC_E_INVALID, w + "destination " + std::to_string(i) + " out of range");
        if (seen[d]) return fail(LMPC_E_INVALID, w + "controller " + std::to_string(d) + " is a destination twice");
        if (r < 0 || r >= nrec) return fail(LMPC_E_INVALID, w + "record index of destination " + std::to_string(i) + " out of range");
        seen[d] = 1;
        idx[i] = d;
        idx[n + i] = r;
    }
    SnapTable t;
    lmpc_snapshot_header hd;
    snap_layout(h, t, hd);
    int* verdict = h->d_snap + SNAP_HDR_WORDS;
    const int init[3] = {INT32_MAX, INT32_MAX, INT32_MIN};
    CK(cudaMemcpyAsync(h->d_snap, &hd, SNAP_HDR_WORDS * 4, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(verdict, init, sizeof(init), cudaMemcpyHostToDevice, h->stream));
    int* d_idx = nullptr;
    if ((rc = snap_indices(h, idx, &d_idx)) != LMPC_OK) return rc;
    SnapCheckArgs a;
    a.hdr = h->d_snap;
    for (int s = 0; s < SN_COUNT; ++s) a.rec_off[s] = t.s[s].rec_off;
    a.trk = tracks(h);
    a.ss_cap = h->ss.cap; a.md_cap = h->mdl.cap; a.numSS_it = h->bk.numSS_it; a.trToUse = h->bk.trToUse; a.Tmax = h->ss.Tmax;
    a.Tcl = hd.Tcl; a.warm_mode = hd.warm_mode;
    a.lane = h->lrule.view();
    a.margin = h->lmar.view();
    snapshot_check_kernel<<<(n + 127) / 128, 128, 0, h->stream>>>(a, n, d_idx, d_idx + n, (const char*)rec_dev, hd.bytes, verdict);
    h->launches += 1;
    int got[3];
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(got, verdict, sizeof(got), cudaMemcpyDeviceToHost, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) {
        cudaFreeAsync(d_idx, h->stream);
        return fail(LMPC_E_CUDA, w + "record check: " + cudaGetErrorString(e));
    }
    int mode = h->warm_mode;
    std::string why;
    if (got[0] != INT32_MAX) {
        const int i = got[0] / 64, f = got[0] % 64;
        why = "record " + std::to_string(idx[n + i]) + " (into controller " + std::to_string(idx[i]) + "): " + snap_field_name(f) +
              (f <= SF_SECTIONS || f == SF_LAP_REPORTS || f == SF_LANE_MARGIN_LAYOUT ? " differs from this handle's" : f == SF_TRACK ? " differs from the controller's track"
               : f == SF_LANE_KEY ? " marks a lane-unsafe lap of a controller whose lane rule is off" : " out of range");
    } else if (h->d_warm && got[1] <= got[2]) {
        if (h->warm_mode < 0 && got[1] != got[2]) why = "the records hold warm-start records of two problem types";
        else mode = got[1];
    }
    if (!why.empty()) {
        cudaFreeAsync(d_idx, h->stream);
        return fail(LMPC_E_INVALID, w + why + "; nothing was restored");
    }
    snapshot_copy_kernel<<<dim3(n, t.nchunk), 256, 0, h->stream>>>(t, 1, d_idx, d_idx + n, (char*)rec_dev, hd.bytes);
    if ((rc = snap_release(h, d_idx, cudaGetLastError(), true)) != LMPC_OK) return rc;
    h->launches += 1;
    h->laps_stored = true;
    if (h->d_warm) h->warm_mode = mode;
    return lane_margin_rows(h, false);      // the restored margins plan from here on
}

int lmpc_rollout_get_clock(lmpc_handle* h, unsigned long long* step) {
    if (int rc = need_rollout(h)) return rc;
    if (!step) return fail(LMPC_E_INVALID, "null output");
    *step = h->sim_step;
    return LMPC_OK;
}

int lmpc_rollout_set_clock(lmpc_handle* h, unsigned long long step) {
    if (int rc = need_rollout(h)) return rc;
    h->sim_step = step;
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
    if (int rc = need_rollout(h)) return rc;
    if (h->has_trace) return fail(LMPC_E_STATE, "trace buffers already created");
    if (n < 1 || n > 1024 || !inst || cap_steps < 1) return fail(LMPC_E_INVALID, "bad trace arguments");
    for (int i = 0; i < n; ++i) if (inst[i] < 0 || inst[i] >= h->batch) return fail(LMPC_E_INVALID, "traced controller out of range");
    TraceBufs& t = h->tr;
    t.n = n; t.cap = cap_steps; t.N = h->N; t.M = h->M > 0 ? h->M : 0;
    const std::vector<DevBuf> rows = dev_bufs(h);
    int rc = alloc_bufs(h, rows, OWN_TRACE, n, "lmpc_rollout_trace_create");
    if (rc != LMPC_OK) return rc;
    cudaError_t e = cudaMemcpyAsync(h->d_trinst, inst, sizeof(int) * n, cudaMemcpyHostToDevice, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) {
        free_bufs(rows, OWN_TRACE);
        return fail(LMPC_E_CUDA, std::string("lmpc_rollout_trace_create: ") + cudaGetErrorString(e));
    }
    t.inst = h->d_trinst;
    h->has_trace = true;
    return LMPC_OK;
}

int lmpc_rollout_trace_get(lmpc_handle* h, int tr, int* steps, double* x, double* xglob, double* u, double* xPred, double* SS_sel, int* lap) {
    if (int rc = need_rollout(h)) return rc;
    if (!h->has_trace || tr < 0 || tr >= h->tr.n || !steps) return fail(LMPC_E_INVALID, "no such trace");
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
