/* include/lmpc_b200.h — C ABI of liblmpc_b200.so (H100 / sm_90a batched LMPC hot path).
 *
 * The reference (urosolia/RacingLMPC) is pure Python and has no FFI; its drop-in boundary is the
 * duck-typed controller protocol  solve(x0) / addPoint(x,u) / addTrajectory(x,u,x_glob)  with results
 * read back as attributes (src/fnc/simulator/SysModel.py:34-38, src/main.py:110,117).  This header is
 * the native surface a ctypes shim (racinglmpc_b200/PredictiveControllers.py) binds to reproduce that
 * protocol for a BATCH of independent controllers.  Each entry point cites the reference code it
 * replaces.  Conventions:
 *   - plain C types only; all arrays are contiguous, row-major, fp64 unless stated, int32 indices;
 *   - `_host` entry points take HOST pointers and perform the H2D/D2H copies themselves (pinned staging
 *     buffers inside the handle); `_dev` entry points take DEVICE pointers and only enqueue work on the
 *     handle's stream (call lmpc_sync() before reading results);
 *   - return value 0 = ok, negative = error code below; no exceptions, no global state; a handle is
 *     not thread-safe; the library never falls back to a CPU path.
 */
#ifndef LMPC_B200_H
#define LMPC_B200_H
#ifdef __cplusplus
extern "C" {
#endif

#define LMPC_OK 0
#define LMPC_E_INVALID -1      /* bad argument / unsupported size                     */
#define LMPC_E_CUDA -2         /* CUDA runtime error (lmpc_last_error() has the text) */
#define LMPC_E_NODEVICE -3     /* no sm_90 (H100-class) device available              */
#define LMPC_E_STATE -4        /* call sequence error (e.g. solve before addTrajectory) */

/* per-instance solver status written to status[] (racinglmpc_b200/csrc/ftocp_pdip.cuh) */
#define LMPC_ST_SOLVED 1       /* == OSQP status_val 1 -> reference `feasible = 1` (PC.py:279-282) */
#define LMPC_ST_MAX_ITER 2
#define LMPC_ST_NUMERICAL 3
#define LMPC_ST_BAD_INPUT 4

#define LMPC_MAX_NCX 4
#define LMPC_MAX_NCU 8
#define LMPC_MAX_SEG 16
#define LMPC_MAX_POOL_GROUPS 64

/* Controller parameters.  Field names/meaning follow MPCParams (PredictiveControllers.py:24-51) and the
 * extra LMPC constructor arguments (PredictiveControllers.py:293).  n = 6, d = 2 are fixed (the
 * reference's vehicle model, PredictiveModel.py:28-30 is hard-wired to them as well). */
typedef struct lmpc_params {
    int N;                        /* horizon                                   MPCParams.N        */
    int ncx, ncu;                 /* rows of Fx (<=4) and Fu (<=8)                                */
    double Q[36], R[4], Qf[36];   /* stage / terminal weights                  MPCParams.Q,R,Qf   */
    double dR[2];                 /* input-rate weight                         MPCParams.dR       */
    double Qslack[2];             /* [quadratic, linear] lane-slack cost (order as used at PC.py:249-250) */
    double xRef[6];               /*                                           MPCParams.xRef     */
    double Fx[LMPC_MAX_NCX * 6], bx[LMPC_MAX_NCX];   /* Fx x <= bx (soft)      MPCParams.Fx,bx    */
    double Fu[LMPC_MAX_NCU * 2], bu[LMPC_MAX_NCU];   /* Fu u <= bu             MPCParams.Fu,bu    */
    int numSS_Points, numSS_it;   /* 0,0 for a plain MPC                       LMPC.__init__      */
    double QterminalSlack[36];    /*                                           LMPC.__init__      */
    /* interior-point settings (no reference counterpart; OSQP's eps are 1e-3 + polish, PC.py:275) */
    double eps_res, eps_gap;      /* <= 0 selects the defaults 1e-9 / 1e-11 (unscaled inf-norms); an instance still
                                     running at iteration 20 is reported solved once all three are <= 1e-6 (safety
                                     net; counted by lmpc_late_accepts, 0 on every recorded workload) */
    int max_iter;                 /* <= 0 selects the default 40               */
    int warm_start;               /* != 0: the controllers of the device-resident step (lmpc_step_* / lmpc_rollout_step) start each
                                     solve from a mid-path interior-point iterate of their previous solve, shifted by one stage
                                     (SURVEY §8f rank 2).  The reference always starts cold (PC.py:124,276: `initvals` unused);
                                     the optimum returned is the same, only the iteration count changes.  A warm start that is
                                     not through after min(16, max_iter) iterations restarts cold inside the same solve, with
                                     the full max_iter of its own (at most min(16, max_iter) + max_iter iterations in all), and
                                     the record is dropped.  0 = cold start. */
    double eps_step;              /* <= 0 selects the default 1e-7: besides the residuals, the last primal step
                                     |alpha (dx, du)|_inf must be below it -- on QPs without strict complementarity the
                                     iterate is O(sqrt(gap)) from the optimum while the residuals are already tiny */
} lmpc_params;

/* Local-regression model parameters: PredictiveModel.__init__ (PredictiveModel.py:12-32) and the
 * track table consumed by Map.curvature (Track.py:292-310). */
typedef struct lmpc_model_params {
    int trToUse;                  /* number of stored laps used     PredictiveModel.usedIt     */
    int MaxNumPoint;              /* 7                              PredictiveModel.MaxNumPoint */
    double h, lamb, dt;           /* 5, 0.0, 0.1                                               */
    double scaling[5];            /* diag(0.1,1,1,1,1)              PredictiveModel.scaling     */
    int nseg;                     /* rows of the track table                                   */
    double seg[LMPC_MAX_SEG * 3]; /* [s_start, length, curvature] = Map.PointAndTangent[:,3:6]  */
    double TrackLength;
} lmpc_model_params;

typedef struct lmpc_handle lmpc_handle;

const char* lmpc_last_error(void);
int lmpc_device_count(void);

/* One handle = `batch` independent controllers on one device, created with identical parameters (see lmpc_set_param_sets for
 * parameter sweeps in one batch). */
int lmpc_create(const lmpc_params* p, int batch, int device, lmpc_handle** out);
/* Per-controller QP parameters (parameter sweeps in one batch; no reference counterpart: the reference runs one controller).
 * sets[nsets] are full lmpc_params; controller b solves its QPs with sets[set_of_instance[b]] (host array [batch]).  Applies to every
 * QP the handle solves: the _host / _host_async / _dev entry points, lmpc_step_* and lmpc_rollout_step.  nsets == 0 (sets,
 * set_of_instance NULL) returns the handle to the parameters it was created with.
 *   - 1 <= nsets <= batch, every index in [0, nsets).
 *   - Every set equals the handle's parameters in N, ncx, ncu, numSS_Points, numSS_it and warm_start; all other fields (weights,
 *     xRef, Fx/bx, Fu/bu, QterminalSlack, tolerances, max_iter) may differ.  Each set is checked and converted as lmpc_create does
 *     it (bu > 0, invertible QterminalSlack when numSS_Points > 0, values <= 0 select the default tolerances).
 *   - Any failed check returns LMPC_E_INVALID and leaves the handle as it was.
 *   - The call synchronises the handle's streams before it replaces the table: batches enqueued earlier (e.g. through the _async
 *     entry points) complete with the parameters they were enqueued with.
 *   - It invalidates the warm-start records (lmpc_params.warm_start): the next solve of every controller starts cold.
 *   - The pooled safe-set exchange (lmpc_pool_*) hands laps between the controllers of one pool group (lmpc_set_pool_groups)
 *     whatever their set; a clean sweep (each tuning learning from its own tuning's laps only) puts each set in its own group.
 *     lmpc_ss_import_laps_dev hands laps wherever the caller says.
 * A handle with sets installed launches a QP kernel variant that stages the instance's parameter record (1 776 B) in shared
 * memory next to its stage model (DESIGN.md, "Per-controller parameters"); handles without sets launch the uniform kernel. */
int lmpc_set_param_sets(lmpc_handle* h, const lmpc_params* sets, int nsets, const int* set_of_instance);
int lmpc_destroy(lmpc_handle* h);
int lmpc_sync(lmpc_handle* h);
void* lmpc_stream(lmpc_handle* h);            /* cudaStream_t the handle enqueues on */
long long lmpc_kernel_launches(lmpc_handle* h); /* kernels launched by this handle so far */
/* Number of QPs (since lmpc_create) that were reported LMPC_ST_SOLVED by the late-acceptance safety net of the interior-point
 * loop -- residuals and gap <= 1e-6 at iteration >= 20 / at max_iter -- instead of at eps_res / eps_gap (see lmpc_params).
 * Synchronises the handle's streams; -1 on error.  0 on every recorded BASELINE workload (tests assert it). */
long long lmpc_late_accepts(lmpc_handle* h);

/* Pinned host memory for the arrays handed to the `_host` / `_host_async` entry points (no reference counterpart: NumPy arrays
 * in the reference never leave the host).  The pages are placed on the NUMA node the device's PCIe link hangs off
 * (/sys/bus/pci/devices/<bus id>/numa_node; an anonymous mapping bound with mbind(MPOL_PREFERRED), touched, then pinned with
 * cudaHostRegister), which is what a single DMA stream needs to run at link rate on a multi-socket host; zero-filled.
 * lmpc_host_numa_node: that node, -1 = unknown / switched off with LMPC_B200_NUMA=off (LMPC_B200_NUMA=<n> forces node n).
 * lmpc_host_page_nodes: node of n (<= 64) evenly sampled pages of a block (diagnostics; -1 = unknown, on hosts that forbid the
 * move_pages query).  Plain pinned or pageable arrays remain
 * valid arguments of every entry point. */
int lmpc_host_alloc(int device, size_t bytes, void** out);
int lmpc_host_free(void* p);
int lmpc_host_numa_node(int device);
int lmpc_host_page_nodes(const void* p, size_t bytes, int n, int* nodes_out);

/* ---- FTOCP solve with the model given by the caller ("fixed A/B/C") ---------------------------------
 * Replaces, per instance: buildCost + buildEqConstr + addTerminalComponents + osqp_solve_qp +
 * unpackSolution (PredictiveControllers.py:110-137,200-283) for an MPC-type problem (no safe set).
 *   x0[B,6], uOld[B,2]            current state, previously applied input (OldInput, PC.py:136)
 *   abc                           stage model, per stage [A(36) row-major | B(12) | C(6)] = 54 doubles
 *   abc_inst_stride / abc_stage_stride   in doubles; (N*54, 54) = per-instance LTV (PC.py:212-215),
 *                                 (0, 0) = one LTI model shared by all (PC.py:216-218, C = 0 is the caller's job)
 * Outputs (caller-allocated): xPred[B,N+1,6], uPred[B,N,2] (PC.py:163-164), slack[B,N*ncx] or NULL,
 *   status[B] int32, iters[B] int32, resid[B,3] = (r_prim, r_dual, gap) in the unscaled inf-norm.
 */
int lmpc_solve_mpc_host(lmpc_handle* h, const double* x0, const double* uOld, const double* abc,
                        long long abc_inst_stride, long long abc_stage_stride, double* xPred, double* uPred,
                        double* slack, int* status, int* iters, double* resid);
int lmpc_solve_mpc_dev(lmpc_handle* h, const double* x0, const double* uOld, const double* abc,
                       long long abc_inst_stride, long long abc_stage_stride, double* xPred, double* uPred,
                       double* slack, int* status, int* iters, double* resid);

/* ---- FTOCP solve with a sampled safe set given by the caller -------------------------------------------
 * Adds addSafeSetEqConstr/addSafeSetCost + LMPC.unpackSolution + feasibleStateInput
 * (PredictiveControllers.py:345-384).  M = numSS_Points.
 *   SS_sel[B,6,M], Qfun_sel[B,M]          SS_PointSelectedTot, Qfun_SelectedTot (PC.py:411-412)
 *   Succ_SS[B,6,M], Succ_uSS[B,2,M]       successor states/inputs (PC.py:409-410), may be NULL
 * Extra outputs: lambd[B,M] (PC.py:374), slackTerminal[B,6] (PC.py:375) or NULL,
 *   zt[B,6], zt_u[B,2] (PC.py:383-384) or NULL when Succ_* are NULL.
 */
int lmpc_solve_lmpc_host(lmpc_handle* h, const double* x0, const double* uOld, const double* abc,
                         long long abc_inst_stride, long long abc_stage_stride, const double* SS_sel,
                         const double* Qfun_sel, const double* Succ_SS, const double* Succ_uSS, double* xPred,
                         double* uPred, double* slack, double* lambd, double* slackTerminal, double* zt,
                         double* zt_u, int* status, int* iters, double* resid);
/* Asynchronous forms of the two *_host entry points, for streaming batch after batch: the call enqueues the copies and the
 * solve on buffer set `slot` (0 .. 3; the further sets of device buffers are allocated on first use) and returns;
 * lmpc_host_wait(h, slot) returns once the results of that slot are in the caller's output arrays.  With two batches in
 * flight the H2D copy of one overlaps the solve of the other; a third keeps the copy engine busy while the host waits for the
 * oldest batch and enqueues the next (measured: 8.7 -> see DESIGN §4 M solves/s on configs[1]).  All host arrays must stay valid (and should be pinned) until
 * the wait; a slot must be waited for before it is reused.  lmpc_solve_*_host == *_async(slot 0) + lmpc_host_wait(0). */
int lmpc_solve_mpc_host_async(lmpc_handle* h, int slot, const double* x0, const double* uOld, const double* abc,
                              long long abc_inst_stride, long long abc_stage_stride, double* xPred, double* uPred,
                              double* slack, int* status, int* iters, double* resid);
int lmpc_solve_lmpc_host_async(lmpc_handle* h, int slot, const double* x0, const double* uOld, const double* abc,
                               long long abc_inst_stride, long long abc_stage_stride, const double* SS_sel,
                               const double* Qfun_sel, const double* Succ_SS, const double* Succ_uSS, double* xPred,
                               double* uPred, double* slack, double* lambd, double* slackTerminal, double* zt,
                               double* zt_u, int* status, int* iters, double* resid);
int lmpc_host_wait(lmpc_handle* h, int slot);
/* Instance ranges (1 .. 4, each on its own stream: H2D | solve | D2H overlap inside one batch) the most recent enqueue on `slot`
 * was cut into: 4 for a batch of >= 2048 QPs solved through the synchronous entry points; through the asynchronous ones 1 when
 * another buffer set is in flight (the overlap then comes from the other batches, and fewer, larger pieces cost the enqueueing
 * thread less), else 2.
 * Diagnostics; -1 on a bad argument. */
int lmpc_host_chunks(lmpc_handle* h, int slot);
int lmpc_solve_lmpc_dev(lmpc_handle* h, const double* x0, const double* uOld, const double* abc,
                        long long abc_inst_stride, long long abc_stage_stride, const double* SS_sel,
                        const double* Qfun_sel, const double* Succ_SS, const double* Succ_uSS, double* xPred,
                        double* uPred, double* slack, double* lambd, double* slackTerminal, double* zt,
                        double* zt_u, int* status, int* iters, double* resid);

/* ===== device-resident lap stores, k-NN regression, safe-set selection, fused controller step =========
 *
 * lmpc_store_create: allocates, per instance, `ss_cap` safe-set lap slots (x[T,6], u[T,2], Qfun[T]) and
 * `model_cap` regression lap slots (x, u) of at most Tmax rows, plus the controller state
 * (xLin, uLin, zt, OldInput, timeStep, previous xPred) that MPC/LMPC keep between solves (PC.py:88-93,129-137,330).
 * Which slots are "the numSS_it fastest laps" (PC.py:395-402) and "usedIt" (PredictiveModel.py:31,35-46) is
 * decided by the host shim at addTrajectory time (once per lap) and passed as small index arrays.
 */
int lmpc_store_create(lmpc_handle* h, const lmpc_model_params* mp, int ss_cap, int model_cap, int Tmax);

/* A circuit: the table Map.curvature reads (Track.py:292-310) and the lap length. */
typedef struct lmpc_track_params {
    int nseg;                         /* rows of the table, 1 .. LMPC_MAX_SEG                        */
    double seg[LMPC_MAX_SEG * 3];     /* [s_start, length, curvature] = Map.PointAndTangent[:,3:6]   */
    double TrackLength;
} lmpc_track_params;
/* Per-controller tracks (several circuits in one batch; no reference counterpart: the reference drives one track).  Controller b
 * uses sets[set_of_instance[b]] (host arrays) in every later regression (curvature), safe-set selection (lap-wrap fix, Q-function
 * shift), addPoint, lap cost, lap hand-over and simulator launch, host-driven and device-resident alike.  nsets == 0 (sets,
 * set_of_instance NULL) returns every controller to the track of lmpc_store_create, which every store starts with.
 *   - Requires lmpc_store_create (else LMPC_E_STATE), and no lap stored yet in either pool by any entry point (put_lap, seeding,
 *     commit, import; else LMPC_E_STATE): a stored lap is in the s-coordinate of the track it was driven on.
 *   - 1 <= nsets <= batch, every index in [0, nsets); per set: 1 <= nseg <= LMPC_MAX_SEG, all values finite, lengths >= 0,
 *     seg start 0 == 0, start i == start i-1 + length i-1 exactly, TrackLength == start + length of the last row exactly and > 0
 *     (the way Track.py:54-133 builds the table).  Any failed check returns LMPC_E_INVALID and leaves the handle as it was.
 *   - The call synchronises the handle's streams before it replaces the table.
 *   - The track index is independent of the parameter-set and the vehicle index (crossed designs work).  The lane half-width
 *     enters the QP through Fx/bx (lmpc_set_param_sets), not through this table.
 *   - While more than one set is installed, a lap driven on another circuit is not a trajectory of this one: the pooled exchange
 *     (lmpc_pool_export_dev, lmpc_pool_import_dev) returns LMPC_E_STATE unless pool groups are installed and the controllers of
 *     every group on this rank share one track index; lmpc_ss_import_laps_dev always returns LMPC_E_STATE. */
int lmpc_set_tracks(lmpc_handle* h, const lmpc_track_params* sets, int nsets, const int* set_of_instance);

/* The constants of the local regression model (PredictiveModel.py:18-31): the regression constants of lmpc_model_params. */
typedef struct lmpc_regression_params {
    int trToUse;                  /* stored laps used: 1 for the LTV-MPC, 4 for LMPC  main.py:88,102; PM.py:31 */
    int MaxNumPoint;              /* 7                                               PM.py:18              */
    double h, lamb;               /* 5, 0.0                                          PM.py:19-20           */
    double scaling[5];            /* diag(0.1,1,1,1,1)                               PM.py:22-26           */
} lmpc_regression_params;
/* Per-controller regression models (studies of the learned model's settings in one batch; no reference counterpart: the reference
 * builds one PredictiveModel per controller).  Controller b regresses with sets[set_of_instance[b]] (host arrays) in every later
 * K1 launch -- lmpc_identify_host, lmpc_step_*, lmpc_rollout_step -- host-driven and device-resident alike.  nsets == 0 (sets,
 * set_of_instance NULL) returns every controller to the constants of lmpc_store_create, which every store starts with.
 *   - Requires lmpc_store_create (else LMPC_E_STATE).
 *   - 1 <= nsets <= batch, every index in [0, nsets).  Per set: 1 <= trToUse <= the store's trToUse; 1 <= MaxNumPoint <= 7;
 *     h finite, 2^-1022 <= h <= 2^1022 (a normal bandwidth with a normal reciprocal); lamb finite and >= 0; every scaling entry
 *     finite with |s| == 0 or 2^-32 <= |s| <= 2^32, taken as |s| as lmpc_store_create does (the range in which the fp32
 *     pre-filter of the neighbour scan is certified: DESIGN.md, "Per-controller regression models").  Any failed check returns
 *     LMPC_E_INVALID and leaves the handle as it was.
 *   - The store's trToUse still sizes the lap books, the regression scratch and the snapshot record.  A set with a smaller
 *     trToUse regresses on the first trToUse entries of the controller's usedIt list: its trToUse shortest laps, which is what a
 *     store created with that trToUse selects (PM.py:31,35-46).
 *   - The call synchronises the handle's streams before it replaces the table.  It is allowed at any time: a change applies from
 *     the next regression on; warm-start records stay (the QP's optimum does not depend on them).
 *   - The regression index is independent of the parameter-set, vehicle, track, noise and pool-group indices.  The pooled
 *     exchange does not look at it: a lap driven under another model setting is still a trajectory of this car on this circuit.
 *   - dt stays per handle (it is the simulator's control period too).  Sets stay with the handle: the snapshot record does not
 *     carry them. */
int lmpc_set_regression_sets(lmpc_handle* h, const lmpc_regression_params* sets, int nsets, const int* set_of_instance);

/* Per-controller shape: the horizon N and the safe-set size numSS_Points (numSS_Points / numSS_it points per lap). */
typedef struct lmpc_shape_params {
    int N, numSS_Points;
} lmpc_shape_params;
/* Per-controller horizons and safe-set sizes (the horizon / safe-set trade-off of Rosolia & Borrelli, TCST 2019, in one batch).
 * Controller b is controlled with the shape sets[set_of_instance[b]] (host arrays): its regression (K1), safe-set selection (K2),
 * QP and state shift work on N_b stages and M_b safe-set points.  nsets == 0 (sets, set_of_instance NULL) returns every controller
 * to the handle's own (N, numSS_Points).
 *   - Requires lmpc_store_create, and no lap stored yet in either pool (as lmpc_set_tracks; else LMPC_E_STATE): xLin, uLin and
 *     the previous prediction have the length of the horizon they were made for.  Refused on a handle created with warm_start
 *     (LMPC_E_STATE): the warm-start record is laid out per (N, M).
 *   - 1 <= nsets <= batch, every index in [0, nsets).  Per set: (N, numSS_Points) is a pair of the instantiated grid; N <= the
 *     handle's N and numSS_Points <= the handle's; numSS_Points > 0 exactly when the handle's is, a multiple of numSS_it with an
 *     even number of points per lap.  Any failed check returns LMPC_E_INVALID and leaves the handle as it was.
 *   - The call synchronises the handle's streams before it replaces the table.  It is independent of every other table; parameter
 *     sets keep the handle's N and numSS_Points (the weights do not depend on the horizon).
 *   - Honoured by lmpc_step_host / _dev / _profile, lmpc_identify_host, lmpc_select_host, lmpc_rollout_step (modes 0, 1, 2), the
 *     seeding calls and the trace.  While shapes are installed the caller-problem entry points (lmpc_solve_*) return LMPC_E_STATE:
 *     their arrays have no per-controller shape.  Shapes are not part of a snapshot record; records keep the handle's layout.
 * Layout: every buffer keeps the handle's N and numSS_Points as its per-controller stride, and a controller of shape (N_b, M_b) uses
 * the leading part of its region: a [N+1,6] / [N,2] block (xPred, uPred, xLin, uLin, the trace's xPred) holds N_b + 1 / N_b rows,
 * abc holds N_b stages, SS_sel / Succ_SS / Succ_uSS hold a row-major [6,M_b] / [2,M_b] block at the start of the controller's
 * region, Qfun_sel and lambd hold M_b entries.  A shaped controller never writes the tails.
 * A shaped handle runs one QP launch per distinct shape present (per distinct N for the MPC-type QPs of modes 0 and 2), each over
 * the controllers of that shape (DESIGN.md, "Per-controller horizons and safe-set sizes").
 * With a lap-count table installed (lmpc_set_ss_laps) every controller's numSS_Points must instead be its own numSS_it times an
 * even number of points per lap; a pair that breaks this is refused with LMPC_E_INVALID, whichever table is installed first. */
int lmpc_set_shapes(lmpc_handle* h, const lmpc_shape_params* sets, int nsets, const int* set_of_instance);

/* Per-controller safe-set lap count: numSS_it, the number of fastest past laps the sampled safe set draws from (PC.py:395-407). */
typedef struct lmpc_ss_laps_params {
    int numSS_it;
} lmpc_ss_laps_params;
/* Per-controller safe-set lap counts (how to split the safe set between laps and points per lap, in one batch).  Controller b
 * selects its safe set from its numSS_it_b = sets[set_of_instance[b]].numSS_it fastest laps, M_b / numSS_it_b points per lap, M_b
 * being its numSS_Points (lmpc_set_shapes, else the handle's).  nsets == 0 (sets, set_of_instance NULL) returns every controller
 * to the handle's numSS_it.
 *   - Requires lmpc_store_create and an LMPC handle (numSS_Points > 0), and no lap stored yet in either pool (as lmpc_set_tracks
 *     and lmpc_set_shapes; else LMPC_E_STATE): the lap books evict laps against the controller's value, so raising it later would
 *     select laps already gone, where the reference's unbounded lists still hold them.
 *   - 1 <= nsets <= batch, every index in [0, nsets).  Per set: 1 <= numSS_it <= the handle's numSS_it, which keeps sizing sel,
 *     is_prev, min_index, K2's block and the snapshot record.  Per controller: M_b is numSS_it_b times an even number of points per
 *     lap (checked against the installed shapes here, and by lmpc_set_shapes against this table).  Any failed check returns
 *     LMPC_E_INVALID and leaves the handle as it was.
 *   - The call synchronises the handle's streams before it replaces the table.
 *   - Honoured by lmpc_select_host, lmpc_step_host / _dev / _profile, lmpc_rollout_step mode 1, the device lap hand-over
 *     (lmpc_rollout_commit_laps_dev) and seeding (lmpc_rollout_seed_from_record_dev), lmpc_pool_import_dev (an importer ranks a
 *     lap against its own numSS_it_b; the exporter is unchanged, so pool groups may mix values) and lmpc_books_set.  The device
 *     books then rank, evict and flag (8: fewer than numSS_it_b laps; 64: pool too small) exactly as a handle created with
 *     numSS_it_b and the same ss_cap.  Seeding still stores the copies the caller asks for: a controller whose numSS_it_b exceeds
 *     them gets flag 8, as the handle does.
 *   - Layout: sel / is_prev / min_index keep the handle's numSS_it entries per controller.  Entries c < numSS_it_b are the
 *     controller's selection; entries c >= numSS_it_b of sel repeat its last selected slot and those of is_prev are 0 (valid and
 *     deterministic, so records pack and restore bit for bit); min_index keeps what it held there.  K2 writes columns
 *     c * P_b + l, P_b = M_b / numSS_it_b, of the controller's [6, M_b] block.
 *   - Unchanged: lmpc_set_param_sets still requires the handle's numSS_it, the snapshot header keeps the handle's value, and the
 *     table is not part of a snapshot record (restore a record into a controller of the same numSS_it_b to resume it). */
int lmpc_set_ss_laps(lmpc_handle* h, const lmpc_ss_laps_params* sets, int nsets, const int* set_of_instance);

/* Per-controller lap windows: how many of its most recent laps a controller's safe set and learned model draw from (0 =
 * unbounded, the reference's rule). */
typedef struct lmpc_lap_window_params {
    int ss_window;       /* safe set: lap numbers [it - ss_window, it) */
    int model_window;    /* regression model: arrival numbers [md_cnt - model_window, md_cnt) */
} lmpc_lap_window_params;
/* Per-controller lap windows (a controller that trusts only its recent laps, e.g. after the car or the track changed).
 * Controller b reads row sets[set_of_instance[b]].  nsets == 0 (sets, set_of_instance NULL) removes the table: every window is
 * unbounded again.
 *   - Safe set: with ss_window = W > 0 the selection is the stable argsort by (lap time, lap number) of the laps numbered
 *     [it - W, it), first numSS_it_b of them (the reference's order restricted to the window).  Lap it-1 is always in the window,
 *     so is_prev and prev_slot are unchanged; an import is still filed as lap it-1.
 *   - Model: with model_window = Wm > 0 usedIt is the first trToUse laps of the (length, arrival) order among arrival numbers
 *     [md_cnt - Wm, md_cnt); with fewer the slowest repeats, as without a window.
 *   - Storage: under a window a lap stays stored while it is in the window and fewer than numSS_it_b (trToUse) newer laps rank
 *     ahead of it; a new own lap is always stored, an import is left out of the safe set when it is outside the window on arrival
 *     (ss_window 1) or its newer laps already rank ahead of it numSS_it_b times.  Evicted among the laps that can no longer be
 *     selected: the slowest, then the oldest.  With ss_window <= ss_cap and model_window <= model_cap a window never sets health
 *     bit 64.  Without a window the books are exactly as before.
 *   - Requires lmpc_store_create and no lap stored yet in either pool (else LMPC_E_STATE): the books evict against the window,
 *     so a later change would need laps that are already gone.
 *   - 1 <= nsets <= batch, every index in [0, nsets).  Per set: ss_window is 0 or numSS_it_b .. ss_cap for every controller of
 *     the set (numSS_it_b: its value under lmpc_set_ss_laps, else the handle's), and 0 on a handle without a safe set;
 *     model_window is 0 or trToUse .. model_cap (the store's trToUse).  lmpc_set_ss_laps refuses a value above a controller's
 *     installed nonzero ss_window.  Any failed check returns LMPC_E_INVALID and leaves the handle as it was.
 *   - The call synchronises the handle's streams before it replaces the table.
 *   - Honoured by the device books (lmpc_rollout_commit_laps_dev, lmpc_rollout_seed_from_record_dev, lmpc_books_set and
 *     lmpc_pool_import_dev).  The pooled export is unchanged: it ships each controller's latest own lap.
 *   - Not part of a snapshot record (LMPC_SNAPSHOT_VERSION is unchanged): a record resumes exactly only under the same windows. */
int lmpc_set_lap_windows(lmpc_handle* h, const lmpc_lap_window_params* sets, int nsets, const int* set_of_instance);

/* Per-controller lane rules: whether a lap that left the lane may rank among the laps a controller's safe set draws from. */
#define LMPC_LANE_UNSAFE_KEY (1 << 24)       /* added to the safe-set key (ss_time) of a lap judged lane-unsafe */
#define LMPC_REPORT_LANE_UNSAFE (1 << 16)    /* report-only flag bit: the filed own lap was judged lane-unsafe */
typedef struct lmpc_lane_rule_params {
    int mode;            /* 0: the reference's rule (laps ranked by lap time alone); 1: every lap filed is judged */
    int pad;
    double lane_tol;     /* mode 1: a lap is lane-unsafe when a judged row leaves a lane row by more than lane_tol */
} lmpc_lane_rule_params;
/* Per-controller lane rules (LMPC's sampled safe set assumes laps that satisfy the constraints; the QP's lane is soft, so a lap
 * that crossed it is stored like any other and, being faster, is the first one selected).  Controller b reads row
 * sets[set_of_instance[b]].  nsets == 0 (sets, set_of_instance NULL) removes the table: every controller ranks by lap time.
 *   - Judgement (mode 1): a lap is lane-unsafe when one of its judged rows x has a non-finite entry, or when for a lane row i
 *     d_i = (sum over j = 0..5, in order, of Fx[i][j] * x[j], fp64 without fused multiply-adds) - bx[i] > lane_tol: the
 *     arithmetic of the lap reports (lmpc_rollout_enable_lap_reports) with the threshold lane_tol.  Fx, bx are the controller's
 *     untightened lane: its parameter-set row, else the handle's (not the lmpc_set_lane_margins planning lane).  Judged rows: an own lap's rows 0 .. Trec-1 of the closed-loop
 *     record at the hand-over (the rows the controller files: under measurement noise the measured states); the seeded record
 *     once for all its copies; an import's shipped rows 0 .. min(lap time, rows, Tpad)-1, against the importer's own Fx, bx and
 *     lane_tol (the export still chooses and ships by raw lap time).
 *   - Ranking: an unsafe lap is filed with the key ss_time = lap time + LMPC_LANE_UNSAFE_KEY, a safe one with its lap time.  The
 *     books compare (ss_time, lap number) as before, so the selection is the stable argsort by (unsafe, lap time, lap number),
 *     first numSS_it_b; unsafe laps still fill it when fewer safe laps exist (flag 8 and the storage rule are unchanged), and an
 *     unsafe own latest lap stays lap it-1 for addPoint.  The regression model (md_time, usedIt), lap_hist and the reports keep
 *     raw lengths.  The pooled export strips the offset for its ranking, its min_overrun test and meta[.,1].
 *   - Reports: the filed report of an own lap judged unsafe carries LMPC_REPORT_LANE_UNSAFE in its flags (the health word does
 *     not).
 *   - Requires lmpc_store_create and a safe set (numSS_Points > 0), and no lap stored yet in either pool, whether the call
 *     installs or removes (else LMPC_E_STATE).  1 <= nsets <= batch, every index in [0, nsets); mode 0 or 1, lane_tol finite and
 *     >= 0; with a mode 1 row, a rollout of Tcl >= LMPC_LANE_UNSAFE_KEY is refused.  Any failed check returns LMPC_E_INVALID
 *     and leaves the handle as it was.  The call synchronises the handle's streams before it replaces the table.
 *   - While a mode 1 row is installed, the host-slot paths (lmpc_rollout_commit_laps, lmpc_rollout_seed_from_record) return
 *     LMPC_E_STATE (they take the caller's books, which do not judge laps) and lmpc_rollout_create refuses Tcl >=
 *     LMPC_LANE_UNSAFE_KEY.  Keys >= LMPC_LANE_UNSAFE_KEY are only valid where a controller's rule is on: lmpc_books_set and
 *     lmpc_snapshot_unpack_dev (field "lane key") refuse an occupied slot with such a key for a controller whose rule is off.
 *   - Not part of a snapshot record (LMPC_SNAPSHOT_VERSION is unchanged): the keys travel in ss_time, so a record resumes exactly
 *     under the same rules. */
int lmpc_set_lane_rules(lmpc_handle* h, const lmpc_lane_rule_params* sets, int nsets, const int* set_of_instance);

/* Per-controller lane margins: the lane a controller plans in, narrowed by a margin m_b, apart from the lane it is judged against. */
typedef struct lmpc_lane_margin_params {
    int mode;            /* 0: no margin (the reference); 1: fixed margin0; 2: adaptive */
    int pad;
    double margin0;      /* mode 1: the margin; mode 2: the starting value and the floor */
    double margin_max;   /* mode 2: the ceiling */
    double step_up;      /* mode 2: added after a lap that left the lane */
    double step_down;    /* mode 2: removed after a lap that kept to it (0: the margin only ratchets up) */
} lmpc_lane_margin_params;
/* Per-controller lane margins (constraint tightening: the learned model is off by a few centimetres, so a plan that ends at the
 * lane's edge puts the plant over it).  Controller b reads row sets[set_of_instance[b]].  nsets == 0 (sets, set_of_instance NULL)
 * removes the table.
 *   - Margin m_b of every controller: 0 under mode 0, margin0 under mode 1; under mode 2 margin0 at the install and at every
 *     seeding (lmpc_rollout_seed_from_record(_dev)), then adapted at every own-lap hand-over of lmpc_rollout_commit_laps_dev: when
 *     the lap's recorded rows 0 .. Trec-1 (under measurement noise the measured states) leave the lane -- a row with a non-finite
 *     entry, or d_i > 0 with d_i the arithmetic of the lap reports -- m_b = fmin(m_b + step_up, margin_max), else m_b =
 *     fmax(m_b - step_down, margin0), each rounded once.  Imports, the PID lap and retired controllers leave m_b as it is.
 *   - Planning lane: every QP the handle solves (lmpc_solve_*, lmpc_step_*, lmpc_rollout_step, shaped handles included) plans
 *     controller b with bx_i - m_b for every lane row i < ncx at every stage; Fx, Fu, bu, the weights, K1 and K2 are unchanged.
 *   - Judged lane: the lap reports (viol_steps, viol_max), the lane rules and the mode 2 verdict judge against the untightened
 *     row: the controller's parameter-set row, else the handle's.
 *   - Requires lmpc_store_create (else LMPC_E_STATE).  1 <= nsets <= batch, every index in [0, nsets); mode 0, 1 or 2; every
 *     value finite and >= 0, margin0 <= margin_max; a margin must leave a lane: margin0 (mode 1) or margin_max (mode 2) below
 *     min_i bx_i of the QP row the controller reads (lmpc_set_param_sets refuses sets that break this for an installed table).  Any
 *     failed check returns LMPC_E_INVALID and leaves the handle as it was.  Allowed at any time; it synchronises the handle's
 *     streams.  Installing or removing the table invalidates every warm-start record; a hand-over that changes m_b invalidates
 *     that controller's.
 *   - While a mode 2 row is installed, lmpc_rollout_commit_laps returns LMPC_E_STATE (the host-slot hand-over does not adapt).
 *   - Memory: m_b (8 B) and a derived parameter row (the source row with the tightened bx, 1 776 B) per controller, with an
 *     identity index (4 B): 14.6 MB at batch 8192.
 *   - m_b is a snapshot section ("lane_margin", slot 39), absent without a table; lmpc_snapshot_unpack_dev refuses a record of
 *     the other layout ("lane margin layout") and a non-finite or negative value, or under mode 2 one outside [margin0,
 *     margin_max] ("lane margin"): the adaptation never leaves that range, so such a record was captured under another row.  The table itself is not part of a record, and the snapshot version is unchanged. */
int lmpc_set_lane_margins(lmpc_handle* h, const lmpc_lane_margin_params* sets, int nsets, const int* set_of_instance);
/* m[batch] = m_b of every controller (synchronises); LMPC_E_STATE without a table. */
int lmpc_get_lane_margins(lmpc_handle* h, double* m);

/* PredictiveModel.addTrajectory (PredictiveModel.py:35-46): copy one lap into a regression slot. */
int lmpc_model_put_lap(lmpc_handle* h, int inst, int slot, int T, const double* x, const double* u);
/* usedIt order: slots[B,trToUse]. */
int lmpc_model_set_used(lmpc_handle* h, const int* slots);

/* LMPC.addTrajectory (PC.py:418-445): copy one lap into a safe-set slot; qfun == NULL computes
 * LMPC.computeCost (PC.py:447-464) on the device. */
int lmpc_ss_put_lap(lmpc_handle* h, int inst, int slot, int T, const double* x, const double* u, const double* qfun);
/* Selection for the coming lap: slots[B,numSS_it] in argsort(LapTime) order (PC.py:395,402); is_prev[B,numSS_it] = 1
 * where that lap is iteration it-1 (PC.py:506-512); prev_slot[B] = slot receiving addPoint rows (-1: none). */
int lmpc_ss_set_selection(lmpc_handle* h, const int* slots, const int* is_prev, const int* prev_slot);
/* LMPC.addPoint (PC.py:466-476) for every instance: x[B,6], u[B,2] (host).  A non-finite value anywhere is refused with
 * LMPC_E_INVALID and nothing is appended (the reference would store it; the device closed loop skips such a point, flag 512). */
int lmpc_ss_add_point(lmpc_handle* h, const double* x, const double* u);
/* Read a safe-set lap back (tests, plotting): x[Tmax,6], u[Tmax,2], qfun[Tmax] caller-allocated, *T rows valid. */
int lmpc_ss_get_lap(lmpc_handle* h, int inst, int slot, int* T, double* x, double* u, double* qfun);
/* Overwrite one stored state row (used to reproduce the aliased write of PC.py:394 on the very first solve). */
int lmpc_ss_patch_row(lmpc_handle* h, int inst, int slot, int row, const double* x6, int also_model_slot);

/* Controller state (host arrays; any pointer may be NULL = leave / skip):
 * xLin[B,N+1,6], uLin[B,N,2] (PC.py:89-90,131-133,432-433), zt[B,6] (PC.py:330,383), OldInput[B,2] (PC.py:93,136),
 * timeStep[B] (PC.py:107,137,445), has_pred[B] (`self.xPred == []`, PC.py:502), xPred[B,N+1,6]. */
int lmpc_state_set(lmpc_handle* h, const double* xLin, const double* uLin, const double* zt, const double* OldInput,
                   const int* timeStep, const int* has_pred, const double* xPred);
int lmpc_state_get(lmpc_handle* h, double* xLin, double* uLin, double* zt, double* OldInput, int* timeStep);

/* K1 alone — MPC.computeLTVdynamics (PC.py:140-145) from the stored xLin/uLin: abc_out[B,N,54] (may be NULL: result
 * stays on the device for the next solve), flags[B] (0 ok; 1 singular regression, 2 curvature lookup failed,
 * 4 single neighbour in a lap — cases where the reference raises; 32 more than 32 rows fell within the rounding margin of
 * the MaxNumPoint-th neighbour, so the selection is not certified to be the reference's). */
int lmpc_identify_host(lmpc_handle* h, double* abc_out, int* flags);
/* K2 alone — LMPC.addTerminalComponents (PC.py:386-416) for x0[B,6]: outputs as in lmpc_solve_lmpc_host plus
 * min_index[B,numSS_it] (argmin row per lap) and flags[B] (8 = window past the stored lap, or a lap without rows).  The argmin
 * row is np.argmin's for any zt and lap: the first row at a NaN distance if there is one, else the first minimum, +inf included
 * (a lap at distance +inf everywhere selects row 0).  A lap without rows writes neither selection nor min_index. */
int lmpc_select_host(lmpc_handle* h, const double* x0, double* SS_sel, double* Qfun_sel, double* Succ_SS,
                     double* Succ_uSS, int* min_index, int* flags);

/* One full controller step for the whole batch = MPC.solve / LMPC.solve (PC.py:110-137):
 *   mode 0: LTV-MPC   K1 -> QP -> shift          (timeVarying MPC, main.py:91-94)
 *   mode 1: LMPC      K1 -> K2 -> QP -> shift    (main.py:113-120)
 * x0[B,6] host.  Outputs (host, any may be NULL): xPred[B,N+1,6], uPred[B,N,2], lambd[B,M], zt[B,6], zt_u[B,2],
 * SS_sel[B,6,M] (for SSStoredPredTraj, PC.py:379), status[B], iters[B], resid[B,3], flags[B] (K1/K2 bits: 1, 2, 4, 32 as in
 * lmpc_identify_host, 8 as in lmpc_select_host). */
int lmpc_step_host(lmpc_handle* h, int mode, const double* x0, double* xPred, double* uPred, double* lambd, double* zt,
                   double* zt_u, double* SS_sel, int* status, int* iters, double* resid, int* flags);
/* Same with x0 already on the device; results stay in the handle's device buffers (lmpc_device_buffer). */
int lmpc_step_dev(lmpc_handle* h, int mode, const double* x0_dev);
/* lmpc_step_dev with CUDA events between its kernels: ms4 = milliseconds of K1 (k-NN regression), K2 (safe-set selection, 0 for
 * mode 0), the QP kernel and the state shift.  Measurement support for per-kernel rooflines; synchronises.  With a prediction-model
 * table installed (lmpc_set_prediction_models), ms4[0] covers K1 and the nominal-model kernel together. */
int lmpc_step_profile(lmpc_handle* h, int mode, const double* x0_dev, float* ms4);
/* QP status / iterations / residuals [B,3] / step flags of the most recent lmpc_step_dev or lmpc_rollout_step (any NULL). */
int lmpc_step_results(lmpc_handle* h, int* status, int* iters, double* resid, int* flags);
/* Inspection: copy `bytes` from the named device buffer (names as lmpc_device_buffer) at `offset_bytes` to host memory.
 * The caller is responsible for staying inside the buffer (sizes follow from batch, N and numSS_Points). */
int lmpc_read_buffer(lmpc_handle* h, const char* name, size_t offset_bytes, void* dst, size_t bytes);
/* Device address of an internal buffer by name: "xPred","uPred","lambd","zt","zt_u","abc","SS_sel","Qfun_sel",
 * "Succ_SS","Succ_uSS","status","iters","resid","flags","xLin","uLin","x0","OldInput","slack","slackT" (lane slacks [B,N*ncx] and
 * terminal slack [B,6] of the most recent step), "abc_lti", "x_meas" (the measured state [B,6] of the closed loop's current
 * step under lmpc_rollout_set_measurement_noise), "x_est" (the state [B,6] the controllers read in that step under
 * lmpc_rollout_set_observers), "xPredPrev" (the previous step's prediction [B,N+1,6]) and "has_pred" (int [B]: 1 when it is
 * one), the observer's prior, "x_prior" (the prior [B,6] the observer formed in that step under
 * lmpc_rollout_set_observer_priors), and "obs_jac", "obs_cov", "obs_gain" (A, P and K [B,6,6] of the step's model gains under
 * lmpc_rollout_set_observer_gains). */
void* lmpc_device_buffer(lmpc_handle* h, const char* name);

/* ===== device-resident closed loop (the caller of the hot path, SURVEY §8f rank 1) =======================================
 * Simulator.sim's loop body (SysModel.py:33-48) for every instance without host round trips:
 *   Controller.solve(x) -> u = uPred[0] -> Controller.addPoint(x,u) -> x+ = Simulator.dynModel(x, x_glob, u)
 * (100 explicit-Euler sub-steps of the dynamic bicycle model with Pacejka tyres, SysModel.py:56-147).
 * z_host[B,3] = standard-normal draws for the (vx, vy, wz) noise in the reference's order; NULL = Philox4x32-10 on the
 * device keyed by (seed, stream, step), stream = instance unless lmpc_rollout_set_noise_streams says otherwise.  The visited (x, u) pairs are recorded per instance (Tcl rows). */
int lmpc_rollout_create(lmpc_handle* h, int Tcl);
int lmpc_rollout_set_state(lmpc_handle* h, const double* x, const double* xglob);              /* [B,6] host, may be NULL */
int lmpc_rollout_get_state(lmpc_handle* h, double* x, double* xglob, int* done, int* cl_len);  /* any may be NULL      */
int lmpc_rollout_step(lmpc_handle* h, int mode, const double* z_host, unsigned long long seed);   /* mode 0 LTV-MPC, 1 LMPC, 2 LTI-MPC */
/* Since lmpc_rollout_create: OR of the per-step flags (bits as in lmpc_step_host) and number of steps whose QP was not
 * reported solved (the reference would have driven on with feasible = 0, PC.py:279-283), per instance; either may be NULL.
 * The simulator adds two bits of its own, in lmpc_rollout_step and lmpc_rollout_pid_step alike: 128 = a curvature lookup of
 * the plant failed (s < 0, s exactly at the finish line, s not finite or beyond 64 laps: the reference raises, Track.py:292-310;
 * the step went on with curvature 0), 256 = a step found the closed-loop record full (Tcl rows) and was not recorded, so the
 * lap is longer than the record and its hand-over files it truncated.  Mode 1 adds 512 = the controller's state or input was not
 * finite, so addPoint did not append it to lap it-1 (the lap the pooled exchange exports). */
int lmpc_rollout_get_health(lmpc_handle* h, int* flags_or, int* unsolved_steps);                 /* [B] host             */
/* The rest of main.py's pipeline on the device (SURVEY §8f rank 3).
 * lmpc_rollout_pid_step: one closed-loop step under the PID path follower (Utilities.py:42-68, target speed vt); z_pid_host[B,2]
 *   and z_sim_host[B,3] are the reference's standard-normal draws in its order, NULL = Philox.  1000 such steps from
 *   x = [0.5,0,0,0,0,0] are main.py:65-66's PID lap (the record must hold them: lmpc_rollout_create(h, Tcl >= 1000)).
 * lmpc_rollout_sysid: Regression(x, u, lamb) (Utilities.py:5-28) of every record -> device buffer "abc_lti" [B,54] = A | B | 0
 *   (and abc_host / flags_host when given; flag bit 1 = singular normal matrix).  lmpc_rollout_step(mode 2) then runs the LTI
 *   MPC of main.py:72-80 with it.
 * lmpc_rollout_seed_from_record: main.py:99-110 -- the record becomes `copies` identical laps in the safe set and in the
 *   regression model (the caller's lap books must say the same: lmpc_ss_set_selection / lmpc_model_set_used), xLin/uLin/zt/
 *   OldInput/timeStep are initialised as LMPC.__init__/addTrajectory do, the record restarts. */
int lmpc_rollout_pid_step(lmpc_handle* h, double vt, const double* z_pid_host, const double* z_sim_host, unsigned long long seed);

/* Vehicle of the device simulator: the ten constants of Simulator.dynModel (SysModel.py:61-70). */
typedef struct lmpc_vehicle_params {
    double m, lf, lr, Iz;         /* mass, CoG to front / rear axle, yaw inertia: 1.98, 0.125, 0.125, 0.024 */
    double Df, Cf, Bf;            /* front Pacejka: Fyf = Df sin(Cf atan(Bf alpha_f)); 0.8 * m * 9.81 / 2.0, 1.25, 1.0 */
    double Dr, Cr, Br;            /* rear, the same form */
} lmpc_vehicle_params;
/* Per-controller vehicles (Monte-Carlo over the plant; no reference counterpart: the reference simulates one car).  Controller b is
 * simulated with sets[set_of_instance[b]] (host arrays) by every later lmpc_rollout_step (modes 0, 1, 2) and lmpc_rollout_pid_step,
 * so the PID lap that seeds both stores, the LTI sysid and the learned models all see that controller's own car.  nsets == 0
 * (sets, set_of_instance NULL) returns to the reference vehicle, which every handle starts with.
 *   - 1 <= nsets <= batch, every index in [0, nsets); m, Iz, lf, lr > 0 and all ten values finite.
 *   - Any failed check returns LMPC_E_INVALID and leaves the handle as it was.
 *   - The call synchronises the handle's streams before it replaces the table.
 *   - The vehicle index is independent of the parameter-set index of lmpc_set_param_sets (crossed designs work).  The QP entry
 *     points, the noise model, dt and the 1 ms sub-step are unchanged.
 *   - The pooled safe-set exchange (lmpc_pool_*) hands laps between the controllers of one pool group whatever their car; a lap
 *     another car drove is not a feasible trajectory of this one, so a clean plant sweep puts each car in its own group
 *     (lmpc_set_pool_groups). */
int lmpc_rollout_set_vehicles(lmpc_handle* h, const lmpc_vehicle_params* sets, int nsets, const int* set_of_instance);

/* Track surface of the device simulator: friction zones along the circuit (a wet corner, a dusty straight). */
#define LMPC_MAX_ZONES 16
typedef struct lmpc_surface_params {
    int nzone;                           /* 0 .. LMPC_MAX_ZONES; 0 = a dry row (no zone) */
    int pad;
    double zone[LMPC_MAX_ZONES * 4];     /* per zone: s_start, s_end, mu_f, mu_r; entries past nzone are not read */
} lmpc_surface_params;
/* Per-controller track surfaces (DESIGN.md, "Track surfaces"; no reference counterpart: the reference's grip is the same all
 * round the lap).  Controller b is simulated on row sets[set_of_instance[b]] (host arrays).  nsets == 0 (sets, set_of_instance
 * NULL) removes the table; every handle starts without one.
 *   - Rule, per sub-step i of the simulator's loop: s_w is the sub-step's starting s -- the value its curvature lookup takes --
 *     wrapped as that lookup wraps it (repeated subtraction of TrackLength while s > TrackLength, only when s <= 64 TrackLength).
 *     Zone k matches when s_start_k <= s_w < s_end_k; it gives the sub-step the peak tyre forces fl(mu_f Df) and fl(mu_r Dr), the
 *     rest of the sub-step unchanged.  Otherwise -- no zone matches, s is not finite or s is beyond 64 laps -- the sub-step uses
 *     Df and Dr exactly, so a sub-step off every zone computes what it computes without a table.  Df and Dr are the controller's
 *     vehicle row (under a vehicle lap schedule, the scheduled row).  Scaling D is how a friction coefficient enters the
 *     reference's car (D = mu m g / 2): a zone is a stretch with mu_f / mu_r times the car's grip.
 *   - Zones are not checked against TrackLength: a zone past the lap never matches, and [0, 2 TrackLength) covers the whole lap,
 *     a wrapped s == TrackLength included.
 *   - Read by every lmpc_rollout_step (modes 0, 1, 2; through the surface lap schedule when one is installed, LMPC_SCHEDULE_SURFACE),
 *     by lmpc_rollout_pid_step (set_of_instance; the PID lap ignores schedules) and by the mode 2 nominal model
 *     (lmpc_set_prediction_models).  A retired controller reads nothing.  The caller-problem solves, the host-driven steps (except
 *     through a mode 2 nominal model), K1, K2, the lap books, lmpc_rollout_sysid, the measurement kernel, the reports and the trace
 *     ignore it.  A mode 1 controller plans on the car it believes in without a surface; a surface it believes in is not covered.
 *   - The pooled exchange hands laps between the controllers of a pool group whatever their surface: a clean surface study puts
 *     each surface in its own group (lmpc_set_pool_groups).
 *   - 1 <= nsets <= batch, every index in [0, nsets); per row 0 <= nzone <= LMPC_MAX_ZONES and, for every zone k < nzone, all
 *     four values finite, 0 <= s_start < s_end, mu_f >= 0, mu_r >= 0, and the zones ascending without overlap
 *     (s_end_k <= s_start_{k+1}).  While a surface lap schedule is installed, a table that does not cover its largest entry and
 *     the removal are refused.  Any failed check returns LMPC_E_INVALID and leaves the handle as it was.
 *   - Allowed at any time; it synchronises the handle's streams and applies from the next step.  Not part of a snapshot record
 *     (LMPC_SNAPSHOT_VERSION is unchanged).  Without a table the kernels run the code they run without this feature. */
int lmpc_rollout_set_surfaces(lmpc_handle* h, const lmpc_surface_params* sets, int nsets, const int* set_of_instance);

/* Per-controller prediction model: where rows 0..2 (vx, vy, wz) of a controller's LTV model come from. */
#define LMPC_FLAG_NOMINAL_NONFINITE 1024     /* step flag: an entry of a nominal controller's rows 0..2 is not finite */
typedef struct lmpc_prediction_model_params {
    int mode;                     /* 0 learned (the reference's k-NN regression), 1 nominal: `vehicle`, 2 nominal: the plant's own vehicle row */
    int pad;
    lmpc_vehicle_params vehicle;  /* the car a mode 1 controller believes it drives; not read under modes 0 and 2 */
} lmpc_prediction_model_params;
/* Per-controller prediction models (what the learned model costs or buys, against a controller that plans with the exact
 * linearisation of a car).  Controller b reads row sets[set_of_instance[b]].  nsets == 0 (sets, set_of_instance NULL) removes
 * the table.  Honoured wherever the k-NN regression runs: lmpc_identify_host, lmpc_step_host / _dev / _profile (modes 0, 1) and
 * lmpc_rollout_step (modes 0, 1).
 *   - Mode 0 is the k-NN regression, unchanged.
 *   - Modes 1 and 2: stage i < N_b is identified at (xbar, ubar) = (xLin[i], uLin[i]).  Phi is the noise-free map of the velocity
 *     subsystem (vx, vy, wz, delta, a) -> (vx, vy, wz) over one control period, the simulator's loop exactly (h = 0.001 s while
 *     (i + 1) h <= dt, the reference's lf in alpha_r).  Rows 0..2 of A are dPhi/d(vx, vy, wz) with columns 3..5 zero; rows 0..2
 *     of B are dPhi/d(delta, a), both columns filled; C_r = Phi_r(xbar, ubar) - (sum_j A_rj xbar_j + sum_k B_rk ubar_k), summed
 *     left to right.  Rows 3..5 are the reference's closed-form kinematic rows, bit for bit what the regression writes for the
 *     same xLin.  The sensitivities are propagated through the sub-steps (forward mode, fp64).
 *   - Vehicle: mode 1 uses the row's own; mode 2 the row the simulator uses for b: in lmpc_rollout_step its vehicle-table row
 *     through the vehicle lap schedule when one is installed (lap_n as the step starts), in the host-driven entry points its
 *     vehicle-table row (set_of_instance of lmpc_rollout_set_vehicles).
 *   - Flags: a nominal controller never sets 1, 4 or 32; it sets 2 as the regression does, and LMPC_FLAG_NOMINAL_NONFINITE when
 *     an entry of its rows 0..2 is not finite (the rollout health word ORs it in like the other step flags).
 *   - Rollout mode 2 (LTI), the model pool, the lap books and the pooled exchange do not look at the table: a nominal controller
 *     keeps filing laps, and a return to mode 0 regresses on them.  Retired controllers identify nothing; shaped handles
 *     identify stages < N_b.
 *   - Requires lmpc_store_create (else LMPC_E_STATE).  1 <= nsets <= batch, every index in [0, nsets); mode 0, 1 or 2; all ten
 *     vehicle values finite in every row, and m, lf, lr, Iz > 0 in a mode 1 row.  Any failed check returns LMPC_E_INVALID and
 *     leaves the handle as it was.  Allowed at any time; it synchronises the handle's streams and applies from the next
 *     identification; warm-start records stay.
 *   - Not part of a snapshot record (LMPC_SNAPSHOT_VERSION is unchanged).
 *   - While a table is installed, lmpc_step_profile's ms4[0] covers the regression and the nominal-model kernel together. */
int lmpc_set_prediction_models(lmpc_handle* h, const lmpc_prediction_model_params* sets, int nsets, const int* set_of_instance);

/* Noise model of the device closed loop: the clipped Gaussian noise of Simulator.dynModel and of the PID path follower. */
typedef struct lmpc_noise_params {
    double sim_sigma[3];          /* vx, vy, wz: 0.01, 0.01, 0.005      SysModel.py:139-141 */
    double sim_clip[3];           /* 0.05, 0.05, 0.05                                       */
    double sim_gain;              /* 0.01                               SysModel.py:143-145 */
    double pid_sigma[2];          /* steering, acceleration: 0.25, 0.10 Utilities.py:42-68  */
    double pid_clip[2];           /* 0.9, 0.2                                               */
} lmpc_noise_params;
/* Per-controller noise models (robustness studies; no reference counterpart: the reference has one noise level).  Controller b
 * draws its noise with sets[set_of_instance[b]] (host arrays) in every later lmpc_rollout_step (modes 0, 1, 2) and
 * lmpc_rollout_pid_step, in the reference's form and operation order per channel j:
 *   simulator  n_j = fmax(-sim_clip_j, fmin(z_j * sim_sigma_j, sim_clip_j)),  x_j += sim_gain * n_j  (curvilinear copy only)
 *   PID        u_j += fmax(-pid_clip_j, fmin(z_j * pid_sigma_j, pid_clip_j))
 * with z_j the standard-normal draws (Philox, or z_host / z_pid_host / z_sim_host when given).  nsets == 0 (sets,
 * set_of_instance NULL) returns to the reference's constants, which every handle starts with.
 *   - 1 <= nsets <= batch, every index in [0, nsets); every value finite and >= 0 (zero sigma or clip: a noise-free channel).
 *   - Any failed check returns LMPC_E_INVALID and leaves the handle as it was.
 *   - The call synchronises the handle's streams before it replaces the table.  It is allowed at any time: a noise change in
 *     the middle of a run applies from the next step on.
 *   - The noise index is independent of the parameter-set, vehicle, track and pool-group indices. */
int lmpc_rollout_set_noise(lmpc_handle* h, const lmpc_noise_params* sets, int nsets, const int* set_of_instance);
/* Noise streams (common random numbers): the Philox draws of controller b are keyed by (seed, stream_of_instance[b], clock) in
 * the simulator and by (seed ^ constant, stream_of_instance[b], clock) in the PID, so controllers on one stream meet the same
 * draws -- two tunings run on one stream share their PID lap, their seeded stores and every later draw, and compare in pairs.
 * stream_of_instance is a host array [batch] of numbers >= 0; repeats are allowed.  NULL returns to stream b = b, which every
 * handle starts with.  Host-given draws (z_host, z_pid_host, z_sim_host) do not use the streams.  Checks, refusal and
 * synchronisation as lmpc_rollout_set_noise. */
int lmpc_rollout_set_noise_streams(lmpc_handle* h, const int* stream_of_instance);
/* Measurement noise of the device closed loop: the clipped Gaussian sensor noise on the six curvilinear channels every
 * controller sees (no reference counterpart: the reference's controllers read the simulator's exact state). */
typedef struct lmpc_measurement_params {
    double sigma[6];              /* vx, vy, wz, epsi, s, ey */
    double clip[6];
} lmpc_measurement_params;
/* Per-controller measurement noise.  With a table installed, every lmpc_rollout_step (modes 0, 1, 2) and lmpc_rollout_pid_step
 * first forms, for every controller that is not retired, the measurement
 *   y_j = x_j + n_j,   n_j = fmax(-clip_j, fmin(z_j * sigma_j, clip_j))   (y_j = x_j exactly where n_j == 0)
 * of the plant state x, z_j standard normal from Philox4x32-10 keyed by (seed ^ constant, stream, clock) with the stream of
 * lmpc_rollout_set_noise_streams and a constant of its own (the process and PID draws are unchanged).  Everything the controller
 * knows comes through y: the QP's x0 (modes 0, 1, 2), the safe-set selection, addPoint's row, the PID's input and the state rows
 * of the closed-loop record, and through the record the lap hand-over, lmpc_rollout_sysid, the seeding and the pooled exchange.
 * The plant (the simulator, done, the lap wrap, lmpc_rollout_get_state) and the trace keep the true state; the inputs of the
 * record are the inputs applied.  y of the current step is the device buffer "x_meas" [B,6] (lmpc_read_buffer).
 * controller b measures with sets[set_of_instance[b]] (host arrays); nsets == 0 (sets, set_of_instance NULL) removes the table,
 * which every handle starts without: then no kernel is launched and every consumer reads the plant state, as before.
 *   - 1 <= nsets <= batch, every index in [0, nsets); every value finite and >= 0 (zero sigma or clip: a noise-free channel).
 *   - Needs lmpc_rollout_create (LMPC_E_STATE otherwise); any failed check returns LMPC_E_INVALID and leaves the handle as it was.
 *   - The call synchronises the handle's streams before it replaces the table.  It is allowed at any time: a change in the
 *     middle of a run applies from the next step on.  The table stays with the handle and is not part of a snapshot record.
 *   - The host-driven entry points (lmpc_step_*, lmpc_solve_*) take the caller's x0 and are not affected. */
int lmpc_rollout_set_measurement_noise(lmpc_handle* h, const lmpc_measurement_params* sets, int nsets, const int* set_of_instance);
/* State observer of the device closed loop: a fixed-gain predictor-corrector on the state a controller reads (no reference
 * counterpart; DESIGN.md, "Per-controller state observers"). */
#define LMPC_FLAG_OBSERVER_RESET 2048        /* step flag: the observer's prior was not finite, the controller read y */
typedef struct lmpc_observer_params {
    int mode;                     /* 0 no observer (the controller reads y), 1 observer */
    int pad;
    double gain[6];               /* l_j in [0, 1] per channel vx, vy, wz, epsi, s, ey; not read under mode 0 */
} lmpc_observer_params;
/* Per-controller state observers.  Controller b reads row sets[set_of_instance[b]] (host arrays); nsets == 0 (sets,
 * set_of_instance NULL) removes the table, which every handle starts without: then no kernel is launched and every kernel runs
 * the code it runs without this feature.  With a table installed, every lmpc_rollout_step (modes 0, 1, 2) and
 * lmpc_rollout_pid_step launches one more kernel, right after the measurement kernel, which forms the state x_hat [B,6] the
 * controller reads from y, the measured state under lmpc_rollout_set_measurement_noise and the plant state otherwise:
 *   - Mode 0 rows: x_hat = y exactly.
 *   - Mode 1 rows in a step of mode 0 or 1: the prior is p = xPred[1] of the QP the controller solved in its previous step (row 1
 *     of the state section xPredPrev), read only when has_pred == 1.  Lap wrap: when p_s - y_s > TrackLength / 2 (the plant
 *     wrapped s at a hand-over, p did not), p_s = fmax(p_s - TrackLength, 0), the rule of the safe-set selection's terminal
 *     guess.  Then per channel j
 *       x_hat_j = p_j + l_j (y_j - p_j)   in fp64 without fused multiply-adds, rounded per operation,
 *     except that l_j == 1 copies y_j and l_j == 0 takes p_j exactly.  Without a prior (has_pred == 0: the first step after the
 *     seeding, after a PID or LTI step, after lmpc_state_set) x_hat = y exactly.  A prior with a non-finite entry on a channel
 *     with l_j < 1 is not used: x_hat = y and the step sets LMPC_FLAG_OBSERVER_RESET, which reaches the health word and the lap
 *     reports like every step flag.  A row whose gains are all 1 never reads the prior and never sets the flag.
 *   - Mode 1 rows in a PID step or a rollout step of mode 2: xPredPrev is only written by the state shift of modes 0 and 1, so
 *     such a step clears has_pred and the controller reads x_hat = y.
 *   - x_hat replaces y as the QP's x0 (and so the safe-set selection), addPoint's row and the state rows of the closed-loop
 *     record (and so the lap hand-over, the safe set, the learned model, the lane rules and the adapted lane margins).  The PID's
 *     input and the LTI QP's x0 read x_hat = y.  The plant, done, the lap wrap, lmpc_rollout_get_state, the trace and the lap
 *     reports keep the true state.  x_hat of the current step is the device buffer "x_est" [B,6] (lmpc_read_buffer).
 *   - A retired controller (lmpc_rollout_set_lap_budget) reads, writes and flags nothing.
 *   - 1 <= nsets <= batch, every index in [0, nsets); mode 0 or 1; every gain finite and in [0, 1].
 *   - Needs lmpc_rollout_create (LMPC_E_STATE otherwise); any failed check returns LMPC_E_INVALID.  Every refusal leaves the
 *     handle as it was.
 *   - The call synchronises the handle's streams before it replaces the table.  It is allowed at any time: a change in the middle
 *     of a run applies from the next step on.  The table stays with the handle, is not part of a snapshot record and is not
 *     schedulable; the observer's memory (xPredPrev, has_pred) is part of every record, so a restored controller under the same
 *     table continues exactly.
 *   - The host-driven entry points (lmpc_step_*, lmpc_solve_*) take the caller's x0 and are not affected. */
int lmpc_rollout_set_observers(lmpc_handle* h, const lmpc_observer_params* sets, int nsets, const int* set_of_instance);
/* Where a mode 1 observer takes its prior from (DESIGN.md, "Observer priors").  The row mirrors lmpc_prediction_model_params:
 * "a believed car" and "the plant's own car" mean the same in both tables. */
typedef struct lmpc_observer_prior_params {
    int source;                   /* 0 own plan (xPred[1] of the previous QP), 1 a believed car: `vehicle`, 2 the plant's own car */
    int pad;
    lmpc_vehicle_params vehicle;  /* read under source 1 only */
} lmpc_observer_prior_params;
/* Per-controller observer priors.  Controller b reads row sets[set_of_instance[b]] (host arrays); nsets == 0 (sets,
 * set_of_instance NULL) removes the table, which every handle starts without.  The table changes what the observer kernel of
 * lmpc_rollout_set_observers computes and adds no launch; without an observer table it is stored and does nothing.
 *   - Source 0: the prior is the controller's own plan, exactly as without a prior table (bit for bit).
 *   - Sources 1 and 2, in a rollout step of mode 0 or 1, for a controller whose observer row is mode 1 with has_pred == 1 and a
 *     gain below 1: the prior is p = Phi_car(xPredPrev[b][0], OldInput[b]), the estimate the controller read in its previous
 *     step (row 0 of its previous QP's prediction is its x0) carried over one control period under the input applied in that
 *     step.  Phi_car is the simulator's noise-free control period on the six curvilinear states: its sub-step loop (h = 0.001 s
 *     while (i + 1) h <= dt, the reference's lf in alpha_r, the same curvature lookup) with the same expressions, without the
 *     global frame and the process noise.
 *       source 1  the row's `vehicle`, no surface (prediction model mode 1);
 *       source 2  the vehicle row and, with a surface table, the surface row the plant drove the previous step with, both through
 *                 their lap schedules.  That step's lap is lap_n - 1 when xPredPrev[b][0].s - y.s > TrackLength / 2 (a hand-over
 *                 came in between and moved lap_n on), else lap_n.
 *     Then, as for source 0: the lap-wrap fix of p_s against y_s and the blend x_hat_j = p_j + l_j (y_j - p_j).
 *   - The prior is not used (x_hat = y and the step sets LMPC_FLAG_OBSERVER_RESET) when an input of Phi (xPredPrev[b][0],
 *     OldInput[b]) is not finite, a sub-step's curvature lookup failed, or p_j is not finite on a channel with l_j < 1.  A row
 *     whose gains are all 1 forms no prior and never sets the flag.
 *   - "x_prior" [B,6] (lmpc_read_buffer) holds the prior the observer formed in the current step, after the lap-wrap fix, for
 *     every controller that is not retired, and NaN where it formed none.  It is written only while a prior table is installed.
 *   - 1 <= nsets <= batch, every index in [0, nsets); source 0, 1 or 2; under source 1 all ten vehicle values finite and
 *     m, lf, lr, Iz > 0.
 *   - While an observer gain table (lmpc_rollout_set_observer_gains) gives a controller a mode 1 row, a table or a removal that
 *     would give that controller source 0 is refused.
 *   - Needs lmpc_rollout_create (LMPC_E_STATE otherwise); any failed check returns LMPC_E_INVALID.  Every refusal leaves the
 *     handle as it was.
 *   - The call synchronises the handle's streams before it replaces the table.  It is allowed at any time and applies from the
 *     next step on.  Not schedulable and not part of a snapshot record (LMPC_SNAPSHOT_VERSION is unchanged): the prior's inputs
 *     (xPredPrev, OldInput, has_pred) are already part of every record. */
int lmpc_rollout_set_observer_priors(lmpc_handle* h, const lmpc_observer_prior_params* sets, int nsets, const int* set_of_instance);
/* Model-based observer gains (DESIGN.md, "Observer gains"): the frozen-time Kalman gain of the linearised car in place of the
 * observer row's fixed gains. */
#define LMPC_FLAG_OBSERVER_GAIN 4096         /* step flag: the model gain could not be formed, the controller read y */
typedef struct lmpc_observer_gain_params {
    int mode;                     /* 0 the observer row's fixed gains, 1 model gains */
    int pad;
    double q[6];                  /* process covariance diagonal per control period, (vx, vy, wz, epsi, s, ey); read under mode 1 */
    double r[6];                  /* measurement covariance diagonal; read under mode 1 */
} lmpc_observer_gain_params;
/* Per-controller observer gains.  Controller b reads row sets[set_of_instance[b]] (host arrays); nsets == 0 (sets,
 * set_of_instance NULL) removes the table, which every handle starts without.
 *   - Mode 0: the observer computes exactly what it computes without a gain table (bit for bit).
 *   - Mode 1, in a rollout step of mode 0 or 1, for a controller whose observer row is mode 1 with has_pred == 1 (its prior row is
 *     source 1 or 2, see below): the prior p = Phi_car(xPredPrev[b][0], OldInput[b]) of lmpc_rollout_set_observer_priors,
 *     unchanged, and the Jacobian A = dPhi_car/dx [6,6] at the same point, by forward mode through the same sub-steps and
 *     expressions (the curvature and the surface zones' forces, piecewise constant in s, count as constants; the input is not
 *     differentiated).  P solves the filter DARE P = A P A' - A P (P + R)^-1 P A' + Q, Q = diag(q), R = diag(r) (structured
 *     doubling in fp64, at most 64 doublings, stopped once max|H' - H| <= 1e-13 max|H'|), and K = P (P + R)^-1.  After the
 *     lap-wrap fix of p_s: e_j = y_j - p_j and x_hat_i = p_i + (K_i0 e_0 + K_i1 e_1 + ... + K_i5 e_5), summed left to right,
 *     every product and sum rounded on its own.  The observer row's gains are not read.  There is no covariance carried from
 *     step to step (this is not an extended Kalman filter): the gain is a function of the step's own inputs.
 *   - A non-finite input, a failed curvature lookup or a non-finite p gives x_hat = y and LMPC_FLAG_OBSERVER_RESET, as without a
 *     gain table.  A non-finite A, P or K, or a DARE that did not converge, gives x_hat = y and LMPC_FLAG_OBSERVER_GAIN, which
 *     reaches the health word and the lap reports like every step flag.  PID and mode 2 steps clear has_pred and read y.
 *   - "obs_jac", "obs_cov", "obs_gain" [B,6,6] (lmpc_read_buffer) hold A, P and K of the current step for every controller that
 *     is not retired, NaN where no model gain was formed (K also where A, P or K is not finite or the DARE did not converge).
 *   - With a gain table installed, every lmpc_rollout_step of mode 0 or 1 with an observer table launches one more kernel,
 *     between the measurement and the observer kernels; PID and mode 2 steps launch none.
 *   - 1 <= nsets <= batch, every index in [0, nsets); mode 0 or 1; under mode 1 every q_j and r_j finite and > 0 (the DARE then
 *     has a unique stabilising solution).  A mode 1 row for a controller without an observer prior table, or whose prior row is
 *     source 0, is refused; while such rows are installed, lmpc_rollout_set_observer_priors refuses a table or a removal that
 *     would give one of those controllers source 0.
 *   - Needs lmpc_rollout_create (LMPC_E_STATE otherwise); any failed check returns LMPC_E_INVALID.  Every refusal leaves the
 *     handle as it was.
 *   - The call synchronises the handle's streams before it replaces the table.  It is allowed at any time and applies from the
 *     next step on.  Not schedulable and not part of a snapshot record (LMPC_SNAPSHOT_VERSION is unchanged). */
int lmpc_rollout_set_observer_gains(lmpc_handle* h, const lmpc_observer_gain_params* sets, int nsets, const int* set_of_instance);
/* Lap budgets: controller b is retired once it has handed over budget_of_instance[b] laps (lmpc_rollout_commit_laps_dev counts
 * them: lap_n of lmpc_books_get).  A retired controller keeps the state that hand-over left it in (lap filed, books refreshed,
 * record restarted: the start line of its next lap) and no kernel of lmpc_rollout_step (modes 0, 1, 2) or
 * lmpc_rollout_commit_laps_dev works for it: no regression, selection, QP, shift, addPoint, simulator step, health count or trace
 * row, so a batch of controllers with laps of different length stops paying for those that are finished, and every controller
 * ends in the state it would end in alone.  Retired is derived (budget set and lap_n[b] >= budget[b]), not stored: raising the
 * budget later revives a controller where it stopped, lmpc_rollout_seed_from_record_dev (lap_n = 0) revives everybody, and a
 * restored snapshot needs nothing extra.  The budget stays with the handle and is not part of a snapshot record.
 *   - budget_of_instance is a host array [batch] of numbers >= 1; NULL removes the budgets (every handle starts without).
 *   - Needs lmpc_rollout_create (LMPC_E_STATE otherwise); an entry < 1 returns LMPC_E_INVALID and leaves the handle as it was.
 *   - The call synchronises the handle's streams before it replaces the array.  It is allowed at any time.
 *   - The simulator clock counts on for the whole handle, so the Philox draws of the live controllers do not depend on who retired.
 *   - lmpc_rollout_stats / lmpc_rollout_group_stats leave retired controllers out of the minimum laps driven and of the steps into
 *     the current lap (they still count in the maximum and in the flagged count); a batch or group whose controllers have all
 *     retired reports { INT32_MAX, max laps driven, INT32_MAX, flagged }.
 *   - The PID lap, the host-driven entry points (lmpc_step_*, lmpc_solve_*, lmpc_identify_host, lmpc_select_host), the host-slot
 *     hand-over (lmpc_rollout_commit_laps) and the pooled exchange (lmpc_pool_*) ignore the budget: a retired controller still
 *     files imported laps, and its last lap, which nobody extends past the finish line, never ships under
 *     lmpc_set_pool_min_overrun. */
int lmpc_rollout_set_lap_budget(lmpc_handle* h, const int* budget_of_instance);
/* Per-lap reports of the device closed loop (no reference counterpart; DESIGN.md, "Per-lap reports"): one row per lap a controller
 * drives and hands over, accumulated on the device by the kernels every step already runs.  Over the steps of the lap: */
typedef struct lmpc_lap_report {
    int steps;                    /* closed-loop steps driven, including any that found the record full (flag 256) */
    int flags;                    /* OR of the step flags and the simulator's bits: the rule of lmpc_rollout_get_health's flags_or */
    int unsolved;                 /* steps whose QP status != 1: the rule of its unsolved_steps */
    int viol_steps;               /* steps whose plant state x violates a row i of the controller's own Fx x <= bx (see below) */
    int ipm_iters;                /* sum of the interior-point iterations of the steps' QPs */
    int ipm_iters_max;            /* their maximum */
    double viol_max;              /* max over the steps and rows of Fx[i] . x - bx[i]; -inf for a lap without steps */
} lmpc_lap_report;
/* lmpc_rollout_enable_lap_reports: keep up to max_laps (1 .. 1024) report rows per controller; 0 turns reports off and frees them.
 *   - x is the plant state the step was driven from (the row the rollout trace records), never the measured state of
 *     lmpc_rollout_set_measurement_noise.  Fx, bx are the controller's untightened lane: its parameter-set row, else the handle's
 *     (never the bx - m_b its QPs plan with under lmpc_set_lane_margins).
 *     Row i is violated when d_i = (sum over j = 0..5, in order, of Fx[i][j] * x[j], fp64 without fused multiply-adds) - bx[i]
 *     is > 0; viol_max = fmax over the d_i.  A step whose x has a non-finite entry counts as violated and sets viol_max = +inf.
 *   - lmpc_rollout_step (modes 0, 1, 2) adds every field; lmpc_rollout_pid_step adds steps, flags and the violation fields only.
 *     A retired controller (lap budget) adds nothing.
 *   - The running row describes the record under way: a lap hand-over (lmpc_rollout_commit_laps_dev, lmpc_rollout_commit_laps)
 *     files it as report n (stored when n < max_laps), counts n on and resets the row; the seeding (lmpc_rollout_seed_from_record,
 *     lmpc_rollout_seed_from_record_dev) consumes the PID record without a report and starts the table afresh (n = 0).  Imported
 *     laps (lmpc_pool_*) are not driven and file nothing.  lmpc_rollout_set_state does not restart the record or the row.
 *   - Needs lmpc_rollout_create (LMPC_E_STATE otherwise).  Enabling (max_laps >= 1) is refused with LMPC_E_STATE while any
 *     controller's closed-loop record holds rows, so every report covers a whole record; enable before the PID lap or right after a
 *     hand-over or seeding.  Enabling again with another max_laps starts an empty table.  Any refusal leaves the handle as it was.
 *   - Memory: batch * max_laps * 32 bytes + batch * 48 (64 MB at batch 8192, 256 laps).  Both buffers are snapshot sections
 *     (absent, 0 bytes, without reports: such records are unchanged); a restore refuses records whose report sections differ.
 *   - Without reports the kernels read no report buffer: they test for them at run time. */
int lmpc_rollout_enable_lap_reports(lmpc_handle* h, int max_laps);
/* Report rows rows[B][max_laps] and the count n[B] of laps filed (which may exceed max_laps; rows >= min(n, max_laps) are
 * unused) into host arrays, either may be NULL.  LMPC_E_STATE without reports.  Synchronises. */
int lmpc_rollout_get_lap_reports(lmpc_handle* h, lmpc_lap_report* rows, int* n);
int lmpc_sizeof_lap_report(void);
/* Lap schedules (no reference counterpart; DESIGN.md, "Per-lap schedules"): a plant-side table whose row changes at the laps a
 * controller reaches -- a track that gets wet at lap 10, a car whose mass changes, a sensor that degrades.  For the table `table`
 * (vehicles of lmpc_rollout_set_vehicles, process and PID noise of lmpc_rollout_set_noise, measurement noise of
 * lmpc_rollout_set_measurement_noise, track surfaces of lmpc_rollout_set_surfaces), row_of_lap is a host array [batch][nlaps],
 * 1 <= nlaps <= 1024:
 *   - In every lmpc_rollout_step (modes 0, 1, 2) controller b reads row row_of_lap[b][min(lap_n[b], nlaps - 1)] of the table in
 *     place of its set_of_instance[b], in the measurement kernel and in the simulator.  lap_n is the count of laps handed over since
 *     the seeding (lmpc_books_get), read as the step starts: a lap is driven entirely under its entry and a change takes effect on
 *     the first step after the hand-over that advanced lap_n.  Entry 0 is the first LMPC (or LTV / LTI-MPC) lap after the seeding;
 *     the last entry holds for every later lap.
 *   - The PID lap (lmpc_rollout_pid_step, its pid_input_kernel noise included) and the host-driven entry points ignore schedules,
 *     as they ignore lap budgets: the seeding lap is driven under set_of_instance.  The host-slot hand-over
 *     (lmpc_rollout_commit_laps) does not advance lap_n, so a run that hands over through it stays at the entry lap_n names.
 *   - A retired controller (lmpc_rollout_set_lap_budget) reads nothing.  The schedule stays with the handle and is not part of a
 *     snapshot record; lap_n is, so a restored controller resumes at its entry.
 *   - Tracks, QP parameters, regression models, shapes and safe-set lap counts are not schedulable: a track change invalidates every
 *     stored lap, and schedules of the controller's own tables are a separate question.
 *   - nlaps == 0 with row_of_lap == NULL removes the schedule.  Refusals, each leaving the handle as it was: LMPC_E_STATE without
 *     lmpc_store_create (the lap books hold lap_n) or lmpc_rollout_create, or for LMPC_SCHEDULE_MEASUREMENT without a measurement
 *     table; LMPC_E_INVALID for LMPC_SCHEDULE_SURFACE without a surface table (its entries name rows of no table), an unknown table, nlaps outside 1 .. 1024 with an array, nlaps != 0 without one or the reverse, or
 *     an entry outside [0, nsets) of the table as installed (a table reverted with nsets == 0 has one row).
 *   - Both install orders: while a schedule is installed, lmpc_rollout_set_vehicles / _noise / _measurement_noise / _surfaces
 *     refuse (LMPC_E_INVALID) a table whose rows do not cover the schedule's largest entry, an nsets == 0 revert to one row and the
 *     removal of the measurement or surface table included.
 *   - The call synchronises the handle's streams before it replaces the schedule.  It is allowed at any time.  Without a schedule
 *     the kernels read set_of_instance[b]. */
#define LMPC_SCHEDULE_VEHICLE      0
#define LMPC_SCHEDULE_NOISE        1
#define LMPC_SCHEDULE_MEASUREMENT  2
#define LMPC_SCHEDULE_SURFACE      3     /* the track surfaces of lmpc_rollout_set_surfaces, under the measurement kind's rules */
int lmpc_rollout_set_lap_schedule(lmpc_handle* h, int table, int nlaps, const int* row_of_lap);
int lmpc_rollout_sysid(lmpc_handle* h, double lamb, double* abc_host, int* flags_host);
int lmpc_rollout_seed_from_record(lmpc_handle* h, int copies, int ss_slot0, int model_slot0);
int lmpc_rollout_get_lap(lmpc_handle* h, int inst, int* T, double* x, double* u);              /* closed-loop record   */
/* Lap hand-over on the device = LMPC.addTrajectory + PredictiveModel.addTrajectory of the lap just driven, then
 * s -= TrackLength (SysModel.py:50), record restarted, timeStep = 0 (PC.py:445), for every instance with fin_host[b] != 0 in
 * one launch; per instance a safe-set and a regression slot, either of which may be -1 ([B] host arrays). */
int lmpc_rollout_commit_laps(lmpc_handle* h, const int* fin_host, const int* ss_slots_host, const int* model_slots_host);

/* ---- pooled-safe-set exchange (SURVEY §8e; no reference counterpart: the reference runs one controller) ------------------
 * Send side: pack stored lap slots_host[b] (-1: none, lens = 0) of every instance, including the rows LMPC.addPoint
 * appended after the finish line (PC.py:466-476), into rows_dev[B,Tpad,9] = (x 6 | u 2 | Qfun 1), lens_dev[B] -- device
 * buffers of the caller, which all-gathers them (NCCL) across ranks.
 * Receive side: instance b stores gathered lap src_host[b] (index into rows_dev[n_src,Tpad,9]; -1: nothing) in safe-set slot
 * ss_slots_host[b] (-1: skip) with its Qfun, i.e. LMPC.addTrajectory (PC.py:418-445) of a lap driven by another
 * controller, and in regression-model slot model_slots_host[b] (NULL or -1: skip; rows up to the finish line only), i.e.
 * PredictiveModel.addTrajectory (PredictiveModel.py:35-46).  Which laps are "the numSS_it fastest" stays the caller's
 * bookkeeping (lmpc_ss_set_selection / lmpc_model_set_used), exactly as for laps driven locally. */
int lmpc_ss_export_laps_dev(lmpc_handle* h, const int* slots_host, int Tpad, double* rows_dev, int* lens_dev);
int lmpc_ss_import_laps_dev(lmpc_handle* h, const int* ss_slots_host, const int* model_slots_host, const int* src_host, int n_src,
                            int Tpad, const double* rows_dev, const int* lens_dev);

/* ---- lap bookkeeping on the device (SURVEY §8f rank 3; racinglmpc_b200/csrc/lapbooks.cuh) -------------------------------------
 * The reference decides once per lap, from Python lists, which stored laps the next lap uses: np.argsort(LapTime)[:numSS_it]
 * (PC.py:395,402), lap it-1 (PC.py:466-476,506-512) and usedIt = the trToUse shortest laps (PredictiveModel.py:31,35-46).  The
 * host-driven entry points above take those decisions as index arrays (lmpc_ss_set_selection / lmpc_model_set_used); the
 * entry points below keep the books on the device instead, so that a Monte-Carlo batch hands laps over without the host.
 * Slot tables per controller: safe set ss_time[B,ss_cap], ss_lap[B,ss_cap] (lap number, -1 = free), it[B]; regression model
 * md_time[B,model_cap], md_seq[B,model_cap] (arrival number, -1 = free), md_cnt[B].  lmpc_books_set uploads them (e.g. after
 * seeding through the host-driven path) and derives the selection of the uploaded tables, so that K2, addPoint, K1 and the
 * pooled export read them from then on; lmpc_books_get reads them back with the derived selection (any pointer may be NULL):
 * sel/is_prev[B,numSS_it], prev_slot[B], used[B,trToUse], lap_hist[B,16] = lengths of the laps driven since, lap_n[B]. */
int lmpc_books_set(lmpc_handle* h, const int* ss_time, const int* ss_lap, const int* it, const int* md_time, const int* md_seq,
                   const int* md_cnt);
int lmpc_books_get(lmpc_handle* h, int* ss_time, int* ss_lap, int* it, int* md_time, int* md_seq, int* md_cnt, int* sel, int* is_prev,
                   int* prev_slot, int* used, int* lap_hist, int* lap_n);
/* main.py:113-119 for every controller whose lap just ended (its done flag is set): LMPC.addTrajectory + PredictiveModel.addTrajectory
 * of the recorded lap with the bookkeeping above, s -= TrackLength, timeStep = 0.  Enqueues one kernel; no host data. */
int lmpc_rollout_commit_laps_dev(lmpc_handle* h);
/* main.py:99-110 with device books: the record becomes `copies` laps of both stores (books are reset first). */
int lmpc_rollout_seed_from_record_dev(lmpc_handle* h, int copies);
/* Progress of the batch: out4 = { min laps driven, max laps driven, min steps into the current lap among the controllers at the
 * minimum, controllers with a health flag }.  Synchronises. */
int lmpc_rollout_stats(lmpc_handle* h, int* out4);
/* The same four numbers per pool group: out[G][4] (host), G = the handle's pool groups (1 without groups, where the row equals
 * lmpc_rollout_stats).  Row g is taken over the controllers of group g only; a group without a controller on this handle reports
 * { INT32_MAX, 0, INT32_MAX, 0 }, so that a MIN over ranks takes the other ranks' values.  Preconditions as for
 * lmpc_rollout_stats.  Synchronises. */
int lmpc_rollout_group_stats(lmpc_handle* h, int* out);
/* Pooled safe-set exchange with device books (SURVEY §8e), separately within each of G pool groups (G = 1 without groups: every
 * controller in group 0).  Only the fastest laps of a group are ever selected (PC.py:395), so a rank ships, per group, its `kbest`
 * fastest latest-own laps instead of all of them: rows_dev[G,kbest,Tpad,9] = (x | u | Qfun) incl. the rows addPoint appended so
 * far, meta_dev[G,kbest,4] = (rows, lap time, gid_base + controller, group); a group without a lap on this rank ships rows with
 * global id -1.  After the all-gather, lmpc_pool_import_dev ranks the n_src <= 64 * G gathered rows of each group g (meta[.,3] ==
 * g; at most 64 per group; rows of a group outside [0, G) are never ranked) by (lap time, global id) and every controller files
 * the `share` fastest laps of its own group it does not own before its own latest lap (addTrajectory of a lap another controller
 * drove, into both stores).  took_host (may be NULL; non-NULL synchronises) receives the number of laps stored.
 * Every rank must install the same group numbering.  With more than one track installed both calls return LMPC_E_STATE unless
 * every group's controllers on this rank share one track (lmpc_set_tracks). */
int lmpc_pool_export_dev(lmpc_handle* h, int kbest, int Tpad, long long gid_base, double* rows_dev, int* meta_dev);
/* lmpc_pool_export_dev for the pool groups with ship_host[g] == 1 only (host array [G], every entry 0 or 1; else, or NULL,
 * LMPC_E_INVALID and the handle is left as it was).  A group with ship_host[g] == 0 ships its kbest rows with global id -1
 * (meta = { 0, INT32_MAX, -1, g }), so lmpc_pool_import_dev files nothing of it and leaves the books of its controllers as they
 * were: the groups exchange on schedules of their own.  The same checks as lmpc_pool_export_dev otherwise.  Every rank must pass
 * the same mask: a group shipped by one rank and masked out by another exchanges laps of some ranks only.  The mask is copied
 * before the call returns. */
int lmpc_pool_export_groups_dev(lmpc_handle* h, int kbest, int Tpad, long long gid_base, const int* ship_host, double* rows_dev,
                                int* meta_dev);
int lmpc_pool_import_dev(lmpc_handle* h, int n_src, int share, int Tpad, long long gid_base, const double* rows_dev, const int* meta_dev,
                         int* took_host);
/* Pool groups of the exchange (fleet learning per design cell: per circuit, car or tuning of a sweep; no reference counterpart).
 * Controller b exchanges laps only with the controllers of group group_of_instance[b] (host array [batch]); group numbers are
 * global labels, the same on every rank, and a group may be empty.  ngroups == 0 (group_of_instance NULL) returns to one pool.
 *   - Requires lmpc_store_create (else LMPC_E_STATE).  Allowed after laps are stored: it affects the exchanges that follow.
 *   - 0 <= ngroups <= min(batch, LMPC_MAX_POOL_GROUPS), ngroups == 0 exactly when group_of_instance is NULL, every index in
 *     [0, ngroups).  Any failed check returns LMPC_E_INVALID and leaves the handle as it was.
 *   - The call synchronises the handle's streams before it replaces the index.
 *   - Groups are not checked against parameter sets or vehicles: a group mixing tunings or cars shares laps between them. */
int lmpc_set_pool_groups(lmpc_handle* h, int ngroups, const int* group_of_instance);
/* Rows past the finish line a latest own lap must ship (min(stored rows, Tpad) - lap time; LMPC.addPoint appends them during the
 * next lap) before lmpc_pool_export_dev ships it; 0 (every handle's default) ships any latest lap, whatever its length.  An importer's safe-set window
 * (PC.py:492-495) near the finish line reaches into these rows: a lap shipped right after its controller crossed the line sends
 * the importers' selection past the stored lap (K2 flag 8; the reference raises IndexError).  A group without such a lap on this
 * rank ships rows with global id -1.  rows >= 0 (else LMPC_E_INVALID). */
int lmpc_set_pool_min_overrun(lmpc_handle* h, int rows);

/* ---- controller snapshots (no reference counterpart beyond pickling an LMPC object; racinglmpc_b200/csrc/snapshot.cuh) --------
 * What a controller of the device-resident step has learned and where it is, as one fixed-size byte record per controller:
 * both lap pools, the lap books, the controller state, the warm-start record, and with a rollout the simulator state, the
 * closed-loop record, the health counters and the LTI model (DESIGN.md, "Controller snapshots", lists every per-controller buffer
 * as carried or scratch).  Not in a record: what the handle is told to drive -- parameter sets, vehicles, tracks, noise sets,
 * noise streams, measurement sets, regression sets, pool groups -- and handle-wide counters.  The lap books travel in the record, so a caller that keeps its own host copy of them (the
 * host-driven bookkeeping of lmpc_ss_set_selection / lmpc_model_set_used) must not restore into its handle.
 * Record = header (below) + sections at 16-byte aligned offsets; every section is one controller's slice of one [B][...] buffer. */
#define LMPC_SNAPSHOT_MAGIC 0x50414e53      /* "SNAP" */
#define LMPC_SNAPSHOT_VERSION 1
#define LMPC_SNAPSHOT_SECTIONS 40           /* section slots of the header, fixed order (DESIGN.md); bytes 0 = absent */
typedef struct lmpc_snapshot_header {
    int magic, version;
    int bytes;                              /* record size, header included, a multiple of 16 */
    int N, M, ncx, ncu, numSS_it, trToUse, ss_cap, model_cap, Tmax;
    int Tcl;                                /* closed-loop record rows, 0 = the handle has no rollout */
    int warm_start;
    int warm_mode;                          /* problem type the warm-start record belongs to: -1 none, 0 LTV-MPC, 1 LMPC */
    int nsect;                              /* LMPC_SNAPSHOT_SECTIONS */
    int sect_off[LMPC_SNAPSHOT_SECTIONS];   /* byte offset of every section in the record */
    int sect_bytes[LMPC_SNAPSHOT_SECTIONS]; /* its bytes (0 = absent in this layout) */
    lmpc_track_params track;                /* the controller's own track row: a stored lap is in its circuit's s-coordinate */
} lmpc_snapshot_header;
int lmpc_sizeof_snapshot_header(void);
/* Bytes of one record of this handle (a multiple of 16).  Requires lmpc_store_create. */
int lmpc_snapshot_bytes(lmpc_handle* h, size_t* bytes);
/* Records of controllers inst_host[0..n) (host array; NULL = every controller, n == batch; repeats allowed) into the caller's
 * device buffer rec_dev[n][bytes] (16-byte aligned).  Enqueued on the handle's stream, like lmpc_pool_export_dev. */
int lmpc_snapshot_pack_dev(lmpc_handle* h, int n, const int* inst_host, void* rec_dev);
/* Controller dst_host[i] takes record rec_of_dst_host[i] (NULL = i) of rec_dev[nrec][bytes], i < n (host arrays).  One record
 * may be restored into many controllers.  A repeated destination or an index out of range returns LMPC_E_INVALID.  Records are
 * outside input: one check kernel first validates every record used -- magic, version and layout equal to this handle's, the
 * circuit (nseg, its nseg rows, TrackLength; bit for bit) the destination controller's, every index or bound field in range -- the
 * call synchronises, and copies only if all passed; a refused call returns LMPC_E_INVALID naming the first failing record and
 * field (lmpc_last_error) and leaves the handle as it was.  Warm start: the handle takes the records' warm_mode when it has none
 * yet (no device-resident step since lmpc_store_create); otherwise every record's mode must be -1 or the handle's.  A successful
 * unpack counts as a stored lap (lmpc_set_tracks then returns LMPC_E_STATE).  The copy is enqueued on the handle's stream. */
int lmpc_snapshot_unpack_dev(lmpc_handle* h, const void* rec_dev, int nrec, int n, const int* dst_host, const int* rec_of_dst_host);
/* The simulator's step counter, which keys the Philox noise with (seed, stream, step).  Requires lmpc_rollout_create. */
int lmpc_rollout_get_clock(lmpc_handle* h, unsigned long long* step);
int lmpc_rollout_set_clock(lmpc_handle* h, unsigned long long step);

/* ---- presentation support (SURVEY §8f rank 4: the inputs of the reference's plot.py for device-resident batches) --------------
 * lmpc_track_global_position: Map.getGlobalPosition (Track.py:135-189) for n points; table6[nseg,6] = Map.PointAndTangent
 *   (x_end, y_end, psi_end, s_start, length, curvature), host arrays, xy[n,2] out, ok[n] (may be NULL) = 0 where the reference
 *   would raise (no segment holds s).
 * lmpc_rollout_trace_create: from now on every lmpc_rollout_step records, for the n chosen controllers, what
 *   LMPC.unpackSolution keeps per step for plotting (PC.py:377-379) -- the prediction xPred[N+1,6], the selected safe-set points
 *   SS_sel[6,M] -- plus the closed-loop state x[6], the global state x_glob[6] (SysModel.py), the applied input u[2] and the
 *   number of laps the controller had driven (to split the trace into laps), at most cap_steps rows each.
 * lmpc_rollout_trace_get: rows of trace `tr` (index into the chosen controllers); any array pointer may be NULL. */
int lmpc_track_global_position(int device, const double* table6, int nseg, double TrackLength, int n, const double* s, const double* ey,
                               double* xy, int* ok);
int lmpc_rollout_trace_create(lmpc_handle* h, int n, const int* inst, int cap_steps);
int lmpc_rollout_trace_get(lmpc_handle* h, int tr, int* steps, double* x, double* xglob, double* u, double* xPred, double* SS_sel, int* lap);

/* fp64 micro-benchmarks on `device` (no reference counterpart; measurement support for the roofline of the QP kernel, which is
 * bound by fp64 issue and dependent-chain latency rather than HBM): out8 = { DFMA TFLOP/s, DMMA m8n8k4 TFLOP/s,
 * latency in SM cycles of: DFMA, DMMA (accumulator chain), DMMA (result -> A operand), LDS (dependent), SHFL of a double,
 * rsqrt(double) }. */
int lmpc_probe_fp64(int device, double* out8);

int lmpc_sizeof_params(void);
int lmpc_sizeof_model_params(void);
int lmpc_sizeof_vehicle_params(void);
int lmpc_sizeof_track_params(void);
int lmpc_sizeof_noise_params(void);
int lmpc_sizeof_measurement_params(void);
int lmpc_sizeof_observer_params(void);
int lmpc_sizeof_observer_prior_params(void);
int lmpc_sizeof_observer_gain_params(void);
int lmpc_sizeof_regression_params(void);
int lmpc_sizeof_shape_params(void);
int lmpc_sizeof_ss_laps_params(void);
int lmpc_sizeof_lap_window_params(void);
int lmpc_sizeof_lane_rule_params(void);
int lmpc_sizeof_lane_margin_params(void);
int lmpc_sizeof_prediction_model_params(void);
int lmpc_sizeof_surface_params(void);

#ifdef __cplusplus
}
#endif
#endif /* LMPC_B200_H */
