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
 * mode 0), the QP kernel and the state shift.  Measurement support for per-kernel rooflines; synchronises. */
int lmpc_step_profile(lmpc_handle* h, int mode, const double* x0_dev, float* ms4);
/* QP status / iterations / residuals [B,3] / step flags of the most recent lmpc_step_dev or lmpc_rollout_step (any NULL). */
int lmpc_step_results(lmpc_handle* h, int* status, int* iters, double* resid, int* flags);
/* Inspection: copy `bytes` from the named device buffer (names as lmpc_device_buffer) at `offset_bytes` to host memory.
 * The caller is responsible for staying inside the buffer (sizes follow from batch, N and numSS_Points). */
int lmpc_read_buffer(lmpc_handle* h, const char* name, size_t offset_bytes, void* dst, size_t bytes);
/* Device address of an internal buffer by name: "xPred","uPred","lambd","zt","zt_u","abc","SS_sel","Qfun_sel",
 * "Succ_SS","Succ_uSS","status","iters","resid","flags","xLin","uLin","x0","OldInput","slack","slackT" (lane slacks [B,N*ncx] and
 * terminal slack [B,6] of the most recent step), "abc_lti", "x_meas" (the measured state [B,6] of the closed loop's current
 * step under lmpc_rollout_set_measurement_noise). */
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
 *     lmpc_rollout_set_measurement_noise.  Fx, bx are the controller's QP constants: its parameter-set row, else the handle's.
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
 *   - Without reports the kernels run the code they run without this feature (template instantiations). */
int lmpc_rollout_enable_lap_reports(lmpc_handle* h, int max_laps);
/* Report rows rows[B][max_laps] and the count n[B] of laps filed (which may exceed max_laps; rows >= min(n, max_laps) are
 * unused) into host arrays, either may be NULL.  LMPC_E_STATE without reports.  Synchronises. */
int lmpc_rollout_get_lap_reports(lmpc_handle* h, lmpc_lap_report* rows, int* n);
int lmpc_sizeof_lap_report(void);
/* Lap schedules (no reference counterpart; DESIGN.md, "Per-lap schedules"): a plant-side table whose row changes at the laps a
 * controller reaches -- a track that gets wet at lap 10, a car whose mass changes, a sensor that degrades.  For the table `table`
 * (vehicles of lmpc_rollout_set_vehicles, process and PID noise of lmpc_rollout_set_noise, measurement noise of
 * lmpc_rollout_set_measurement_noise), row_of_lap is a host array [batch][nlaps], 1 <= nlaps <= 1024:
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
 *     table; LMPC_E_INVALID for an unknown table, nlaps outside 1 .. 1024 with an array, nlaps != 0 without one or the reverse, or
 *     an entry outside [0, nsets) of the table as installed (a table reverted with nsets == 0 has one row).
 *   - Both install orders: while a schedule is installed, lmpc_rollout_set_vehicles / _noise / _measurement_noise refuse
 *     (LMPC_E_INVALID) a table whose rows do not cover the schedule's largest entry, an nsets == 0 revert to one row and the removal
 *     of the measurement table included.
 *   - The call synchronises the handle's streams before it replaces the schedule.  It is allowed at any time.  Without a schedule
 *     the kernels run the code they run without this feature (template instantiations). */
#define LMPC_SCHEDULE_VEHICLE      0
#define LMPC_SCHEDULE_NOISE        1
#define LMPC_SCHEDULE_MEASUREMENT  2
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
int lmpc_sizeof_regression_params(void);
int lmpc_sizeof_shape_params(void);
int lmpc_sizeof_ss_laps_params(void);

#ifdef __cplusplus
}
#endif
#endif /* LMPC_B200_H */
