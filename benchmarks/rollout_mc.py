#!/usr/bin/env python
"""BASELINE.json configs[3]: LMPC Monte-Carlo rollouts sharded over the GPUs of one node, with the once-per-lap NCCL
all-gather of finished laps (pooled-safe-set exchange, SURVEY §8e).

Every instance is an independent LMPC controller + vehicle (its own 1000-step PID lap as initial safe set, Philox process
noise), advanced entirely on the device: K1 regression -> K2 selection -> QP -> shift -> addPoint -> dynModel per step, lap
hand-over and lap bookkeeping included (csrc/lapbooks.cuh).  The host launches kernels and, every `poll` steps, reads four
integers of progress; ranks agree on exchanging / stopping through one tiny all-reduce at those polls, so no rank can enter
a collective the others skip.

  --mode independent   reference semantics: no data-path collective (replicas).
  --mode pooled        once every controller of every rank is `--ship-after` steps into lap r+1, each rank packs its
                       `share + 1` fastest laps r on the device (only the globally fastest laps are ever selected, PC.py:395, so
                       a rank's candidates are its own fastest few: ~60 KB per rank instead of every lap), all ranks all-gather
                       them over NCCL, rank them by (lap time, global id) and every controller files the `share` fastest laps
                       it does not own as additional stored laps (safe set + regression model).
With pool groups (run(pool_groups=...)) the exchange runs within each group.  One schedule (sharding.ExchangeSchedule) decides
every poll, on one row for the whole batch or, with run(readiness="group"), one row and round counter per group, so a group
exchanges once its own slowest controller is `ship_after` steps into lap r+1 (the ranks agree on the ready rows per poll).

  python benchmarks/rollout_mc.py --batch 8192 --laps 3            (1 GPU)
  python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 benchmarks/rollout_mc.py --batch 8192
Prints one JSON line (rank 0): closed-loop steps/s over all GPUs (device events, max over ranks), lap-length statistics per
LMPC lap, exchange time and bytes."""
import argparse
import collections
import ctypes as C
import json
import os
import sys
import time
import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from racinglmpc_b200 import workloads, sharding, reference_params as rp, _native      # noqa: E402
from racinglmpc_b200.controller import BatchedController                      # noqa: E402

# the controllers of every run: horizon, regression laps and the sizes of the lap stores and the closed-loop record
N_HORIZON, TR_TO_USE, TMAX, SS_CAP, MODEL_CAP, TCL = 12, 4, 1280, 7, 5, 1024


def handle_shape(shape_sets=None):
    """(N, numSS_Points) of run()'s handle: the reference's (12, 48) without shape_sets, else the smallest pair of the instantiated
    grid that dominates every shape of shape_sets = (shapes, index), e.g. (14, 96) for any shapes at N <= 14 and (48, 48) for any
    horizon at 48 points.  Raises ValueError when no pair of the grid dominates them all."""
    numSS_Points = rp.lmpc_params(N_HORIZON)[1]
    if shape_sets is None:
        return N_HORIZON, numSS_Points
    try:
        shapes = [(int(n), int(m)) for n, m in shape_sets[0]]
    except (TypeError, ValueError):
        raise ValueError("shape_sets is (shapes, index) with (N, numSS_Points) pairs")
    if not shapes:
        raise ValueError("shape_sets needs at least one shape")
    cover = sorted((n, m) for n, m in _native.SHAPE_GRID
                   if m > 0 and all(n >= sn and m >= sm for sn, sm in shapes))
    if not cover:
        raise ValueError("no (N, numSS_Points) pair of the instantiated grid dominates the shapes %s" % sorted(set(shapes)))
    return cover[0]


def layout(warm=False, shape_sets=None, lap_reports=None):
    """The snapshot layout (BatchedController.snapshot_layout without "bytes") of run()'s controllers; "lap_reports" only when
    reports are on."""
    numSS_it = rp.lmpc_params(N_HORIZON)[0]
    N, numSS_Points = handle_shape(shape_sets)
    out = dict(N=N, M=numSS_Points, ncx=2, ncu=4, numSS_it=numSS_it, trToUse=TR_TO_USE, ss_cap=SS_CAP, model_cap=MODEL_CAP,
               Tmax=TMAX, Tcl=TCL, warm_start=int(bool(warm)))
    if lap_reports:
        out["lap_reports"] = int(lap_reports)
    return out


def check_lap_reports(lap_reports, laps):
    """The refusals of run(lap_reports=...), before any device work: None needs laps <= 16 (lap_hist's length), else an integer
    capacity L with laps <= L <= 1024.  Returns L, or 0 for no reports."""
    if lap_reports is None:
        if int(laps) > 16:
            raise ValueError("laps = %d: the lap books keep the lengths of 16 laps; pass lap_reports >= laps to report longer runs"
                             % int(laps))
        return 0
    L = _native.check_lap_reports(lap_reports)
    if L < max(int(laps), 1):
        raise ValueError("lap_reports = %d keeps fewer rows than the %d laps of the run" % (L, int(laps)))
    return L


def check_lap_schedules(lap_schedules, batch, lap_reports, tables):
    """The refusals of run(lap_schedules=...), before any device work: every kind is one of BatchedController.set_lap_schedule's,
    has its table in `tables` ({kind: (rows, index) or None}) and a schedule the table's rows cover, and the run keeps lap reports
    (the per-lap statistics come from them).  Returns {kind: [batch, L] int32 schedule}, empty without schedules."""
    if lap_schedules is None:
        return {}
    if not isinstance(lap_schedules, dict):
        raise ValueError("lap_schedules is a dict {kind: rows} with kind in %s" % sorted(_native.LAP_SCHEDULE_TABLES))
    out = {}
    for kind, rows in lap_schedules.items():
        if kind not in _native.LAP_SCHEDULE_TABLES:
            raise ValueError("lap_schedules: kind is one of %s, got %r" % (sorted(_native.LAP_SCHEDULE_TABLES), kind))
        if tables.get(kind) is None:
            raise ValueError("a %s lap schedule needs %s_sets: the schedule names rows of that table" % (kind, kind))
        out[kind] = _native.make_lap_schedule(rows, int(batch), len(tables[kind][0]))
    if out and not lap_reports:
        raise ValueError("lap_schedules need lap_reports >= laps: the per-lap statistics of a schedule come from the reports")
    return out


def lap_row_summary(reps, schedules, laps):
    """Per schedule kind, LMPC lap k < laps and table row r, over the controllers that filed a report of lap k while on row r
    (schedule[b][min(k, L - 1)] == r): how many, their mean steps, the share with a lane violation (viol_steps > 0) and the unsolved
    QPs in total.  From the reports (BatchedController.lap_reports) and the host schedules alone."""
    out = {}
    for kind, sched in schedules.items():
        L = sched.shape[1]
        rows = []
        for k in range(laps):
            on = sched[:, min(k, L - 1)]
            filed = reps["n"] > k
            for r in np.unique(on):
                m = filed & (on == r)
                n = int(m.sum())
                rows.append({"lap": k + 1, "row": int(r), "controllers": n,
                             "steps_mean": float(reps["steps"][m, k].mean()) if n else 0.0,
                             "violating_share": float((reps["viol_steps"][m, k] > 0).mean()) if n else 0.0,
                             "unsolved": int(reps["unsolved"][m, k].sum(dtype=np.int64))})
        out[kind] = rows
    return out


def _by_index(make, *extra):
    """The pack step of a table installed from (rows, index): make(rows, index, batch, *extra)."""
    return lambda ctx, rows, index=None: make(rows, index, ctx["B"], *extra)


def _pack_params(ctx, params, index=None, QterminalSlack=None):
    rows, idx = _native.make_param_sets(ctx["params"], params, index, ctx["B"], ctx["M"], ctx["numSS_it"], QterminalSlack)
    ctx["bx_min"] = np.array([min(r.bx[:r.ncx]) for r in rows])[idx]
    return rows, idx


def _pack_shapes(ctx, shapes, index=None):
    if ctx["warm"]:
        raise ValueError("shape_sets and warm start: the warm-start record is laid out per (N, numSS_Points)")
    rows, idx = _native.make_shape_sets(shapes, index, ctx["B"], ctx["N"], ctx["M"], ctx["numSS_it"])
    ctx["points"] = [rows[k].numSS_Points for k in idx]
    return rows, idx


def _pack_ss_laps(ctx, values, index=None):
    rows, idx = _native.make_ss_laps_sets(values, index, ctx["B"], ctx["numSS_it"], ctx["points"])
    ctx["laps_of"] = [rows[k].numSS_it for k in idx]
    return rows, idx


# One table argument of run(): its keyword, its name in messages, the BatchedController method that installs it, the result key of
# its per-row statistics (or None), the row fields copied into each per-row entry and whether that entry gets the row's sampled
# interior-point iterations, pack(ctx, *install arguments) -> (rows, index) (rows None for the integer tables: streams, groups),
# and args(value) -> the install arguments.
Table = collections.namedtuple("Table", "keyword name install key fields ipm pack args", defaults=(tuple,))

# every table in install order: the margins need the parameter rows' lanes, the windows the lap counts
TABLES = (
    Table("param_sets", "parameter sets", "set_param_sets", "per_set_rank0", (), False, _pack_params),
    Table("vehicle_sets", "vehicles", "set_vehicles", "per_vehicle_rank0", (), False, _by_index(_native.make_vehicle_sets)),
    Table("noise_sets", "noise sets", "set_noise", "per_noise_rank0", (), False, _by_index(_native.make_noise_sets)),
    Table("noise_streams", "noise streams", "set_noise_streams", None, (), False,
          lambda ctx, streams: (None, _native.make_noise_streams(streams, ctx["B"])), lambda streams: (streams,)),
    Table("measurement_sets", "measurement sets", "set_measurement_noise", "per_measurement_rank0", (), False,
          _by_index(_native.make_measurement_sets)),
    Table("regression_sets", "regression sets", "set_regression", "per_regression_rank0", (), False,
          _by_index(_native.make_regression_sets, TR_TO_USE)),
    Table("track_sets", "tracks", "set_tracks", "per_track_rank0", (), False, _by_index(_native.make_track_sets)),
    Table("pool_groups", "pool groups", "set_pool_groups", None, (), False,
          lambda ctx, index, ngroups: (None, _native.make_pool_groups(index, ngroups, ctx["B"]))),
    Table("shape_sets", "shapes", "set_shapes", "per_shape_rank0", ("N", "numSS_Points"), True, _pack_shapes),
    Table("ss_laps_sets", "lap counts", "set_ss_laps", "per_ss_laps_rank0", ("numSS_it",), True, _pack_ss_laps),
    Table("lap_window_sets", "lap windows", "set_lap_windows", "per_lap_window_rank0", ("ss_window", "model_window"), True,
          lambda ctx, windows, index=None: _native.make_lap_window_sets(windows, index, ctx["B"], ctx["laps_of"], SS_CAP, TR_TO_USE,
                                                                        MODEL_CAP)),
    Table("lane_rule_sets", "lane rules", "set_lane_rules", "per_lane_rule_rank0", ("mode", "lane_tol"), True,
          _by_index(_native.make_lane_rule_sets, True, TCL)),
    Table("lane_margin_sets", "lane margins", "set_lane_margins", "per_lane_margin_rank0",
          ("mode", "margin0", "margin_max", "step_up", "step_down"), True,
          lambda ctx, margins, index=None: _native.make_lane_margin_sets(margins, index, ctx["B"], ctx["bx_min"])),
    Table("prediction_model_sets", "prediction models", "set_prediction_models", "per_prediction_model_rank0", ("mode",), False,
          _by_index(_native.make_prediction_model_sets)),
    Table("surface_sets", "surfaces", "set_surfaces", "per_surface_rank0", (), False, _by_index(_native.make_surface_sets)),
)


def pack_tables(batch, warm=False, **given):
    """Packs every table of `given` ({keyword: run() argument}, None for none) on the host, in install order, with the
    _native.make_* call and the arguments its install in run() will use, so it raises that call's ValueError before any device
    work.  Returns ({keyword: (rows, index)} of the given tables, ctx): ctx holds the handle's (N, M) and numSS_it (handle_shape)
    and what later tables take from earlier ones, every controller's numSS_Points ("points"), numSS_it ("laps_of") and min_i
    bx_i of its QP row ("bx_min")."""
    B = int(batch)
    N, M = handle_shape(given.get("shape_sets"))
    numSS_it, _, _, _, Qts, par = rp.lmpc_params(N)
    base = _native.make_params(par, M, numSS_it, Qts, warm_start=warm)            # the Params row run()'s handle is created with
    ctx = dict(B=B, N=N, M=M, numSS_it=numSS_it, warm=bool(warm), params=base, points=[M] * B, laps_of=[numSS_it] * B,
               bx_min=np.full(B, min(base.bx[:base.ncx])))
    packed = {}
    for t in TABLES:
        if given.get(t.keyword) is not None:
            packed[t.keyword] = t.pack(ctx, *t.args(given[t.keyword]))
    return packed, ctx


def table_rows(packed):
    """What capture records of the tables (pack_tables' first result): {keyword: every controller's row, controller by controller,
    as the bytes the library is given}, the int32 values for streams and groups."""
    return {k: idx.tobytes() if rows is None else np.frombuffer(rows, np.uint8).reshape(len(rows), -1)[idx].tobytes()
            for k, (rows, idx) in packed.items()}


def check_start_tables(had, mine):
    """start's refusal of other tables: `had` the captured table_rows, `mine` this run's.  No table is part of a record, and the
    records were learned under the rows installed when they were captured."""
    for t in TABLES:
        if had.get(t.keyword) != mine.get(t.keyword):
            raise ValueError("start was captured with other %s: a record resumes exactly only under the tables it was captured with"
                             % t.name)


def run(batch=8192, laps=3, mode="pooled", share=2, tpad=288, ship_after=40, poll=8, max_steps=0, seed=1234, local=None, warm=False,
        final=None, param_sets=None, vehicle_sets=None, books=None, track_sets=None, pool_groups=None, readiness="batch",
        capture=None, start=None, noise_sets=None, noise_streams=None, regression_sets=None, lap_budget=None, measurement_sets=None,
        shape_sets=None, ss_laps_sets=None, lap_reports=None, lap_schedules=None, lap_window_sets=None,
        lane_rule_sets=None, lane_margin_sets=None, prediction_model_sets=None, trace=None, surface_sets=None):
    """One Monte-Carlo run on this rank's GPU (torch.distributed may or may not be initialised).  Returns a dict (all ranks).
    final: None, or a dict that receives the closed loop's end state (rollout_state) and the last step's solver report (step_results).
    books: None, or a dict that receives the lap books (books) and the health counters (flags_or, unsolved), and with lap_reports
    the reports (BatchedController.lap_reports) under "lap_reports", and with lane_margin_sets every controller's final margin under
    "lane_margins".
    The table arguments below (TABLES, in install order) are each None or the arguments of their BatchedController install,
    called after enable_rollout, before the PID lap.  Before any device work every given table is packed with the call its install
    uses (pack_tables), so a row or an index the install would refuse raises its ValueError first.  capture records every
    installed table under "tables" ({keyword: every controller's packed row}, table_rows), and start refuses a start whose tables
    or rows differ: no table is part of a record, and a record resumes exactly only under the tables it was captured with.  A table
    with a result key adds one entry per row: the lap statistics of its controllers (_set_stats), its row fields and, for some,
    their mean interior-point iterations sampled at the polls (table_stats).
    param_sets: (params, index, QterminalSlack) for set_param_sets (a parameter sweep over the batch); "per_set_rank0".
    vehicle_sets: (vehicles, index) for set_vehicles (a sweep over the plant, PID lap included); "per_vehicle_rank0".  The pooled
    mode exchanges laps between the controllers of a pool group whatever their car, so a pooled plant sweep groups by car.
    noise_sets: (noises, index) for set_noise (the simulator's and the PID's noise, PID lap included); "per_noise_rank0".
    noise_streams: the [batch] stream numbers for set_noise_streams (common random numbers: controllers on one stream meet the same
    draws).  Streams are local to a rank: every rank keys its Philox draws with its own seed (seed + rank).
    measurement_sets: (meas, index) for set_measurement_noise (the sensor noise the controllers see, PID lap included: its record,
    and so the seeded stores, are measured data); "per_measurement_rank0".  The draws pair on noise_streams like the others.
    regression_sets: (regs, index) for set_regression (the learned model's bandwidth, neighbour count, ridge, feature scaling and
    laps used, trToUse up to the store's 4); "per_regression_rank0".  The pooled mode exchanges laps whatever the model setting.
    track_sets: (tracks, index) for set_tracks (several circuits in one batch); "per_track_rank0".  A lap of another circuit is not
    a trajectory of this one, so the pooled mode with more than one track needs pool_groups in which every group drives one
    circuit.
    pool_groups: (index, G) for set_pool_groups (e.g. sharding.design_groups(track index, parameter-set index)): the pooled mode
    then exchanges laps within each group; the exchange buffers hold G * (share + 1) laps per rank and the result holds the laps
    filed per group under "laps_filed_per_group_rank0" (stored laps counted from the books; too low for a controller with health
    flag 64).  A lap ships only once it has `ship_after` rows past its finish line (lmpc_set_pool_min_overrun), so a group lapping
    faster ships the fastest of its laps that qualify.
    shape_sets: (shapes, index) for set_shapes: (N, numSS_Points) pairs of the instantiated grid (a horizon / safe-set size sweep);
    "per_shape_rank0" with N, numSS_Points and the sampled iterations.  The handle is created at handle_shape(shape_sets), the
    smallest grid pair that dominates every shape (ValueError when there is none, or with warm start); the result then holds it
    under "handle_shape".
    ss_laps_sets: (values, index) for set_ss_laps: numSS_it per controller, 1 .. the handle's 4, and every controller's
    numSS_Points its value times an even number of points per lap; "per_ss_laps_rank0" with numSS_it and the sampled iterations.
    With shape_sets as well, "per_shape_ss_laps_rank0" holds the statistics of every (shape, value) cell.
    lap_window_sets: (windows, index) for set_lap_windows: ss_window (0 or the controller's numSS_it .. ss_cap 7) and model_window
    (0 or trToUse 4 .. model_cap 5), 0 = unbounded (controllers that trust only their most recent laps); "per_lap_window_rank0"
    with both windows and the sampled iterations.
    lane_rule_sets: (rules, index) for set_lane_rules: mode (0: the reference's ranking, 1: a lap that left the lane by more than
    lane_tol ranks behind every lap that kept to it) and lane_tol; "per_lane_rule_rank0" with both and the sampled iterations.
    With lap reports the share of laps judged lane-unsafe per lap is added to every lap_reports_rank0 row and every per-rule report
    row ("lane_unsafe_share"), and "lane_unsafe_selected_share_rank0" is the share of controllers whose final selection holds a
    lane-unsafe lap.
    lane_margin_sets: (margins, index) for set_lane_margins: mode (0: none, 1: the fixed margin0, 2: adapted lap by lap within
    [margin0, margin_max] by step_up / step_down) that narrow the lane every QP plans in while reports and lane rules judge the
    given lane; "per_lane_margin_rank0" with the row's five values and the sampled iterations, and per row the min / mean / max
    of the final margins under "lane_margin_final_rank0".
    prediction_model_sets: (models, index) for set_prediction_models: mode (0: the learned k-NN model, 1: the exact linearisation
    of their vehicle, 2: that of the plant's own vehicle row, through its lap schedule) and vehicle.  Needs lap_reports >= laps;
    "per_prediction_model_rank0" with the mode and the per-lap reports.
    surface_sets: (surfaces, index) for set_surfaces (friction zones along the circuit, PID lap included); "per_surface_rank0".
    The pooled mode exchanges laps whatever the surface, so a clean pooled surface study puts each surface in its own pool group.
    readiness: when the pooled mode exchanges round r (sharding.ready_groups at every poll, agreed over the ranks).
      "batch"  every group together, once the slowest controller of the whole batch is `ship_after` steps into lap r + 1;
      "group"  each pool group on its own round counter, once the slowest controller of that group is; one export / all-gather /
               import per poll exchanges every group that is ready (lmpc_pool_export_groups_dev masks the others out), so a
               group's controllers follow the schedule they would follow alone.  Groups with no controller on any rank never
               exchange.  Needs the pooled mode (ValueError otherwise, before any device work).  Without groups it makes the
               same decisions at the same steps as "batch".
    With pool_groups or readiness="group" the result holds the readiness and the closed-loop steps at which each group
    exchanged under "exchange_steps_per_group_rank0".
    capture: None, or a dict that receives, at the end of the run, everything a later run needs to go on from here: "records"
    (every controller's snapshot record, a uint8 CUDA tensor), "clock" (the simulator step that keys the Philox noise), the loop's
    scheduler state ("steps", "next_round", "next_rounds", the groups that exchanged at the last poll, the exchange steps so far)
    and what it has to match (batch, laps, mode, readiness, poll, warm, pool groups, record layout, tables).  torch.save stores it.
    "diverged_step" is None unless, under group readiness, some group was ready for a round >= laps before the last poll: a
    longer run exchanged there and this one did not, so a resumed run cannot equal it (the result of that resumed run says so
    under "resume_exact").
    start: None, or a capture dict: instead of the PID lap and the seeding, every controller is restored from its record, the
    clock and the scheduler state are set, and the run first repeats the poll the capture was taken at, under the new `laps`
    (groups that exchanged at that poll are not exchanged again), then steps on.  A run to 3 laps captured and resumed to 5
    therefore equals a run to 5 laps bit for bit (books, end states, health, exchange steps).  ValueError before any device work
    when start does not match the batch, the layout, the mode, the readiness, the poll interval, the pool groups or the tables,
    or when laps is not above the captured laps.
    lap_budget: None (every controller is stepped until the slowest has its laps), or the laps every controller drives before it
    retires, one integer or [batch] (BatchedController.set_lap_budget, installed after the seeding or the restore).  A retired
    controller costs no kernel time and keeps the state its last hand-over left it in, so with lap_budget = laps a controller ends
    where it would end alone, whoever else is in the batch; the polls leave retired controllers out, so the run stops once every
    controller has `laps` laps or has retired.  The result then holds the closed-loop steps the controllers really drove during
    the run ("driven_controller_steps_rank0", from the lap books and the records) and "driven_steps_per_s" beside
    controller_steps_per_s, which keeps meaning batch x steps / time; in the pooled mode also, per group, whether a controller had
    retired when the group last exchanged ("retired_before_last_exchange_rank0"): a retired controller's last lap never ships
    (nobody drives its rows past the finish line), so the exchange equals the run without a budget exactly when that is False
    everywhere.  capture records the budget; start refuses a budget below the captured one for any controller (raising it revives
    the controller where it stopped, with the noise draws of the later clock).
    lap_reports: None, or the report capacity L >= laps (BatchedController.enable_lap_reports, enabled before the PID lap): every
    controller then files one report per lap (steps, flags, unsolved QPs, lane violations of its plant state, interior-point
    iterations).  The result gains "lap_reports_rank0", a summary per lap (lap_report_summary), every per-table entry gains the same
    list under "reports", and "lap_stats_rank0" covers every lap, taken from the reports' steps (equal to the lap books' lengths
    wherever no step found the record full, flag 256).  Without reports laps is at most 16, the laps the lap books keep.  capture
    records L and start refuses another.  ValueError before any device work.
    lap_schedules: None, or {kind: rows} handed to BatchedController.set_lap_schedule after the seeding (or the restore), kind in
    "vehicle", "noise", "measurement", "surface" and rows [L] or [batch, L] naming rows of vehicle_sets, noise_sets,
    measurement_sets or surface_sets
    (conditions that change at the laps each controller reaches; entry 0 is the first LMPC lap).  Each kind needs its table and the
    run needs lap_reports >= laps.  The result gains "per_lap_row_rank0": per kind, lap and row, the controllers on that row, their
    mean steps, the share with a lane violation and the unsolved QPs (lap_row_summary).  capture records the schedules and start
    refuses others.  ValueError before any device work.
    trace: None, or a dict with "inst" (controller numbers) and "cap" (rows per controller): those controllers' LMPC steps are
    traced (lmpc_rollout_trace_create, after the seeding) and the dict receives per traced controller "steps" and the arrays "x"
    [cap, 6] (the plant state the step started from), "xPred" [cap, N+1, 6] and "lap" [cap]."""
    arguments = dict(locals())                                     # run()'s arguments, before any other name is bound
    given = {t.keyword: arguments[t.keyword] for t in TABLES}
    L = check_lap_reports(lap_reports, laps)
    packed, ctx = pack_tables(batch, warm, **given)
    # the rules between tables
    if "prediction_model_sets" in packed and not L:
        raise ValueError("prediction_model_sets needs lap_reports >= laps: the per-row summary is taken from the lap reports")
    if "track_sets" in packed and mode == "pooled" and len(packed["track_sets"][0]) > 1:
        if "pool_groups" not in packed:
            raise ValueError("the pooled mode exchanges laps between controllers: with %d tracks it needs pool groups that each drive "
                             "one track" % len(packed["track_sets"][0]))
        tidx, gidx = packed["track_sets"][1], packed["pool_groups"][1]
        for g in np.unique(gidx):
            if len(np.unique(tidx[gidx == g])) > 1:
                raise ValueError("pool group %d spans two tracks: a lap of another circuit is not a trajectory of this one" % g)
    scheds = check_lap_schedules(lap_schedules, batch, L, {kind: given[kind + "_sets"] for kind in _native.LAP_SCHEDULE_TABLES})
    budget = _native.make_lap_budget(lap_budget, int(batch))       # ValueError where set_lap_budget would refuse, before any device work
    rows_of = table_rows(packed)
    if start is not None:
        _check_start(start, batch, laps, mode, readiness, poll, warm, pool_groups, budget, shape_sets, L, scheds, rows_of)
    if capture is not None and not isinstance(capture, dict):
        raise ValueError("capture is a dict that receives the run's end state")
    if readiness not in ("batch", "group"):
        raise ValueError("readiness is 'batch' or 'group', got %r" % (readiness,))
    if readiness == "group" and mode != "pooled":
        raise ValueError("readiness='group' schedules the pooled exchange; the %s mode exchanges nothing" % mode)
    rank = dist.get_rank() if dist.is_initialized() else 0
    world = dist.get_world_size() if dist.is_initialized() else 1
    local = int(os.environ.get("LOCAL_RANK", 0)) if local is None else local
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    B = int(batch)
    N, M, numSS_it = ctx["N"], ctx["M"], ctx["numSS_it"]
    _, _, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, B, workloads.track_seg_table(), rp.TRACK_LENGTH, trToUse=TR_TO_USE, numSS_Points=M,
                          numSS_it=numSS_it, QterminalSlack=Qts, device=local, Tmax=TMAX, ss_cap=SS_CAP, model_cap=MODEL_CAP,
                          warm_start=warm)
    c.enable_rollout(Tcl=TCL)                            # before the tables: the measurement noise belongs to the closed loop
    if L:
        c.enable_lap_reports(L)                          # before the PID lap (its record is consumed by the seeding, unreported)
    for t in TABLES:
        if t.keyword in packed:
            getattr(c, t.install)(*t.args(given[t.keyword]))
    # every shipped lap has at least `ship_after` rows past its finish line: the readiness poll below guarantees it for the
    # slowest controllers of the batch, the export for the others (a group lapping faster holds laps that just ended)
    c.set_pool_min_overrun(ship_after)
    G = c.pool_groups
    stream = torch.cuda.ExternalStream(c.stream, device=dev)
    x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (B, 1))
    # ---- main.py:65-66 + 99-110 on the device: every controller drives its OWN PID lap (the full 100 s) and is seeded with it
    t0 = time.perf_counter()
    if start is None:
        c.rollout_set_state(x0, x0)
        for _ in range(1000):
            c.rollout_pid_step(0.8, seed=4321 + rank)
        c.rollout_seed_from_record_dev(copies=4)
        c.sync()
        pid_s = time.perf_counter() - t0
        c.rollout_set_state(x0, x0)
    else:                                                # the controllers and the clock of the captured run
        c.restore(start["records"])
        c.rollout_clock = int(start["clock"])
        c.sync()
        pid_s = 0.0
        restore_s = time.perf_counter() - t0
    for kind, row_of_lap in scheds.items():                # after the seeding: entry 0 is the first LMPC lap
        c.set_lap_schedule(kind, row_of_lap)
    if budget is not None:
        c.set_lap_budget(budget)
        driven0 = _driven_steps(c.books(), c.rollout_state())
        retired_at_last = [False] * G
    if trace is not None:
        tr_inst = np.ascontiguousarray(np.asarray(trace["inst"]).reshape(-1), np.int32)
        _native.check(_native.lib().lmpc_rollout_trace_create(c._h, len(tr_inst), _native.ptr(tr_inst), int(trace["cap"])))
    kbest = share + 1
    rows = torch.zeros(G * kbest, tpad, 9, dtype=torch.float64, device=dev)
    meta = torch.zeros(G * kbest, 4, dtype=torch.int32, device=dev)
    rows_all, meta_all = (rows, meta) if world == 1 else (torch.zeros(world * G * kbest, tpad, 9, dtype=torch.float64, device=dev),
                                                          torch.zeros(world * G * kbest, 4, dtype=torch.int32, device=dev))
    gidx = np.zeros(B, np.int64) if pool_groups is None else np.asarray(pool_groups[0]).reshape(B)
    # a group with no controller on any rank reports the empty-group sentinel everywhere and would count as ready: never exchange it
    live = sharding.sum_over_ranks(np.bincount(gidx, minlength=G), dev) > 0 if readiness == "group" else None
    sched = sharding.ExchangeSchedule(G, laps, ship_after, poll, readiness, mode == "pooled", live, capture is not None, start)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    max_steps = int(max_steps) or 300 * laps
    steps, n_xchg, xchg_s, took_total = sched.start_step, 0, 0.0, 0
    it_sum, it_n, it_max = 0.0, 0, 0                     # interior-point iterations, sampled at the polls
    it_ctrl = np.zeros(B)                                # ... per controller (the per-shape and per-lap-count means)
    l0 = c.kernel_launches
    e0.record(stream)
    while steps < max_steps or sched.repeat:
        if not sched.repeat:
            c.rollout_step(seed=seed + rank)
            c.rollout_commit_laps_dev()                   # every controller whose lap just ended hands it over, on the device
            steps += 1
            if steps % poll:
                continue
        # ---- poll: four integers of progress (per group); ranks agree on what happens next (same decision everywhere, no deadlock)
        prog = c.rollout_group_stats() if readiness == "group" else np.array([c.rollout_stats()])
        if not sched.repeat:                              # the repeated poll of a resumed run has no step of its own
            its = c.step_results()["iters"]
            it_sum += float(its.mean()); it_n += 1; it_max = max(it_max, int(its.max()))
            it_ctrl += its
        ready_g, done = sched.poll(steps, prog, dev)
        if ready_g.any():
            tx = time.perf_counter()
            with torch.cuda.stream(stream):
                c.pool_export(kbest, tpad, rank * B, rows, meta, groups=None if ready_g.all() else ready_g)
                if world > 1:
                    dist.all_gather_into_tensor(rows_all, rows)
                    dist.all_gather_into_tensor(meta_all, meta)
                took_total += c.pool_import(world * G * kbest, share, tpad, rank * B, rows_all, meta_all, count=True)
            xchg_s += time.perf_counter() - tx
            n_xchg += 1
            if budget is not None:
                retired = c.books()["lap_n"] >= budget
                for g in np.nonzero(ready_g)[0]:
                    retired_at_last[g] = bool(retired[gidx == g].any())
        if done:
            break
    e1.record(stream)
    c.sync()
    torch.cuda.synchronize()
    ms = sharding.max_over_ranks(e0.elapsed_time(e1), dev)
    bk = c.books()
    if capture is not None:
        tc = time.perf_counter()
        capture.update(records=c.snapshot(), clock=c.rollout_clock)
        c.sync()
        capture.update(capture_s=time.perf_counter() - tc, **sched.state(steps), batch=B, laps=laps, mode=mode, readiness=readiness,
                       poll=poll, warm=bool(warm), pool_groups=G, layout=c.snapshot_layout(),
                       lap_budget=None if budget is None else budget.tolist(),
                       lap_schedules={kind: row_of_lap.tolist() for kind, row_of_lap in scheds.items()}, tables=rows_of)
    if trace is not None:
        cap = int(trace["cap"])
        trace.update(steps=[], x=[], xPred=[], lap=[])
        for t in range(len(tr_inst)):
            n, x, xp, lp = C.c_int(0), np.zeros((cap, 6)), np.zeros((cap, N + 1, 6)), np.zeros(cap, np.int32)
            _native.check(_native.lib().lmpc_rollout_trace_get(c._h, t, C.byref(n), _native.ptr(x), None, None, _native.ptr(xp), None,
                                                               _native.ptr(lp)))
            for k, v in (("steps", n.value), ("x", x), ("xPred", xp), ("lap", lp)):
                trace[k].append(v)
    flags_or, unsolved = c.rollout_health()
    reps = c.lap_reports() if L else None
    bk.update(flags_or=flags_or, unsolved=unsolved, **({"lap_reports": reps} if L else {}),
              **({"lane_margins": c.lane_margin_values()} if "lane_margin_sets" in packed else {}))
    lens, n_laps = (reps["steps"], reps["n"]) if L else (bk["lap_hist"], bk["lap_n"])
    stats = []
    for r in range(laps):
        a = lens[n_laps > r, r]
        a = a if a.size else np.array([0])
        stats.append({"lap": r + 1, "n": int((n_laps > r).sum()), "mean": float(a.mean()), "min": int(a.min()), "max": int(a.max())})
    out = {"benchmark": "configs[3] LMPC Monte-Carlo rollouts", "mode": mode, "n_gpus": world, "batch_per_gpu": B,
           "closed_loop_steps": steps, "ms_total": ms, "controller_steps_per_s": B * world * (steps - sched.start_step) / (ms * 1e-3),
           "kernel_launches_rank0": int(c.kernel_launches - l0), "lap_stats_rank0": stats, "device_pid_laps_s": pid_s,
           "exchanges": n_xchg, "exchange_s_total": xchg_s, "exchange_ms_each": 1e3 * xchg_s / max(n_xchg, 1),
           "allgather_bytes_per_rank": int(rows.numel() * 8 + meta.numel() * 4), "laps_filed_rank0": took_total,
           "share": share, "ship_after": ship_after, "poll_every": poll, "warm_start": bool(warm),
           "ipm_iters_mean_sampled": it_sum / max(it_n, 1), "ipm_iters_max_sampled": it_max,
           "instances_with_flags_rank0": int((flags_or != 0).sum()), "flag_bits_rank0": int(np.bitwise_or.reduce(flags_or)),
           "unsolved_steps_rank0": int(unsolved.sum()), "late_accepts_rank0": c.late_accepts}
    if L:
        out["lap_reports"] = L
        out["lap_reports_rank0"] = lap_report_summary(reps, np.ones(B, bool), laps)
    if scheds:
        out["per_lap_row_rank0"] = lap_row_summary(reps, scheds, laps)
    out.update(table_stats(packed, ctx, bk, it_ctrl, it_n, laps))
    if pool_groups is not None:
        # a stored lap advances `it`: 4 seeded copies + every own lap handed over + every imported lap filed.  Exact unless an
        # own lap found the safe-set pool full (health flag 64): then that controller's count is one too low per such lap.
        filed = bk["it"].astype(np.int64) - 4 - bk["lap_n"]
        out["pool_groups"] = G
        out["laps_filed_per_group_rank0"] = [int(filed[gidx == g].sum()) for g in range(G)]
    if pool_groups is not None or readiness == "group":
        out["readiness"] = readiness
        out["exchange_steps_per_group_rank0"] = sched.exchange_steps
    if budget is not None:
        driven = _driven_steps(bk, c.rollout_state()) - driven0
        out["lap_budget"] = int(budget[0]) if (budget == budget[0]).all() else "per controller, %d .. %d" % (budget.min(), budget.max())
        out["driven_controller_steps_rank0"] = driven
        out["driven_steps_per_s"] = driven / (ms * 1e-3)
        if mode == "pooled":
            out["retired_before_last_exchange_rank0"] = retired_at_last
    if start is not None:
        out["resumed_from_step"] = int(start["steps"])
        out["restore_s"] = restore_s
        out["resume_exact"] = start["diverged_step"] is None
    if capture is not None:
        out["capture_s"] = capture["capture_s"]
    if final is not None:
        final.update(c.rollout_state())
        final.update(c.step_results())
    if books is not None:
        books.update(bk)
    c.close()
    return out


def _driven_steps(bk, state):
    """Closed-loop steps the controllers have driven since the seeding: the laps handed over plus the lap under way."""
    n = np.minimum(bk["lap_n"], bk["lap_hist"].shape[1])
    filed = np.where(np.arange(bk["lap_hist"].shape[1])[None, :] < n[:, None], bk["lap_hist"], 0)
    return int(filed.sum(dtype=np.int64) + state["cl_len"].sum(dtype=np.int64))


def _check_start(start, batch, laps, mode, readiness, poll, warm, pool_groups, budget=None, shape_sets=None, lap_reports=0,
                 lap_schedules=None, tables=None):
    """The refusals of run(start=...), before any device work: a start that does not match this run (report capacity, lap
    schedules and tables, {keyword: rows} of table_rows, included; a start without "tables" was captured without any), laps not
    above the captured laps, or a lap budget below the captured one."""
    if not isinstance(start, dict):
        raise ValueError("start is a capture dict of an earlier run")
    need = ("records", "clock") + sharding.ExchangeSchedule.FIELDS + ("batch", "laps", "mode", "readiness", "poll", "warm",
                                                                      "pool_groups", "layout")
    missing = [k for k in need if k not in start]
    if missing:
        raise ValueError("start lacks %s: pass the dict run(capture=...) filled" % ", ".join(missing))
    for key, mine in (("batch", int(batch)), ("mode", mode), ("readiness", readiness), ("poll", int(poll)), ("warm", bool(warm))):
        if start[key] != mine:
            raise ValueError("start was captured with %s = %r, this run has %r" % (key, start[key], mine))
    G = 1 if pool_groups is None else int(pool_groups[1])
    if int(start["pool_groups"]) != G:
        raise ValueError("start was captured with %d pool groups, this run has %d" % (int(start["pool_groups"]), G))
    if int(laps) <= int(start["laps"]):
        raise ValueError("laps (%d) must be above the captured run's laps (%d)" % (int(laps), int(start["laps"])))
    had = start.get("lap_budget")
    if had is not None and budget is not None and (budget < np.asarray(had)).any():
        raise ValueError("lap_budget is below the captured run's for %d controller(s): a budget can only be raised or removed"
                         % int((budget < np.asarray(had)).sum()))
    rec = start["records"]
    if getattr(rec, "shape", (None,))[0] != int(batch):
        raise ValueError("start holds %s records, this run has %d controllers" % (getattr(rec, "shape", ("no",))[0], int(batch)))
    had = int(start["layout"].get("lap_reports", 0))
    if had != int(lap_reports):
        raise ValueError("start records have lap_reports = %d, this run %d" % (had, int(lap_reports)))
    had = {k: np.asarray(v) for k, v in (start.get("lap_schedules") or {}).items()}
    mine = lap_schedules or {}
    if sorted(had) != sorted(mine) or any(not np.array_equal(had[k], mine[k]) for k in had):
        raise ValueError("start was captured with lap_schedules for %s, this run has %s (or other rows): a run resumes under the "
                         "schedules it was captured with" % (sorted(had) or "none", sorted(mine) or "none"))
    for k, v in layout(warm, shape_sets).items():
        if int(start["layout"].get(k, -1)) != v:
            raise ValueError("start records have %s = %s, this run's controllers %d" % (k, start["layout"].get(k), v))
    check_start_tables(start.get("tables", {}), tables or {})                 # a start without "tables" was taken without any


def table_stats(packed, ctx, bk, it_ctrl, it_n, laps):
    """The result's entries of the tables (pack_tables' packed and ctx): per row of every table with a result key, _set_stats of
    its controllers, its declared fields and, where declared, their interior-point iterations per poll (it_ctrl: every
    controller's sum over it_n sampled polls); then the entries that join tables: "handle_shape", the (shape, lap count) cells
    "per_shape_ss_laps_rank0", under lane rules the lane-unsafe shares (lap_reports_rank0 again, with them) and
    "lane_unsafe_selected_share_rank0", and under lane margins "lane_margin_final_rank0".  bk holds the lap books, "flags_or",
    "unsolved" and, where run() has them, "lap_reports" and "lane_margins"."""
    flags_or, unsolved, reps = bk["flags_or"], bk["unsolved"], bk.get("lap_reports")
    everyone = np.ones(len(flags_or), bool)

    def entry(sel):
        return _set_stats(bk, flags_or, unsolved, sel, laps, reps)

    def ipm(sel):
        return float(it_ctrl[sel].mean() / max(it_n, 1)) if sel.any() else 0.0
    out = {}
    for t in TABLES:
        if t.key is not None and t.keyword in packed:
            rows, idx = packed[t.keyword]
            out[t.key] = []
            for k, row in enumerate(rows):
                s = entry(idx == k)
                s.update({f: getattr(row, f) for f in t.fields})
                if t.ipm:
                    s["ipm_iters_mean_sampled"] = ipm(idx == k)
                out[t.key].append(s)
    if "shape_sets" in packed:
        out["handle_shape"] = [ctx["N"], ctx["M"]]
    if "shape_sets" in packed and "ss_laps_sets" in packed:
        (shapes, sidx), (values, lidx) = packed["shape_sets"], packed["ss_laps_sets"]
        out["per_shape_ss_laps_rank0"] = []
        for j, sh in enumerate(shapes):
            for k, v in enumerate(values):
                cell = (sidx == j) & (lidx == k)
                if cell.any():
                    s = entry(cell)
                    s.update(N=sh.N, numSS_Points=sh.numSS_Points, numSS_it=v.numSS_it, ipm_iters_mean_sampled=ipm(cell))
                    out["per_shape_ss_laps_rank0"].append(s)
    if "lane_rule_sets" in packed:
        idx = packed["lane_rule_sets"][1]
        if reps is not None:
            for k, s in enumerate(out["per_lane_rule_rank0"]):
                _add_unsafe_share(s["reports"], reps, idx == k, laps)
            out["lap_reports_rank0"] = lap_report_summary(reps, everyone, laps)
            _add_unsafe_share(out["lap_reports_rank0"], reps, everyone, laps)
        _, unsafe = _native.split_lane_key(bk["ss_time"])
        held = np.array([unsafe[b, bk["sel"][b, :nit]].any() for b, nit in enumerate(ctx["laps_of"])])
        out["lane_unsafe_selected_share_rank0"] = float(held.mean())
    if "lane_margin_sets" in packed:
        idx, m_end = packed["lane_margin_sets"][1], bk["lane_margins"]
        out["lane_margin_final_rank0"] = []
        for k in range(len(packed["lane_margin_sets"][0])):
            m = m_end[idx == k]
            out["lane_margin_final_rank0"].append({"row": k, "n": int(m.size), "min": float(m.min()) if m.size else 0.0,
                                                   "mean": float(m.mean()) if m.size else 0.0,
                                                   "max": float(m.max()) if m.size else 0.0})
    return out


def _add_unsafe_share(rows, reps, sel, laps):
    """Adds "lane_unsafe_share" to every per-lap row of lap_report_summary: the share of the controllers `sel` that filed lap r whose
    report carries the lane-unsafe bit (their own lap was judged lane-unsafe at its hand-over)."""
    for r, row in enumerate(rows[:laps]):
        m = sel & (reps["n"] > r)
        row["lane_unsafe_share"] = float(((reps["flags"][m, r] & _native.REPORT_LANE_UNSAFE) != 0).mean()) if m.any() else 0.0


def _set_stats(bk, flags_or, unsolved, sel, laps, reps=None):
    """Lap lengths (mean / min per LMPC lap), unsolved steps and flagged controllers of the controllers `sel` of one parameter set or
    vehicle; with reports (BatchedController.lap_reports) the lengths are the reports' steps and "reports" holds lap_report_summary."""
    lens, n_laps = (reps["steps"], reps["n"]) if reps is not None else (bk["lap_hist"], bk["lap_n"])
    laps_out = []
    for r in range(laps):
        m = sel & (n_laps > r)
        a = lens[m, r]
        laps_out.append({"lap": r + 1, "n": int(m.sum()), "mean": float(a.mean()) if a.size else 0.0, "min": int(a.min()) if a.size else 0})
    out = {"controllers": int(sel.sum()), "laps": laps_out, "unsolved_steps": int(unsolved[sel].sum()),
           "instances_with_flags": int((flags_or[sel] != 0).sum())}
    if reps is not None:
        out["reports"] = lap_report_summary(reps, sel, laps)
    return out


def lap_report_summary(reps, sel, laps):
    """Per lap r < laps, over the controllers `sel` that filed a report of lap r (BatchedController.lap_reports): how many, their
    steps (mean / min / max), how many violated a lane constraint at some step and the mean violating steps, the max and mean of
    viol_max, the unsolved QPs in total and the interior-point iterations per step (total iterations over total steps)."""
    out = []
    for r in range(laps):
        m = sel & (reps["n"] > r)
        k = int(m.sum())
        st, vs, vm = reps["steps"][m, r], reps["viol_steps"][m, r], reps["viol_max"][m, r]
        tot = int(st.sum(dtype=np.int64))
        out.append({"lap": r + 1, "controllers": k,
                    "steps_mean": float(st.mean()) if k else 0.0, "steps_min": int(st.min()) if k else 0, "steps_max": int(st.max()) if k else 0,
                    "violating": int((vs > 0).sum()), "viol_steps_mean": float(vs.mean()) if k else 0.0,
                    "viol_max_max": float(vm.max()) if k else 0.0, "viol_max_mean": float(vm.mean()) if k else 0.0,
                    "unsolved": int(reps["unsolved"][m, r].sum(dtype=np.int64)),
                    "ipm_iters_per_step": float(reps["ipm_iters"][m, r].sum(dtype=np.int64)) / tot if tot else 0.0})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8192, help="instances per GPU")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps every instance has to finish")
    ap.add_argument("--max-steps", type=int, default=0, help="0 = 300 per lap")
    ap.add_argument("--mode", choices=["independent", "pooled"], default="pooled")
    ap.add_argument("--share", type=int, default=2, help="pooled mode: globally fastest laps handed to every instance per exchange")
    ap.add_argument("--tpad", type=int, default=288, help="rows per exchanged lap (lap + addPoint overrun)")
    ap.add_argument("--ship-after", type=int, default=40, help="pooled mode: steps into the next lap before a lap is shipped")
    ap.add_argument("--poll", type=int, default=8, help="closed-loop steps between progress polls")
    ap.add_argument("--warm", action="store_true", help="warm-started interior-point solves (lmpc_params.warm_start)")
    ap.add_argument("--lap-budget", type=int, default=0, help="laps after which a controller retires and costs no kernel time; 0 = none")
    args = ap.parse_args()
    world, local = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    out = run(args.batch, args.laps, args.mode, args.share, args.tpad, args.ship_after, args.poll, args.max_steps, local=local, warm=args.warm,
              lap_budget=args.lap_budget or None)
    if (dist.get_rank() if dist.is_initialized() else 0) == 0:
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
