"""Batched LTV-MPC / LMPC controllers: B independent reference controllers advanced in lock-step.

State machine = src/fnc/controller/PredictiveControllers.py (MPC.solve :110-137, LMPC.addTrajectory :418-445,
LMPC.addPoint :466-476, LMPC.addTerminalComponents :386-416) + PredictiveModel.addTrajectory
(PredictiveModel.py:35-46).  Everything numeric runs on the GPU (csrc/safeset.cuh, csrc/ftocp_pdip.cuh);
this file only does the once-per-lap bookkeeping that decides WHICH stored laps are "the numSS_it fastest"
and "usedIt", exactly as the reference's Python lists do.
"""
import ctypes as C
import numpy as np
from . import _native as nat
from . import reference_params


class _LapBook:
    """Host-side index of one instance's laps in a device pool (slot ids, lengths, lap numbers)."""

    def __init__(self, cap):
        self.cap = cap
        self.slot_of = {}          # lap number -> slot
        self.free = list(range(cap))

    def take(self, lap):
        if not self.free:
            raise RuntimeError("lap pool full")
        s = self.free.pop(0)
        self.slot_of[lap] = s
        return s

    def drop(self, lap):
        self.free.append(self.slot_of.pop(lap))


class BatchedController:
    def __init__(self, params, batch, seg_table, TrackLength, trToUse=1, numSS_Points=0, numSS_it=0,
                 QterminalSlack=None, device=0, Tmax=2048, ss_cap=None, model_cap=None,
                 eps_res=0.0, eps_gap=0.0, max_iter=0, model_kwargs=None, warm_start=False):
        L = nat.lib()
        self._lib = L
        self.B, self.N, self.M = int(batch), int(params.N), int(numSS_Points)
        self.numSS_it, self.trToUse = int(numSS_it), int(trToUse)
        self.TrackLength = float(TrackLength)
        self.lmpc = self.M > 0
        self.ncx = np.asarray(params.Fx).shape[0]
        self.Tmax = int(Tmax)
        self._p = nat.make_params(params, numSS_Points, numSS_it, QterminalSlack, eps_res, eps_gap, max_iter, warm_start=warm_start)
        h = C.c_void_p()
        nat.check(L.lmpc_create(C.byref(self._p), self.B, int(device), C.byref(h)))
        self._h = h
        self._device = int(device)
        self.ss_cap = int(ss_cap) if ss_cap is not None else (self.numSS_it + 2 if self.lmpc else 0)
        self.model_cap = int(model_cap) if model_cap is not None else self.trToUse + 1
        self._mp = nat.make_model_params(seg_table, TrackLength, trToUse, **(model_kwargs or {}))
        nat.check(L.lmpc_store_create(self._h, C.byref(self._mp), self.ss_cap, self.model_cap, self.Tmax))
        # per-instance bookkeeping (PredictiveModel.lapTime / LMPC.LapTime lists)
        self.model_laps = [[] for _ in range(self.B)]       # ordered (T, lapno) like xStored (ascending T)
        self.model_book = [_LapBook(self.model_cap) for _ in range(self.B)]
        self.model_count = [0] * self.B
        self.LapTime = [[] for _ in range(self.B)]          # LMPC.LapTime
        self.ss_book = [_LapBook(max(self.ss_cap, 1)) for _ in range(self.B)]
        self.it = [0] * self.B
        self.own_laps = [[] for _ in range(self.B)]         # lap numbers of the laps the instance drove itself
        self._sel_dirty = True
        self._used_dirty = False
        # device-side copies of the lap bookkeeping are rebuilt only for instances whose laps changed (None = all)
        self._sel_rows, self._used_rows = None, None
        nit = max(self.numSS_it, 1)
        self.device_books = False
        self._pool_groups = 1
        self._shapes = None                                 # (shapes, index) of set_shapes, or None: the handle's own shape
        self._ss_laps = None                                # numSS_it of every controller (set_ss_laps), or None: the handle's
        self._windows = None                                # [B, 2] (ss_window, model_window) of set_lap_windows, or None: unbounded
        self._lane = None                                   # [(mode, lane_tol)] * B of set_lane_rules, or None: the reference's rule
        self._margins = None                                # (rows, index) of set_lane_margins, or None: no margin
        self._models = None                                 # (rows, index) of set_prediction_models, or None: all learned
        self._bx_min = np.full(self.B, self._row_bx_min(self._p))   # min_i bx_i of the QP row every controller reads
        # rows of the plant-side tables a lap schedule indexes (the defaults: one reference vehicle and noise, no measurement or
        # surface table) and the installed schedules [B, L] of set_lap_schedule
        self._table_rows = {"vehicle": 1, "noise": 1, "measurement": 0, "surface": 0}
        self._surfaces = None                               # (rows, index) of set_surfaces, or None: no surface table
        self._lap_schedules = {}
        self._sel = np.zeros((self.B, nit), np.int32); self._isp = np.zeros((self.B, nit), np.int32)
        self._prev = -np.ones(self.B, np.int32); self._used = np.zeros((self.B, self.trToUse), np.int32)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.lmpc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def kernel_launches(self):
        return int(self._lib.lmpc_kernel_launches(self._h))

    @property
    def late_accepts(self):
        """QPs accepted at the 1e-6 safety-net tolerance instead of eps_res / eps_gap since creation (expected 0)."""
        return int(self._lib.lmpc_late_accepts(self._h))

    def _install(self, call, what, sets, index, pack):
        """One set call of a per-controller table: ``sets=None`` (no index) reverts to the table's default, else ``pack()`` returns
        the rows and the index (raising ValueError where the library would refuse)."""
        if sets is None:
            if index is not None:
                raise ValueError("%s=None reverts to the default and takes no index" % what)
            nat.check(call(self._h, None, 0, None))
            return
        rows, idx = pack()
        nat.check(call(self._h, rows, len(rows), nat.ptr(idx)))

    def set_param_sets(self, params, index=None, QterminalSlack=None):
        """Per-controller QP parameters (a parameter sweep in one batch): controller b solves with ``params[index[b]]`` (objects
        with the reference's MPCParams field names; every field but N and the constraint row counts may differ) and, for LMPC,
        ``QterminalSlack[index[b]]`` (None: the handle's).  ``index`` is required with ``params``.  ``params=None`` (no index)
        returns to the parameters the handle was created with.
        Waits for work already enqueued; warm-start records start over."""
        packed = {}

        def pack():
            rows, idx = nat.make_param_sets(self._p, params, index, self.B, self._p.numSS_Points, self.numSS_it, QterminalSlack)
            packed["bx_min"] = np.array([self._row_bx_min(rows[k]) for k in range(len(rows))])[idx]
            if self._margins is not None:                    # an installed margin must still leave a lane of the new rows
                nat.check_margins_leave_lane(self._margins[0], self._margins[1], packed["bx_min"])
            return rows, idx
        if params is None and self._margins is not None:
            nat.check_margins_leave_lane(self._margins[0], self._margins[1], np.full(self.B, self._row_bx_min(self._p)))
        self._install(self._lib.lmpc_set_param_sets, "params", params, index, pack)
        self._bx_min = packed.get("bx_min", np.full(self.B, self._row_bx_min(self._p)))

    @staticmethod
    def _row_bx_min(p):
        """min_i bx_i of the lane rows of a Params row"""
        return float(min(p.bx[i] for i in range(int(p.ncx))))

    def set_lane_margins(self, margins, index=None):
        """Per-controller lane margins (constraint tightening): every QP controller b solves plans inside its lane narrowed by a
        margin m_b -- bx_i - m_b for every lane row -- while its lap reports, lane rules and adaptation judge the lane it was
        given.  ``margins[index[b]]`` (objects with ``mode``, ``margin0``, ``margin_max``, ``step_up``, ``step_down``, e.g.
        reference_params.LaneMarginParams): mode 0 no margin, mode 1 the fixed margin0, mode 2 a margin that starts at margin0 (at
        this call and at every seeding) and after every own lap handed over on the device rises by step_up (a lap that left the
        lane, capped at margin_max) or falls by step_down (one that kept to it, floored at margin0).  ``index`` is required with
        ``margins``; ``margins=None`` (no index) removes the table.  A margin must leave a lane: margin0 (mode 1) or margin_max
        (mode 2) below min_i bx_i of the controller's QP row.  Allowed at any time; warm-start records start over; under a mode 2
        row the host-slot hand-over is refused.  m_b is part of a snapshot, the table is not.  ValueError before any native call
        where the library would refuse a value.  Waits for work already enqueued."""
        packed = {}

        def pack():
            packed["v"] = nat.make_lane_margin_sets(margins, index, self.B, self._bx_min)
            return packed["v"]
        self._install(self._lib.lmpc_set_lane_margins, "margins", margins, index, pack)
        self._margins = packed.get("v")

    def lane_margins_of(self, inst):
        """(mode, margin0, margin_max, step_up, step_down) of controller ``inst`` under ``set_lane_margins``, None without a
        table."""
        if self._margins is None:
            return None
        r = self._margins[0][int(self._margins[1][int(inst)])]
        return (int(r.mode), float(r.margin0), float(r.margin_max), float(r.step_up), float(r.step_down))

    def lane_margin_values(self):
        """m_b of every controller, float64 [B] (synchronises); ValueError without a lane-margin table."""
        if self._margins is None:
            raise ValueError("lane_margin_values: no lane-margin table is installed")
        m = np.zeros(self.B, np.float64)
        nat.check(self._lib.lmpc_get_lane_margins(self._h, nat.ptr(m)))
        return m

    def set_prediction_models(self, models, index=None):
        """Per-controller prediction models: where rows 0..2 (vx, vy, wz) of controller b's LTV model come from in every later
        ``identify``, ``step`` (modes 0, 1) and ``rollout_step`` (modes 0, 1).  ``models[index[b]]`` (objects with ``mode`` and
        ``vehicle``, e.g. reference_params.PredictionModelParams): mode 0 the k-NN regression (the reference), mode 1 the exact
        linearisation of the simulator's one-period map for ``vehicle``, mode 2 that of the plant's own vehicle row (through
        the vehicle lap schedule in ``rollout_step``).  Rows 3..5 stay the closed-form kinematic rows.  A nominal controller keeps
        filing laps, and never sets step flags 1, 4 or 32; it sets FLAG_NOMINAL_NONFINITE when its rows 0..2 are not finite.
        ``index`` is required with ``models``; ``models=None`` (no index) removes the table.  Allowed at any time; not part of a
        snapshot.  ValueError before any native call where the library would refuse a value.  Waits for work already enqueued."""
        packed = {}

        def pack():
            packed["v"] = nat.make_prediction_model_sets(models, index, self.B)
            return packed["v"]
        self._install(self._lib.lmpc_set_prediction_models, "models", models, index, pack)
        self._models = packed.get("v")

    def prediction_models_of(self, inst):
        """(mode, vehicle as a reference_params.VehicleParams) of controller ``inst`` under ``set_prediction_models``, None
        without a table."""
        if self._models is None:
            return None
        r = self._models[0][int(self._models[1][int(inst)])]
        return (int(r.mode), reference_params.VehicleParams(*[float(getattr(r.vehicle, f)) for f in nat.VEHICLE_FIELDS]))

    def set_vehicles(self, vehicles, index=None):
        """Per-controller vehicles of the device simulator (a Monte-Carlo over the plant in one batch): controller b is driven
        with ``vehicles[index[b]]`` (objects with the reference's ten field names, e.g. reference_params.VehicleParams) by every
        later ``rollout_step`` and ``rollout_pid_step``.  ``index`` is required with ``vehicles``.  ``vehicles=None`` (no index)
        returns to the reference vehicle.  Independent of ``set_param_sets``.  While a vehicle lap schedule is installed the new
        table must cover its largest entry (ValueError).  Waits for work already enqueued."""
        rows = 1 if vehicles is None else len(vehicles)
        self._check_schedule_cover("vehicle", rows)
        self._install(self._lib.lmpc_rollout_set_vehicles, "vehicles", vehicles, index,
                      lambda: nat.make_vehicle_sets(vehicles, index, self.B))
        self._table_rows["vehicle"] = rows

    def set_surfaces(self, surfaces, index=None):
        """Per-controller track surfaces of the device simulator (friction zones along the circuit): in every later
        ``rollout_step`` (through the surface lap schedule when one is installed) and ``rollout_pid_step``, each simulator sub-step
        of controller b whose s -- wrapped as the curvature lookup wraps it -- lies in [s_start, s_end) of a zone of
        ``surfaces[index[b]]`` (objects with ``zones``, e.g. reference_params.SurfaceParams) drives with peak tyre forces
        fl(mu_f Df) and fl(mu_r Dr); every other sub-step drives the car's own Df and Dr exactly.  A mode 2 prediction model
        (``set_prediction_models``) plans with the same surface.  ``index`` is required with ``surfaces``; ``surfaces=None`` (no
        index) removes the table.  While a surface lap schedule is installed the new table must cover its largest entry, and it
        cannot be removed (ValueError).  Allowed at any time; not part of a snapshot.  ValueError before any native call where the
        library would refuse a value.  Waits for work already enqueued."""
        rows = 0 if surfaces is None else len(surfaces)
        self._check_schedule_cover("surface", rows)
        packed = {}

        def pack():
            packed["v"] = nat.make_surface_sets(surfaces, index, self.B)
            return packed["v"]
        self._install(self._lib.lmpc_rollout_set_surfaces, "surfaces", surfaces, index, pack)
        self._surfaces = packed.get("v")
        self._table_rows["surface"] = rows

    def surface_of(self, inst):
        """The zones of controller ``inst``'s surface under ``set_surfaces`` as a reference_params.SurfaceParams, None without a
        table."""
        if self._surfaces is None:
            return None
        r = self._surfaces[0][int(self._surfaces[1][int(inst)])]
        return reference_params.SurfaceParams(tuple(tuple(r.zone[4 * j:4 * j + 4]) for j in range(r.nzone)))

    def set_noise(self, noises, index=None):
        """Per-controller noise models of the device closed loop (a robustness study in one batch): controller b draws the
        simulator's and the PID's noise with ``noises[index[b]]`` (objects with the fields of reference_params.NoiseParams) in
        every later ``rollout_step`` and ``rollout_pid_step``, Philox or host-given draws alike.  ``index`` is required with
        ``noises``.  ``noises=None`` (no index) returns to the reference's noise.  Independent of ``set_param_sets``,
        ``set_vehicles``, ``set_tracks`` and the pool groups; allowed in the middle of a run.  While a noise lap schedule is
        installed the new table must cover its largest entry (ValueError).  Waits for work already enqueued."""
        rows = 1 if noises is None else len(noises)
        self._check_schedule_cover("noise", rows)
        self._install(self._lib.lmpc_rollout_set_noise, "noises", noises, index, lambda: nat.make_noise_sets(noises, index, self.B))
        self._table_rows["noise"] = rows

    def set_noise_streams(self, streams=None):
        """Common random numbers: the Philox draws of controller b are keyed by ``streams[b]`` (integers >= 0, repeats allowed)
        instead of b, so controllers on one stream meet the same noise -- e.g. two tunings interleaved with ``streams = b // 2``
        share their PID lap, their seeded stores and every later draw.  ``streams=None`` returns to stream b = b.  Host-given
        draws do not use the streams.  Waits for work already enqueued."""
        s = nat.make_noise_streams(streams, self.B)
        nat.check(self._lib.lmpc_rollout_set_noise_streams(self._h, nat.ptr(s)))

    def set_measurement_noise(self, meas=None, index=None):
        """Per-controller measurement noise of the device closed loop (how much sensor noise learning from one's own laps
        absorbs): in every later ``rollout_step`` and ``rollout_pid_step`` controller b sees y = x + clip(z * sigma, +-clip) on
        (vx, vy, wz, epsi, s, ey) with ``meas[index[b]]`` (objects with the fields of reference_params.MeasurementParams) instead
        of the plant state x: its QP, safe-set selection, addPoint, PID input and closed-loop record all take y, so its stored
        laps and learned models are measured data.  The plant, ``rollout_state`` and the trace keep x.  The draws are Philox,
        keyed apart from the process and PID noise and paired by ``set_noise_streams``.  ``index`` is required with ``meas``.
        ``meas=None`` (no index) removes the table: the controllers read x again and no kernel is added to a step.  Needs
        ``enable_rollout``; allowed in the middle of a run; not part of a snapshot.  While a measurement lap schedule is installed
        the new table must cover its largest entry, and it cannot be removed (ValueError).  Waits for work already enqueued."""
        rows = 0 if meas is None else len(meas)
        self._check_schedule_cover("measurement", rows)
        self._install(self._lib.lmpc_rollout_set_measurement_noise, "meas", meas, index,
                      lambda: nat.make_measurement_sets(meas, index, self.B))
        self._table_rows["measurement"] = rows

    def set_observers(self, observers=None, index=None):
        """Per-controller state observers of the device closed loop (a fixed-gain predictor-corrector on a noisy sensor): in every
        later ``rollout_step`` of mode 0 or 1 a controller whose row ``observers[index[b]]`` (objects with ``mode`` and ``gain``,
        e.g. reference_params.ObserverParams) has mode 1 reads x_hat_j = p_j + gain_j (y_j - p_j) on (vx, vy, wz, epsi, s, ey) in
        place of y, the measured state (``set_measurement_noise``) or the plant state: p is its own prediction xPred[1] of the
        previous step, its s wrapped back by TrackLength after a hand-over.  Its QP, safe-set selection, addPoint and closed-loop
        record all take x_hat, so its stored laps and learned models are filtered data.  Gain 1 copies y, gain 0 takes p.  Without
        a prior (the first step after the seeding, after a PID or mode 2 step, which clear it) x_hat = y; a non-finite prior
        gives x_hat = y and the step flag FLAG_OBSERVER_RESET.  Mode 0 rows read y.  The plant, ``rollout_state``, the trace and
        the lap reports keep x; x_hat of the step is ``read_buffer("x_est", ...)``.  ``index`` is required with ``observers``.
        ``observers=None`` (no index) removes the table: no kernel is added to a step.  Needs ``enable_rollout``; allowed in the
        middle of a run; not part of a snapshot.  ValueError before any native call where the library would refuse a value.
        Waits for work already enqueued."""
        self._install(self._lib.lmpc_rollout_set_observers, "observers", observers, index,
                      lambda: nat.make_observer_sets(observers, index, self.B))

    def set_observer_priors(self, priors=None, index=None):
        """Where the state observers (``set_observers``) take their prior from, per controller: ``priors[index[b]]`` (objects with
        ``source`` and ``vehicle``, e.g. reference_params.ObserverPrior).  Source 0 is the controller's own plan xPred[1], exactly
        as without a table.  Sources 1 and 2 carry the estimate the controller read in its previous step, xPredPrev[0], over one
        control period under the input it applied, OldInput, with the simulator's noise-free map: source 1 for ``vehicle``
        without a surface, source 2 for the plant's own vehicle and surface rows of that step (through their lap schedules).
        The prior then gets the lap-wrap fix and the observer's blend.  A non-finite input or prior, or a failed curvature
        lookup, gives x_hat = y and FLAG_OBSERVER_RESET.  The prior of the step is ``read_buffer("x_prior", ...)`` (NaN where
        none was formed).  ``index`` is required with ``priors``; ``priors=None`` (no index) removes the table.  Adds no launch;
        without an observer table it does nothing.  Needs ``enable_rollout``; allowed in the middle of a run; not part of a
        snapshot.  ValueError before any native call where the library would refuse a value.  Waits for work already enqueued."""
        self._install(self._lib.lmpc_rollout_set_observer_priors, "priors", priors, index,
                      lambda: nat.make_observer_prior_sets(priors, index, self.B))

    def set_observer_gains(self, gains=None, index=None):
        """Which gains the state observers (``set_observers``) blend with, per controller: ``gains[index[b]]`` (objects with
        ``mode``, ``q`` and ``r``, e.g. reference_params.ObserverGains).  Mode 0 keeps the observer row's fixed gains, exactly as
        without a table.  Mode 1, for a controller whose observer prior (``set_observer_priors``) is a car (source 1 or 2): every
        step of mode 0 or 1 linearises the prior's one-period map at its point, A = dPhi/dx, solves the filter DARE for that A
        with Q = diag(q), R = diag(r), and blends x_hat = p + K (y - p) with K = P (P + R)^-1.  No covariance is carried from step
        to step.  A, P and K of the step are ``read_buffer("obs_jac" / "obs_cov" / "obs_gain", ...)`` [B, 6, 6], NaN where no gain
        was formed; a gain that could not be formed gives x_hat = y and FLAG_OBSERVER_GAIN.  One more launch per step of mode 0 or
        1.  ``index`` is required with ``gains``; ``gains=None`` (no index) removes the table.  Needs ``enable_rollout``; allowed
        in the middle of a run; not part of a snapshot.  ValueError before any native call where the library would refuse a
        row; NativeError for a mode 1 row of a controller without a car prior.  Waits for work already enqueued."""
        self._install(self._lib.lmpc_rollout_set_observer_gains, "gains", gains, index,
                      lambda: nat.make_observer_gain_sets(gains, index, self.B))

    def set_lap_budget(self, budget=None):
        """Lap budgets of the device closed loop: controller b retires once it has handed over ``budget[b]`` laps (one integer
        >= 1 for the whole batch, or one per controller).  A retired controller keeps the state its last hand-over left it in and
        no kernel of ``rollout_step`` / ``rollout_commit_laps_dev`` works for it, so a batch whose controllers need different
        numbers of steps stops paying for the finished ones and each ends in the state it would end in alone.  Raising the budget
        later revives a controller where it stopped.  ``budget=None`` removes the budgets.  Needs ``enable_rollout``; allowed in
        the middle of a run; not part of a snapshot.  Waits for work already enqueued."""
        b = nat.make_lap_budget(budget, self.B)
        nat.check(self._lib.lmpc_rollout_set_lap_budget(self._h, nat.ptr(b)))

    def _check_schedule_cover(self, kind, rows):
        """Both install orders of a lap schedule: a table of `rows` rows must cover the largest entry of an installed schedule."""
        s = self._lap_schedules.get(kind)
        if s is not None and int(s.max()) >= rows:
            raise ValueError("the %s lap schedule names row %d and the new table has %d row(s): install a covering schedule first "
                             "or remove it" % (kind, int(s.max()), rows))

    def set_lap_schedule(self, kind, rows=None):
        """Lap schedules of the device closed loop (conditions that change while the controllers learn: a track that gets wet at
        lap 10, a car whose mass changes, a sensor that degrades, a corner that gets wet): ``kind`` is "vehicle", "noise",
        "measurement" or "surface", and in every later ``rollout_step`` controller b drives LMPC lap k (k = 0 is the first lap after
        the seeding, lap_n of ``books``) under row ``rows[b][min(k, L - 1)]`` of that table (``set_vehicles``, ``set_noise``,
        ``set_measurement_noise``, ``set_surfaces``) in place
        of its index.  ``rows`` is [L] (the same for every controller) or [batch, L], 1 <= L <= 1024, entries in the table's rows;
        ``rows=None`` removes the schedule.  The change takes effect on the first step after the hand-over that advanced lap_n
        (``rollout_commit_laps_dev``; the host-slot hand-over does not count laps).  The PID lap ignores schedules.  Needs
        ``enable_rollout``; allowed at any time; not part of a snapshot (lap_n is, so a restored controller resumes at its entry).
        ValueError before any native call where the library would refuse.  Waits for work already enqueued."""
        if kind not in nat.LAP_SCHEDULE_TABLES:
            raise ValueError("kind is one of %s, got %r" % (sorted(nat.LAP_SCHEDULE_TABLES), kind))
        if not hasattr(self, "Tcl"):
            raise ValueError("set_lap_schedule needs enable_rollout first")
        k = nat.LAP_SCHEDULE_TABLES[kind]
        if rows is None:
            nat.check(self._lib.lmpc_rollout_set_lap_schedule(self._h, k, 0, None))
            self._lap_schedules.pop(kind, None)
            return
        if kind == "measurement" and not self._table_rows[kind]:
            raise ValueError("a measurement lap schedule needs a measurement table (set_measurement_noise)")
        if kind == "surface" and not self._table_rows[kind]:
            raise ValueError("a surface lap schedule needs a surface table (set_surfaces)")
        s = nat.make_lap_schedule(rows, self.B, self._table_rows[kind])
        nat.check(self._lib.lmpc_rollout_set_lap_schedule(self._h, k, s.shape[1], nat.ptr(s)))
        self._lap_schedules[kind] = s

    def lap_schedule_of(self, kind):
        """The installed lap schedule of ``kind`` as [batch, L] int32 (a copy), or None."""
        if kind not in nat.LAP_SCHEDULE_TABLES:
            raise ValueError("kind is one of %s, got %r" % (sorted(nat.LAP_SCHEDULE_TABLES), kind))
        s = self._lap_schedules.get(kind)
        return None if s is None else s.copy()

    def set_regression(self, regs, index=None):
        """Per-controller regression models (a study of the learned model's settings in one batch): controller b identifies its
        local LTV model with ``regs[index[b]]`` (objects with the fields of reference_params.RegressionParams: trToUse up to the
        store's, MaxNumPoint, h, lamb, scaling) in every later ``identify``, ``step`` and ``rollout_step``.  ``index`` is required
        with ``regs``.  ``regs=None`` (no index) returns to the constants the store was created with.  A set with a smaller trToUse
        regresses on the controller's trToUse shortest laps.  Independent of the other tables and of the pool groups (a lap driven
        under another model setting is still a trajectory of this car); allowed in the middle of a run.  Waits for work already
        enqueued."""
        self._install(self._lib.lmpc_set_regression_sets, "regs", regs, index,
                      lambda: nat.make_regression_sets(regs, index, self.B, self.trToUse))

    def set_shapes(self, shapes, index=None):
        """Per-controller horizons and safe-set sizes (the horizon / safe-set trade-off in one batch): controller b plans over
        ``shapes[index[b]] = (N_b, numSS_Points_b)`` in every later ``identify``, ``select``, ``step`` and ``rollout_step``, with
        numSS_Points_b / numSS_it points per lap.  Every pair is one of nat.SHAPE_GRID, at most the controller's own (N,
        numSS_Points) and on the same side of 0.  ``index`` is required with ``shapes``.  ``shapes=None`` (no index) returns every
        controller to the handle's shape.  Only before the first lap is stored and not with warm start; independent of the other
        tables.  While shapes are installed the ``solve*`` entry points on caller arrays are refused.  Device buffers keep the
        handle's (N, numSS_Points) as their stride: ``read_buffer`` and the trace cut a controller's rows to its shape.  Waits for
        work already enqueued."""
        self._install(self._lib.lmpc_set_shapes, "shapes", shapes, index,
                      lambda: nat.make_shape_sets(shapes, index, self.B, self.N, self.M, self.numSS_it, self._ss_laps))
        self._shapes = None if shapes is None else ([tuple(int(v) for v in s) for s in shapes], np.asarray(index).reshape(-1).copy())

    def shape_of(self, inst):
        """(N, numSS_Points) controller ``inst`` plans with: its row of ``set_shapes``, or the handle's."""
        sh = self._shapes
        return (self.N, self.M) if sh is None else sh[0][int(sh[1][int(inst)])]

    def set_ss_laps(self, values, index=None):
        """Per-controller safe-set lap counts (how to split the safe set between laps and points per lap, in one batch):
        controller b draws its safe set from its ``values[index[b]]`` fastest laps, numSS_Points_b / values[index[b]] points per
        lap, in every later ``select``, ``step`` and ``rollout_step`` and in the lap books (host or device), which rank, evict and
        flag as a controller created with that numSS_it and the same ss_cap.  Every value is an integer in 1 .. the handle's
        numSS_it, and every controller's numSS_Points (``shape_of``) must be its value times an even number of points per lap.
        ``index`` is required with ``values``.  ``values=None`` (no index) returns every controller to the handle's numSS_it.
        Only on an LMPC handle and before the first lap is stored; seeding still stores the copies asked for, so a controller
        whose value exceeds them is flagged as the handle would be.  Not part of a snapshot.  Waits for work already enqueued."""
        if values is None:
            points = [self.shape_of(b)[1] for b in range(self.B)]
            if any(not nat._even_split(m, max(self.numSS_it, 1)) for m in points):
                raise ValueError("the installed shapes need their lap counts: the handle's numSS_it does not split them evenly")
        if self._windows is not None:                     # the other install order of set_lap_windows
            for b in range(self.B):
                v = self.numSS_it if values is None else values[int(np.asarray(index).reshape(-1)[b])]
                w = int(self._windows[b, 0])
                if 0 < w < int(v):
                    raise ValueError("controller %d: numSS_it %d exceeds its ss_window (%d)" % (b, int(v), w))
        self._install(self._lib.lmpc_set_ss_laps, "values", values, index,
                      lambda: nat.make_ss_laps_sets(values, index, self.B, self.numSS_it, [self.shape_of(b)[1] for b in range(self.B)]))
        if values is None:
            self._ss_laps = None
        else:
            rows = [int(v) for v in values]
            self._ss_laps = np.array([rows[int(i)] for i in np.asarray(index).reshape(-1)], np.int32)

    def ss_laps_of(self, inst):
        """numSS_it of controller ``inst``: its value of ``set_ss_laps``, or the handle's."""
        return self.numSS_it if self._ss_laps is None else int(self._ss_laps[int(inst)])

    def set_lap_windows(self, windows, index=None):
        """Per-controller lap windows (a controller that trusts only its recent laps, e.g. after its car or the track changed):
        controller b's safe set selects its ``ss_laps_of(b)`` fastest laps among its ``windows[index[b]].ss_window`` most recent
        ones, and its learned model regresses on the trToUse shortest of the last ``model_window`` laps it filed (objects with
        those two fields, e.g. reference_params.LapWindowParams; 0 = unbounded, the reference's rule).  The lap books (host or
        device) then store only the laps that can still be selected under the window, so ss_window <= ss_cap and model_window <=
        model_cap never overflow them.  ss_window is 0 or ``ss_laps_of(b)`` .. ss_cap (0 on an MPC handle), model_window 0 or
        trToUse .. model_cap.  ``index`` is required with ``windows``.  ``windows=None`` (no index) removes the table.  Only before
        the first lap is stored; not part of a snapshot (a record resumes exactly under the same windows).  ValueError before any
        native call where the library would refuse a value.  Waits for work already enqueued."""
        self._install(self._lib.lmpc_set_lap_windows, "windows", windows, index,
                      lambda: nat.make_lap_window_sets(windows, index, self.B, [self.ss_laps_of(b) for b in range(self.B)],
                                                       max(self.ss_cap, 1), self.trToUse, self.model_cap, self.lmpc))
        if windows is None:
            self._windows = None
        else:
            rows = [(int(w.ss_window), int(w.model_window)) for w in windows]
            self._windows = np.array([rows[int(i)] for i in np.asarray(index).reshape(-1)], np.int32).reshape(self.B, 2)

    def lap_windows_of(self, inst):
        """(ss_window, model_window) of controller ``inst`` under ``set_lap_windows``, (0, 0) (unbounded) without a table."""
        return (0, 0) if self._windows is None else (int(self._windows[int(inst), 0]), int(self._windows[int(inst), 1]))

    def set_lane_rules(self, rules, index=None):
        """Per-controller lane rules (lane-safe safe sets): controller b with ``rules[index[b]].mode == 1`` judges every lap it
        files -- its own laps, the seeded record and every import, against its own QP's lane rows Fx x <= bx -- and ranks a lap
        whose rows leave a lane row by more than ``lane_tol`` (or hold a non-finite entry) behind every lap that kept to it; mode 0
        is the reference's rule (objects with ``mode`` and ``lane_tol``, e.g. reference_params.LaneRuleParams).  Such a lap is
        filed with the safe-set key lap time + LANE_UNSAFE_KEY (``_native.split_lane_key`` splits ``books()["ss_time"]``); the
        learned model and the lap history keep raw lengths.  ``index`` is required with ``rules``.  ``rules=None`` (no index)
        removes the table.  Only on an LMPC handle and before the first lap is stored; under a mode 1 row the host-slot hand-over
        and seeding are refused (use the device books).  Not part of a snapshot (a record resumes exactly under the same rules).
        ValueError before any native call where the library would refuse a value.  Waits for work already enqueued."""
        self._install(self._lib.lmpc_set_lane_rules, "rules", rules, index,
                      lambda: nat.make_lane_rule_sets(rules, index, self.B, self.lmpc, getattr(self, "Tcl", 0)))
        if rules is None:
            self._lane = None
        else:
            rows = [(int(r.mode), float(r.lane_tol)) for r in rules]
            self._lane = [rows[int(i)] for i in np.asarray(index).reshape(-1)]

    def lane_rules_of(self, inst):
        """(mode, lane_tol) of controller ``inst`` under ``set_lane_rules``, (0, 0.0) (the reference's rule) without a table."""
        return (0, 0.0) if self._lane is None else self._lane[int(inst)]

    def _no_lane_rule(self, what):
        """The host-slot paths keep the caller's books, which do not judge laps: refused while a mode 1 lane rule is installed."""
        if self._lane is not None and any(m == 1 for m, _ in self._lane):
            raise ValueError("%s: a lane rule is installed; lane rules need the device books (the *_dev methods)" % what)

    def set_tracks(self, tracks, index=None):
        """Per-controller tracks (several circuits in one batch): controller b drives ``tracks[index[b]]`` (objects with
        ``seg_table`` and ``TrackLength``, e.g. reference_params.TrackParams) in every later regression, safe-set selection,
        addPoint, lap cost, lap hand-over and simulator step.  ``index`` is required with ``tracks``.  ``tracks=None`` (no index)
        returns to the track the controller was created with.  Independent of ``set_param_sets`` and ``set_vehicles``.
        Only before the first lap is stored; while more than one track is installed the pooled exchange is refused.
        Waits for work already enqueued."""
        self._install(self._lib.lmpc_set_tracks, "tracks", tracks, index, lambda: nat.make_track_sets(tracks, index, self.B))

    def set_pool_groups(self, index=None, ngroups=None):
        """Pool groups of the pooled exchange (fleet learning per design cell): controller b exchanges laps only with the
        controllers of group ``index[b]`` in ``[0, ngroups)`` (None: ``max(index) + 1``; e.g. sharding.design_groups).  Group
        numbers are global: every rank installs the same numbering.  ``index=None`` returns to one pool.  With several tracks
        installed every group must drive one circuit, or the exchange is refused.  Allowed after laps are stored; waits for work
        already enqueued."""
        if index is None:
            if ngroups not in (None, 0):
                raise ValueError("index=None returns to one pool and takes no ngroups")
            ngroups = 0
        elif ngroups is None:
            ngroups = int(np.max(index)) + 1
        idx = nat.make_pool_groups(index, ngroups, self.B)
        nat.check(self._lib.lmpc_set_pool_groups(self._h, int(ngroups), nat.ptr(idx)))
        self._pool_groups = int(ngroups) or 1

    def set_pool_min_overrun(self, rows):
        """Ship a latest own lap in ``pool_export`` only once it has ``rows`` rows past its finish line (0, the default: any).
        An importer's safe-set window near the finish reaches into those rows."""
        nat.check(self._lib.lmpc_set_pool_min_overrun(self._h, int(rows)))

    @property
    def pool_groups(self):
        """G, the number of pool groups of the exchange (1 without groups): pool_export writes G * kbest rows."""
        return self._pool_groups

    # ------------------------------------------------------------------ PredictiveModel.addTrajectory
    def model_add_trajectory(self, inst, x, u):
        """PredictiveModel.py:35-46: keep laps sorted by length; only the trToUse fastest are ever read."""
        x = np.ascontiguousarray(x, float); u = np.ascontiguousarray(u, float)
        slot = self._model_slot_for(inst, x.shape[0])
        if slot >= 0:
            nat.check(self._lib.lmpc_model_put_lap(self._h, inst, slot, x.shape[0], nat.ptr(x), nat.ptr(u)))
        self._touch(inst, used=True)     # usedIt is pushed once, before the next kernel that reads it

    def _model_slot_for(self, inst, T):
        """Ordering rule of PredictiveModel.py:35-46 for a new lap of T rows; returns the device slot or -1 when the lap
        can never be among the trToUse fastest (it is then not stored on the device)."""
        laps = self.model_laps[inst]
        lapno = self.model_count[inst]
        self.model_count[inst] += 1
        if not laps or T >= laps[-1][0]:
            pos = len(laps)
        else:
            pos = next(i for i, (t, _) in enumerate(laps) if T < t)
        laps.insert(pos, (T, lapno))
        W = self.lap_windows_of(inst)[1]
        if W > 0:                                                               # the new lap is always stored
            book = self.model_book[inst]
            if len(book.slot_of) >= self.model_cap:
                keep = self._window_keep([t for (t, _) in sorted(laps, key=lambda e: e[1])], self.trToUse, W)
                victims = [ln for (_, ln) in laps if ln in book.slot_of and ln not in keep]
                stored = [ln for (_, ln) in laps if ln in book.slot_of]
                book.drop(victims[-1] if victims else stored[-1])             # the slowest that can no longer be used
            return book.take(lapno)
        if pos < self.trToUse or len(laps) <= self.trToUse:
            if len(self.model_book[inst].slot_of) >= self.model_cap:          # evict the slowest stored lap not in usedIt
                stored = [ln for (_, ln) in laps if ln in self.model_book[inst].slot_of and ln != lapno]
                keep = {ln for (_, ln) in laps[:self.trToUse]}
                victims = [ln for ln in stored if ln not in keep]
                self.model_book[inst].drop(victims[-1] if victims else stored[-1])
            return self.model_book[inst].take(lapno)
        return -1

    @staticmethod
    def _window_keep(times, n, W, start=0):
        """Numbers of the laps ``times`` (indexed by lap or arrival number) that can still be among the ``n`` first under a window
        of the W most recent: those in the window with fewer than n newer laps strictly faster (a newer lap of equal time sorts
        after).  ``start``: laps before it are no longer stored and are not counted."""
        m = len(times)
        return {j for j in range(max(m - W, start), m) if sum(1 for i in range(j + 1, m) if times[i] < times[j]) < n}

    def _touch(self, inst, sel=False, used=False):
        """Mark one instance's selection / usedIt rows as stale (rebuilt at the next _flush)."""
        if sel:
            self._sel_dirty = True
            if self._sel_rows is not None:
                self._sel_rows.add(int(inst))
        if used:
            self._used_dirty = True
            if self._used_rows is not None:
                self._used_rows.add(int(inst))

    def _push_used(self, inst=None):
        self._used_dirty = False
        rows = range(self.B) if self._used_rows is None else self._used_rows
        used = self._used
        for b in rows:
            laps = self.model_laps[b]
            W = self.lap_windows_of(b)[1]
            if W > 0:                                     # usedIt among the last W arrivals
                laps = [e for e in laps if e[1] >= self.model_count[b] - W]
            for c in range(self.trToUse):
                if c < len(laps) and laps[c][1] in self.model_book[b].slot_of:
                    used[b, c] = self.model_book[b].slot_of[laps[c][1]]
                elif laps:
                    used[b, c] = self.model_book[b].slot_of.get(laps[min(c, len(laps) - 1)][1], 0)
        self._used_rows = set()
        nat.check(self._lib.lmpc_model_set_used(self._h, nat.ptr(used)))

    # ------------------------------------------------------------------ LMPC.addTrajectory / addPoint
    def add_trajectory(self, inst, x, u, qfun=None, lap_time=None):
        """PC.py:418-445 for one instance (Qfun = computeCost on the device unless given).
        ``qfun``/``lap_time`` exist so that a stored controller state (laps already grown by addPoint) can be
        restored verbatim."""
        x = np.ascontiguousarray(x, float); u = np.ascontiguousarray(u, float)
        lapno = self.it[inst]
        slot = self._ss_slot_for(inst, int(x.shape[0] if lap_time is None else lap_time))
        q = None if qfun is None else np.ascontiguousarray(qfun, float)
        nat.check(self._lib.lmpc_ss_put_lap(self._h, inst, slot, x.shape[0], nat.ptr(x), nat.ptr(u), nat.ptr(q)))
        first = (lapno == 0)
        self.it[inst] += 1
        self._touch(inst, sel=True)
        return first, slot

    def _ss_slot_for(self, inst, lap_time):
        """LMPC.addTrajectory bookkeeping (PC.py:425-428): new lap number = it; keep the controller's numSS_it fastest + lap it-1."""
        lapno = self.it[inst]
        self.LapTime[inst].append(int(lap_time))
        self.own_laps[inst].append(lapno)
        book = self.ss_book[inst]
        W = self.lap_windows_of(inst)[0]
        if W > 0 and not book.free:                       # evict the slowest, then oldest, lap that can no longer be selected
            times = self.LapTime[inst]
            keep = self._window_keep(times, self.ss_laps_of(inst), W)
            victims = [ln for ln in book.slot_of if ln not in keep]
            if not victims:
                raise RuntimeError("safe-set pool too small")
            book.drop(max(victims, key=lambda ln: (times[ln], -ln)))
        elif not book.free:
            order = list(np.argsort(np.array(self.LapTime[inst]), kind="stable"))
            keep = set(order[:self.ss_laps_of(inst)]) | {lapno}
            victims = [ln for ln in book.slot_of if ln not in keep]
            if not victims:
                raise RuntimeError("safe-set pool too small")
            book.drop(max(victims, key=lambda ln: self.LapTime[inst][ln]))
        return book.take(lapno)

    def _flush(self):
        """Push pending lap bookkeeping (usedIt, the numSS_it fastest laps) to the device before a kernel reads it."""
        if self.device_books:
            return                       # the device keeps the books itself
        if self._used_dirty:
            self._push_used()
        if self.lmpc and self._sel_dirty:
            self._push_selection()

    def _push_selection(self):
        sel, isp, prev = self._sel, self._isp, self._prev
        rows = range(self.B) if self._sel_rows is None else self._sel_rows
        for b in rows:
            if not self.LapTime[b]:
                continue
            nit = max(self.ss_laps_of(b), 1)
            if len(self.LapTime[b]) < nit:
                # the reference indexes sortedLapTime[0:numSS_it] lap by lap and raises IndexError here (PC.py:402-403)
                raise IndexError("instance %d has %d stored laps, fewer than numSS_it = %d" % (b, len(self.LapTime[b]), nit))
            W = self.lap_windows_of(b)[0]
            lo = max(len(self.LapTime[b]) - W, 0) if W > 0 else 0                 # the window: lap numbers [it - W, it)
            order = lo + np.argsort(np.array(self.LapTime[b][lo:]), kind="stable")[:nit]     # PC.py:395,402
            for c, jj in enumerate(order):
                sel[b, c] = self.ss_book[b].slot_of[int(jj)]
                isp[b, c] = 0 if int(jj) < self.it[b] - 1 else 1                    # PC.py:506
            sel[b, nit:] = sel[b, nit - 1]                                          # entries K2 does not read, as the device books
            isp[b, nit:] = 0
            prev[b] = self.ss_book[b].slot_of.get(self.it[b] - 1, -1)
        self._sel_rows = set()
        nat.check(self._lib.lmpc_ss_set_selection(self._h, nat.ptr(sel), nat.ptr(isp), nat.ptr(prev)))
        self._sel_dirty = False

    def add_point(self, x, u):
        """PC.py:466-476 for all instances: x[B,6], u[B,2]."""
        self._flush()
        x = np.ascontiguousarray(np.asarray(x, float).reshape(self.B, 6))
        u = np.ascontiguousarray(np.asarray(u, float).reshape(self.B, 2))
        nat.check(self._lib.lmpc_ss_add_point(self._h, nat.ptr(x), nat.ptr(u)))

    def get_lap(self, inst, lapno):
        slot = self.ss_book[inst].slot_of[lapno]
        T = C.c_int(0)
        x, u, q = np.zeros((self.Tmax, 6)), np.zeros((self.Tmax, 2)), np.zeros(self.Tmax)
        nat.check(self._lib.lmpc_ss_get_lap(self._h, inst, slot, C.byref(T), nat.ptr(x), nat.ptr(u), nat.ptr(q)))
        return x[:T.value].copy(), u[:T.value].copy(), q[:T.value].copy()

    def patch_row(self, inst, lapno, row, x6, model_lapno=None):
        ms = -1 if model_lapno is None else self.model_book[inst].slot_of.get(model_lapno, -1)
        x6 = np.ascontiguousarray(x6, float)
        nat.check(self._lib.lmpc_ss_patch_row(self._h, inst, self.ss_book[inst].slot_of[lapno], int(row), nat.ptr(x6), ms))

    # ------------------------------------------------------------------ state
    def set_state(self, xLin=None, uLin=None, zt=None, OldInput=None, timeStep=None, has_pred=None, xPred=None):
        B, N = self.B, self.N
        f = lambda a, shp: None if a is None else np.ascontiguousarray(np.asarray(a, float).reshape(shp))
        g = lambda a: None if a is None else np.ascontiguousarray(np.asarray(a).reshape(B), dtype=np.int32)
        args = [f(xLin, (B, N + 1, 6)), f(uLin, (B, N, 2)), f(zt, (B, 6)), f(OldInput, (B, 2)), g(timeStep), g(has_pred),
                f(xPred, (B, N + 1, 6))]
        nat.check(self._lib.lmpc_state_set(self._h, *[nat.ptr(a) for a in args]))

    def get_state(self):
        B, N = self.B, self.N
        o = dict(xLin=np.zeros((B, N + 1, 6)), uLin=np.zeros((B, N, 2)), zt=np.zeros((B, 6)), OldInput=np.zeros((B, 2)),
                 timeStep=np.zeros(B, np.int32))
        nat.check(self._lib.lmpc_state_get(self._h, nat.ptr(o["xLin"]), nat.ptr(o["uLin"]), nat.ptr(o["zt"]),
                                           nat.ptr(o["OldInput"]), nat.ptr(o["timeStep"])))
        return o

    # ------------------------------------------------------------------ kernels
    def identify(self):
        """K1 only: MPC.computeLTVdynamics (PC.py:140-145).  Returns abc[B,N,54], flags[B]."""
        self._flush()
        abc = np.zeros((self.B, self.N, 54)); flags = np.zeros(self.B, np.int32)
        nat.check(self._lib.lmpc_identify_host(self._h, nat.ptr(abc), nat.ptr(flags)))
        return abc, flags

    def select(self, x0):
        """K2 only: LMPC.addTerminalComponents (PC.py:386-416)."""
        self._flush()
        B, M = self.B, self.M
        x0 = np.ascontiguousarray(np.asarray(x0, float).reshape(B, 6))
        o = dict(SS_sel=np.zeros((B, 6, M)), Qfun_sel=np.zeros((B, M)), Succ_SS=np.zeros((B, 6, M)),
                 Succ_uSS=np.zeros((B, 2, M)), min_index=np.zeros((B, self.numSS_it), np.int32), flags=np.zeros(B, np.int32))
        nat.check(self._lib.lmpc_select_host(self._h, nat.ptr(x0), nat.ptr(o["SS_sel"]), nat.ptr(o["Qfun_sel"]),
                                             nat.ptr(o["Succ_SS"]), nat.ptr(o["Succ_uSS"]), nat.ptr(o["min_index"]), nat.ptr(o["flags"])))
        return o

    def alloc_step_outputs(self):
        B, N, M = self.B, self.N, max(self.M, 1)
        return dict(xPred=np.zeros((B, N + 1, 6)), uPred=np.zeros((B, N, 2)), lambd=np.zeros((B, M)), zt=np.zeros((B, 6)),
                    zt_u=np.zeros((B, 2)), SS_sel=np.zeros((B, 6, M)), status=np.zeros(B, np.int32),
                    iters=np.zeros(B, np.int32), resid=np.zeros((B, 3)), flags=np.zeros(B, np.int32))

    def step(self, x0, out=None, want_ss=True):
        """One MPC.solve / LMPC.solve for every instance (PC.py:110-137)."""
        self._flush()
        x0 = np.ascontiguousarray(np.asarray(x0, float).reshape(self.B, 6))
        o = out if out is not None else self.alloc_step_outputs()
        nat.check(self._lib.lmpc_step_host(self._h, 1 if self.lmpc else 0, nat.ptr(x0), nat.ptr(o["xPred"]), nat.ptr(o["uPred"]),
                                           nat.ptr(o["lambd"]), nat.ptr(o["zt"]), nat.ptr(o["zt_u"]),
                                           nat.ptr(o["SS_sel"]) if want_ss else None, nat.ptr(o["status"]), nat.ptr(o["iters"]),
                                           nat.ptr(o["resid"]), nat.ptr(o["flags"])))
        return o

    def step_dev(self, x0_dev):
        self._flush()
        nat.check(self._lib.lmpc_step_dev(self._h, 1 if self.lmpc else 0, nat.ptr(x0_dev)))

    def step_profile(self, x0_dev):
        """One step with CUDA events between its kernels: milliseconds of (K1, K2, QP, shift)."""
        self._flush()
        ms = np.zeros(4, np.float32)
        nat.check(self._lib.lmpc_step_profile(self._h, 1 if self.lmpc else 0, nat.ptr(x0_dev), nat.ptr(ms)))
        return [float(v) for v in ms]

    def read_buffer(self, name, inst, shape, dtype=np.float64):
        """Inspection: the slice of instance `inst` of a per-instance device buffer ("abc", "SS_sel", "Qfun_sel", ...), ``shape``
        being the handle's per-controller shape of it.  A shaped controller (``set_shapes``) gets its valid part: xPred cut to
        N_b + 1 rows and SS_sel / Succ_SS / Succ_uSS / Qfun_sel / lambd to M_b columns."""
        out = np.zeros(shape, dtype)
        nat.check(self._lib.lmpc_read_buffer(self._h, name.encode(), int(inst) * out.nbytes, nat.ptr(out), out.nbytes))
        return self._cut_to_shape(name, inst, out)

    def _cut_to_shape(self, name, inst, a):
        """The valid part of one controller's slice ``a`` of buffer ``name`` (the handle's shape) under its own shape."""
        Nb, Mb = self.shape_of(inst)
        if (Nb, Mb) == (self.N, self.M):
            return a
        if name == "xPred" and a.shape[0] == self.N + 1:
            return a[:Nb + 1].copy()
        if name in ("SS_sel", "Succ_SS", "Succ_uSS") and a.ndim == 2 and a.shape[1] == self.M:
            return a.reshape(-1)[:a.shape[0] * Mb].reshape(a.shape[0], Mb).copy()
        if name in ("Qfun_sel", "lambd") and a.shape[0] == self.M:
            return a[:Mb].copy()
        return a

    def step_results(self):
        """status, iters, resid[B,3], flags of the most recent step_dev / rollout_step."""
        o = dict(status=np.zeros(self.B, np.int32), iters=np.zeros(self.B, np.int32), resid=np.zeros((self.B, 3)),
                 flags=np.zeros(self.B, np.int32))
        nat.check(self._lib.lmpc_step_results(self._h, nat.ptr(o["status"]), nat.ptr(o["iters"]), nat.ptr(o["resid"]), nat.ptr(o["flags"])))
        return o

    # ------------------------------------------------------------------ device-resident closed loop
    def enable_rollout(self, Tcl=512):
        if int(Tcl) >= nat.LANE_UNSAFE_KEY and self._lane is not None and any(m == 1 for m, _ in self._lane):
            raise ValueError("enable_rollout: a lane rule is installed: Tcl must stay below LANE_UNSAFE_KEY")
        nat.check(self._lib.lmpc_rollout_create(self._h, int(Tcl)))
        self.Tcl = int(Tcl)

    def rollout_set_state(self, x, xglob):
        x = np.ascontiguousarray(np.asarray(x, float).reshape(self.B, 6))
        g = np.ascontiguousarray(np.asarray(xglob, float).reshape(self.B, 6))
        nat.check(self._lib.lmpc_rollout_set_state(self._h, nat.ptr(x), nat.ptr(g)))

    def rollout_state(self):
        o = dict(x=np.zeros((self.B, 6)), xglob=np.zeros((self.B, 6)), done=np.zeros(self.B, np.int32), cl_len=np.zeros(self.B, np.int32))
        nat.check(self._lib.lmpc_rollout_get_state(self._h, nat.ptr(o["x"]), nat.ptr(o["xglob"]), nat.ptr(o["done"]), nat.ptr(o["cl_len"])))
        return o

    def rollout_step(self, z=None, seed=0, mode=None):
        """Simulator.sim loop body (SysModel.py:34-48) for every instance on the device.  z[B,3]: standard-normal draws for
        the process noise (reference order vx, vy, wz); None = Philox on the device.  mode: 0 LTV-MPC, 1 LMPC (defaults by
        how the controller was built), 2 LTI-MPC with the model of ``rollout_sysid``."""
        self._flush()
        zz = None if z is None else np.ascontiguousarray(np.asarray(z, float).reshape(self.B, 3))
        m = (1 if self.lmpc else 0) if mode is None else int(mode)
        nat.check(self._lib.lmpc_rollout_step(self._h, m, nat.ptr(zz), int(seed)))

    def rollout_pid_step(self, vt, z_pid=None, z_sim=None, seed=0):
        """One closed-loop step under the PID path follower (Utilities.py:42-68) for every instance: main.py:65-66's seeding lap
        is 1000 of these.  z_pid[B,2], z_sim[B,3]: the reference's standard-normal draws (None = Philox)."""
        zp = None if z_pid is None else np.ascontiguousarray(np.asarray(z_pid, float).reshape(self.B, 2))
        zs = None if z_sim is None else np.ascontiguousarray(np.asarray(z_sim, float).reshape(self.B, 3))
        nat.check(self._lib.lmpc_rollout_pid_step(self._h, float(vt), nat.ptr(zp), nat.ptr(zs), int(seed)))

    def rollout_sysid(self, lamb=1e-7):
        """Regression(x, u, lamb) (Utilities.py:5-28) of every instance's record.  Returns A[B,6,6], B[B,6,2], flags[B]; the model
        also stays on the device for ``rollout_step(mode=2)``."""
        abc = np.zeros((self.B, 54)); flags = np.zeros(self.B, np.int32)
        nat.check(self._lib.lmpc_rollout_sysid(self._h, float(lamb), nat.ptr(abc), nat.ptr(flags)))
        return abc[:, 0:36].reshape(self.B, 6, 6).copy(), abc[:, 36:48].reshape(self.B, 6, 2).copy(), flags

    def rollout_seed_from_record(self, cl_len, copies=4):
        """main.py:99-110 on the device: the record every instance just drove (cl_len[b] rows, e.g. its PID lap) becomes
        ``copies`` identical laps of the safe set and of the regression model, and the controller state is initialised from it."""
        self._no_lane_rule("rollout_seed_from_record")
        ss0 = m0 = None
        for b in range(self.B):
            T = int(cl_len[b])
            for c in range(copies):
                ms = self._model_slot_for(b, T)
                sl = self._ss_slot_for(b, T) if self.lmpc else -1
                if self.lmpc:
                    self.it[b] += 1
                if c == 0:
                    if ss0 is None:
                        ss0, m0 = sl, ms
                    if (sl, ms) != (ss0, m0):
                        raise RuntimeError("seeding needs the same free slots on every instance (fresh controller)")
                elif (sl, ms) != (ss0 + c, m0 + c):
                    raise RuntimeError("seeding needs consecutive free slots (fresh controller)")
        nat.check(self._lib.lmpc_rollout_seed_from_record(self._h, int(copies), int(max(ss0, 0)), int(m0)))
        self._sel_dirty = self._used_dirty = True
        self._sel_rows = self._used_rows = None          # every instance changed

    def rollout_done(self):
        d = np.zeros(self.B, np.int32); n = np.zeros(self.B, np.int32)
        nat.check(self._lib.lmpc_rollout_get_state(self._h, None, None, nat.ptr(d), nat.ptr(n)))
        return d, n

    def rollout_health(self):
        """(OR of the step flags, number of steps whose QP was not reported solved) per instance since enable_rollout."""
        f = np.zeros(self.B, np.int32); n = np.zeros(self.B, np.int32)
        nat.check(self._lib.lmpc_rollout_get_health(self._h, nat.ptr(f), nat.ptr(n)))
        return f, n

    def enable_lap_reports(self, max_laps):
        """Per-lap reports (lmpc_rollout_enable_lap_reports): from now on every controller files one report per lap it drives and
        hands over, up to ``max_laps`` rows (1 .. 1024; 0 turns reports off).  Needs ``enable_rollout`` and an empty closed-loop
        record (before the PID lap, or right after a hand-over or seeding).  ValueError before any native call on a bad capacity."""
        L = nat.check_lap_reports(max_laps)
        if not hasattr(self, "Tcl"):
            raise ValueError("enable_lap_reports needs enable_rollout first")
        nat.check(self._lib.lmpc_rollout_enable_lap_reports(self._h, L))
        self.lap_report_cap = L

    def lap_reports(self):
        """{"n": int32 [B] laps filed (may exceed the capacity L), field: [B, L] for every lmpc_lap_report field} with the rows
        at or beyond min(n, L) zeroed.  ValueError without reports."""
        L = getattr(self, "lap_report_cap", 0)
        if not L:
            raise ValueError("lap reports are not enabled (enable_lap_reports)")
        rows = np.zeros((self.B, L), nat.LAP_REPORT_DTYPE)
        n = np.zeros(self.B, np.int32)
        nat.check(self._lib.lmpc_rollout_get_lap_reports(self._h, nat.ptr(rows), nat.ptr(n)))
        used = np.arange(L)[None, :] < np.minimum(n, L)[:, None]
        out = {"n": n}
        for f in nat.LAP_REPORT_FIELDS:
            out[f] = np.where(used, rows[f], 0).astype(rows[f].dtype)
        return out

    def rollout_get_lap(self, inst):
        T = C.c_int(0)
        x, u = np.zeros((self.Tcl, 6)), np.zeros((self.Tcl, 2))
        nat.check(self._lib.lmpc_rollout_get_lap(self._h, int(inst), C.byref(T), nat.ptr(x), nat.ptr(u)))
        return x[:T.value].copy(), u[:T.value].copy()

    def rollout_finish_laps(self, done, cl_len, to_model=True):
        """main.py:113-119 for every instance whose lap just ended: lmpc.addTrajectory + predictiveModel.addTrajectory of the
        lap recorded on the device (no host copy of the lap), then the next lap starts from xF (SysModel.py:50)."""
        self._no_lane_rule("rollout_finish_laps")
        if self._margins is not None and any(int(r.mode) == 2 for r in self._margins[0]):
            raise ValueError("rollout_finish_laps: adaptive lane margins need the device hand-over (rollout_commit_laps_dev)")
        finished = np.nonzero(done)[0]
        if not len(finished):
            return finished
        fin = np.zeros(self.B, np.int32); ss_slots = np.full(self.B, -1, np.int32); m_slots = np.full(self.B, -1, np.int32)
        for b in finished:
            T = int(cl_len[b])
            fin[b] = 1
            ss_slots[b] = self._ss_slot_for(b, T) if self.lmpc else -1
            m_slots[b] = self._model_slot_for(b, T) if to_model else -1
            if self.lmpc:
                self.it[b] += 1
        nat.check(self._lib.lmpc_rollout_commit_laps(self._h, nat.ptr(fin), nat.ptr(ss_slots), nat.ptr(m_slots)))
        for b in finished:
            self._touch(b, sel=self.lmpc, used=to_model)
        return finished

    # ------------------------------------------------------------------ pooled-safe-set exchange (SURVEY §8e)
    def own_lap_number(self, inst, j):
        """Current lap number of the j-th lap the instance drove itself (imported laps shift later numbers)."""
        return self.own_laps[inst][j]

    def export_laps(self, lapnos, Tpad, rows_dev, lens_dev):
        """Pack stored lap ``lapnos[b]`` (-1 or not stored: none) of every instance into caller-owned device tensors
        rows[B,Tpad,9] = (x | u | Qfun), lens[B] (int32): the send buffer of the per-lap all-gather."""
        slots = np.full(self.B, -1, np.int32)
        for b in range(self.B):
            slots[b] = self.ss_book[b].slot_of.get(int(lapnos[b]), -1)
        nat.check(self._lib.lmpc_ss_export_laps_dev(self._h, nat.ptr(slots), int(Tpad), nat.ptr(rows_dev), nat.ptr(lens_dev)))

    def import_laps(self, src, lap_times, Tpad, rows_dev, lens_dev, to_model=True):
        """Give instance b the gathered lap ``src[b]`` (index into rows[n_src,Tpad,9]; -1: nothing) as a lap driven BEFORE its
        own most recent one: LMPC.addTrajectory + PredictiveModel.addTrajectory (main.py:117-119) of a lap another controller
        drove.  The lap keeps its own Qfun and lap time ``lap_times[b]``; the instance's latest lap stays lap it-1 (the one
        LMPC.addPoint extends, PC.py:466-476).  An instance for which the lap would not be among its numSS_it fastest leaves it out
        of the safe set, but its regression model still takes it (main.py:117-119 adds every lap to both; with trToUse > numSS_it
        it can be among the trToUse shortest).  Returns the instances whose safe set took a lap."""
        src = np.asarray(src, np.int32).reshape(self.B)
        n_src = int(lens_dev.shape[0])
        ss_slots = np.full(self.B, -1, np.int32); m_slots = np.full(self.B, -1, np.int32); use = np.full(self.B, -1, np.int32)
        for b in range(self.B):
            if src[b] < 0 or self.it[b] < 1:
                continue
            lt, last = int(lap_times[b]), self.it[b] - 1
            times = self.LapTime[b][:last] + [lt] + self.LapTime[b][last:]
            W = self.lap_windows_of(b)[0]
            if W > 0:                                     # the laps that can still be selected under the window
                order = self._window_keep(times, self.ss_laps_of(b), W)
            else:
                order = list(np.argsort(np.array(times), kind="stable"))[:self.ss_laps_of(b)]
            if last not in order:                         # never selected (PC.py:395) -> not in the safe set
                if to_model:
                    m_slots[b] = self._model_slot_for(b, lt)
                    use[b] = src[b]
                continue
            book = self.ss_book[b]
            self.LapTime[b] = times
            if last in book.slot_of:                      # own latest lap moves up one lap number
                book.slot_of[last + 1] = book.slot_of.pop(last)
            if self.own_laps[b] and self.own_laps[b][-1] == last:
                self.own_laps[b][-1] = last + 1
            if not book.free:
                keep = set(order) | {last, last + 1}
                victims = [ln for ln in book.slot_of if ln not in keep]
                if not victims:
                    raise RuntimeError("safe-set pool too small")
                book.drop(max(victims, key=(lambda ln: (times[ln], -ln)) if W > 0 else (lambda ln: times[ln])))
            ss_slots[b] = book.take(last)
            self.it[b] += 1
            use[b] = src[b]
            if to_model:
                m_slots[b] = self._model_slot_for(b, lt)
        given = np.nonzero(use >= 0)[0]
        if len(given):
            nat.check(self._lib.lmpc_ss_import_laps_dev(self._h, nat.ptr(ss_slots), nat.ptr(m_slots) if to_model else None,
                                                        nat.ptr(use), n_src, int(Tpad), nat.ptr(rows_dev), nat.ptr(lens_dev)))
            for b in given:
                self._touch(b, sel=bool(ss_slots[b] >= 0), used=to_model)
        return np.nonzero(ss_slots >= 0)[0]

    # ------------------------------------------------------------------ lap books on the device (csrc/lapbooks.cuh)
    def enable_device_books(self):
        """Hand the once-per-lap bookkeeping (which laps are the fastest / usedIt / lap it-1) over to the device, starting from
        the current host books.  From here on use the *_dev methods; the host-side lists are no longer updated (``books()``
        reads the device tables back)."""
        B, sc, mc = self.B, max(self.ss_cap, 1), self.model_cap
        ss_time = np.full((B, sc), 0x7fffffff, np.int32); ss_lap = -np.ones((B, sc), np.int32)
        md_time = np.full((B, mc), 0x7fffffff, np.int32); md_seq = -np.ones((B, mc), np.int32)
        for b in range(B):
            for lapno, slot in self.ss_book[b].slot_of.items():
                ss_time[b, slot], ss_lap[b, slot] = self.LapTime[b][lapno], lapno
            for T, lapno in self.model_laps[b]:
                slot = self.model_book[b].slot_of.get(lapno)
                if slot is not None:
                    md_time[b, slot], md_seq[b, slot] = T, lapno
        it = np.asarray(self.it, np.int32); cnt = np.asarray(self.model_count, np.int32)
        self._flush()
        nat.check(self._lib.lmpc_books_set(self._h, nat.ptr(ss_time), nat.ptr(ss_lap), nat.ptr(it), nat.ptr(md_time), nat.ptr(md_seq),
                                           nat.ptr(cnt)))
        self.device_books = True

    def books(self):
        """The device lap books and the selection derived from them (host copies)."""
        B, sc, mc, nit, tr = self.B, max(self.ss_cap, 1), self.model_cap, max(self.numSS_it, 1), self.trToUse
        o = dict(ss_time=np.zeros((B, sc), np.int32), ss_lap=np.zeros((B, sc), np.int32), it=np.zeros(B, np.int32),
                 md_time=np.zeros((B, mc), np.int32), md_seq=np.zeros((B, mc), np.int32), md_cnt=np.zeros(B, np.int32),
                 sel=np.zeros((B, nit), np.int32), is_prev=np.zeros((B, nit), np.int32), prev_slot=np.zeros(B, np.int32),
                 used=np.zeros((B, tr), np.int32), lap_hist=np.zeros((B, 16), np.int32), lap_n=np.zeros(B, np.int32))
        nat.check(self._lib.lmpc_books_get(self._h, *[nat.ptr(o[k]) for k in ("ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt", "sel",
                                                                               "is_prev", "prev_slot", "used", "lap_hist", "lap_n")]))
        return o

    def rollout_seed_from_record_dev(self, copies=4):
        """main.py:99-110 entirely on the device (books included); see ``rollout_seed_from_record`` for the host-book variant."""
        nat.check(self._lib.lmpc_rollout_seed_from_record_dev(self._h, int(copies)))
        self.device_books = True
        self._sel_dirty = self._used_dirty = False

    def rollout_commit_laps_dev(self):
        """main.py:113-119 for every controller whose lap just ended; nothing crosses to the host."""
        nat.check(self._lib.lmpc_rollout_commit_laps_dev(self._h))

    def rollout_stats(self):
        """(min laps driven, max laps driven, min steps into the current lap among the controllers at the minimum, flagged)."""
        o = np.zeros(4, np.int32)
        nat.check(self._lib.lmpc_rollout_stats(self._h, nat.ptr(o)))
        return tuple(int(v) for v in o)

    def rollout_group_stats(self):
        """``rollout_stats`` per pool group: int32 [G, 4], G = ``pool_groups``.  A group without a controller here reports
        (INT32_MAX, 0, INT32_MAX, 0)."""
        o = np.zeros((self._pool_groups, 4), np.int32)
        nat.check(self._lib.lmpc_rollout_group_stats(self._h, nat.ptr(o)))
        return o

    def pool_export(self, kbest, Tpad, gid_base, rows_dev, meta_dev, groups=None):
        """Send side of the pooled exchange: per pool group, this rank's ``kbest`` fastest latest-own laps (with at least
        ``set_pool_min_overrun`` rows past the finish line) -> rows[G*kbest,Tpad,9], meta[G*kbest,4] = (rows, lap time, global id
        or -1, group), group-major; G = ``pool_groups``.  ``groups``: None (every group ships), or a length-G bool / 0-1 array;
        a group with False ships rows with global id -1, so ``pool_import`` files nothing of it.  Every rank passes the same mask."""
        if groups is None:
            nat.check(self._lib.lmpc_pool_export_dev(self._h, int(kbest), int(Tpad), int(gid_base), nat.ptr(rows_dev), nat.ptr(meta_dev)))
            return
        mask = np.asarray(groups).reshape(-1)
        if mask.shape[0] != self._pool_groups:
            raise ValueError("pool_export: groups needs one entry per pool group (%d), got %d" % (self._pool_groups, mask.shape[0]))
        if not np.all((mask == 0) | (mask == 1)):
            raise ValueError("pool_export: groups entries must be 0 or 1 (or bool)")
        mask = np.ascontiguousarray(mask, np.int32)
        nat.check(self._lib.lmpc_pool_export_groups_dev(self._h, int(kbest), int(Tpad), int(gid_base), nat.ptr(mask), nat.ptr(rows_dev),
                                                        nat.ptr(meta_dev)))

    def pool_import(self, n_src, share, Tpad, gid_base, rows_dev, meta_dev, count=False):
        """Receive side: every controller files the ``share`` fastest gathered laps of its own pool group that it does not own.
        ``n_src`` rows of rows/meta, world * G * kbest after an all-gather of ``pool_export``'s buffers (at most 64 * G)."""
        took = np.zeros(1, np.int32) if count else None
        nat.check(self._lib.lmpc_pool_import_dev(self._h, int(n_src), int(share), int(Tpad), int(gid_base), nat.ptr(rows_dev),
                                                 nat.ptr(meta_dev), nat.ptr(took)))
        return int(took[0]) if count else None

    # ------------------------------------------------------------------ controller snapshots (csrc/snapshot.cuh)
    def _snapshot_ready(self, restoring=False):
        """Snapshots read and write the device lap books.  Host book mirrors would go stale, so a controller that keeps them
        raises ValueError; one that has stored no lap yet may restore (and keeps device books from then on)."""
        if self.device_books or (restoring and not any(self.it) and not any(self.model_count)):
            return
        raise ValueError("snapshots need device lap books (rollout_seed_from_record_dev or enable_device_books): this controller "
                         "keeps host book mirrors, which a restore would leave stale")

    @property
    def snapshot_bytes(self):
        """Bytes of one controller's snapshot record (a multiple of 16)."""
        n = C.c_size_t(0)
        nat.check(self._lib.lmpc_snapshot_bytes(self._h, C.byref(n)))
        return int(n.value)

    def snapshot_layout(self):
        """The layout a record of this controller has (the keys of nat.SNAPSHOT_LAYOUT and "bytes", "lap_reports" = the report
        capacity when reports are on, and "lane_margin" = 1 under a lane-margin table)."""
        return dict(N=self.N, M=self.M, ncx=int(self._p.ncx), ncu=int(self._p.ncu), numSS_it=max(self.numSS_it, 1),
                    trToUse=self.trToUse, ss_cap=max(self.ss_cap, 1), model_cap=self.model_cap, Tmax=self.Tmax,
                    Tcl=int(getattr(self, "Tcl", 0)), warm_start=int(self._p.warm_start), bytes=self.snapshot_bytes,
                    **({"lap_reports": self.lap_report_cap} if getattr(self, "lap_report_cap", 0) else {}),
                    **({"lane_margin": 1} if self._margins is not None else {}))

    def _ext_stream(self, torch):
        return torch.cuda.ExternalStream(self.stream, device=torch.device("cuda", self.device))

    @property
    def device(self):
        return int(self._device)

    def snapshot(self, inst=None, out=None):
        """Records of controllers ``inst`` (None: every controller, in order; repeats allowed) as a uint8 CUDA tensor
        [n, snapshot_bytes] on this controller's device (``out``: a tensor of that shape to write into).  What a controller learned
        and where it is: lap pools, lap books, controller state, warm-start record, closed loop, health.  Not what it is told to
        drive (parameter sets, vehicles, tracks, pool groups).  Ordered after the work enqueued so far and before later work on the
        current torch stream."""
        import torch
        self._snapshot_ready()
        idx = nat.snapshot_indices(inst, self.B, "inst")
        n = self.B if idx is None else int(idx.size)
        nbytes = self.snapshot_bytes
        dev = torch.device("cuda", self.device)
        if out is None:
            out = torch.empty((n, nbytes), dtype=torch.uint8, device=dev)
        nat.check_snapshot_tensor(out, self.device, nbytes, rows=n, what="out")
        ext, cur = self._ext_stream(torch), torch.cuda.current_stream(dev)
        ext.wait_stream(cur)                               # the buffer may still be in use by work of the current stream
        nat.check(self._lib.lmpc_snapshot_pack_dev(self._h, n, nat.ptr(idx), nat.ptr(out)))
        cur.wait_stream(ext)                               # later work on the current stream (reuse of the buffer included) follows
        return out

    def restore(self, records, inst=None, rec_of=None):
        """Controller ``inst[i]`` (None: 0 .. n-1) takes record ``rec_of[i]`` (None: i) of ``records`` (uint8 CUDA tensor
        [nrec, snapshot_bytes] on this device, e.g. from ``snapshot`` of a controller with the same layout, or torch.load).  One
        record may go to many controllers.  The record's track must be the destination controller's; its car and tuning are
        whatever this controller has installed.  Raises ValueError on a repeated or out-of-range destination, a bad tensor or a
        layout mismatch (named) before any device work; the library then checks every record used and refuses (NativeError,
        nothing restored) unless all pass."""
        import torch
        dst, rec = self._check_restore(records, inst, rec_of)
        dev = torch.device("cuda", self.device)
        ext, cur = self._ext_stream(torch), torch.cuda.current_stream(dev)
        ext.wait_stream(cur)                               # records written on the current stream are complete
        nat.check(self._lib.lmpc_snapshot_unpack_dev(self._h, nat.ptr(records), int(records.shape[0]), int(dst.size), nat.ptr(dst),
                                                     nat.ptr(rec)))
        cur.wait_stream(ext)
        if not self.device_books:                          # a fresh controller: the restored books live on the device
            self.device_books = True
            self._sel_dirty = self._used_dirty = False

    def _check_restore(self, records, inst, rec_of):
        """The pure-Python checks of ``restore``: books, tensor, indices, and the header of every record used against this
        layout.  Returns (destinations, record of each destination) as int32 arrays."""
        import torch
        self._snapshot_ready(restoring=True)
        mine = self.snapshot_layout()
        nat.check_snapshot_tensor(records, self.device, mine["bytes"])
        nrec = int(records.shape[0])
        dst = nat.snapshot_indices(inst, self.B, "inst", unique=True)
        if dst is None:
            dst = np.arange(min(self.B, nrec) if rec_of is None else self.B, dtype=np.int32)
        rec = nat.snapshot_record_map(rec_of, int(dst.size), nrec)
        used = np.unique(rec)
        hsz = C.sizeof(nat.SnapshotHeader)
        heads = records[:, :hsz].index_select(0, torch.from_numpy(used.astype(np.int64)).to(records.device)).cpu().numpy()
        words = np.ascontiguousarray(heads[:, :64]).view(np.int32)     # magic, version, bytes, the layout ints, warm_mode, nsect
        want = np.array([nat.SNAPSHOT_MAGIC, nat.SNAPSHOT_VERSION, mine["bytes"]] + [mine[f] for f in nat.SNAPSHOT_LAYOUT], np.int64)
        bad = np.any(words[:, :14].astype(np.int64) & 0xFFFFFFFF != want & 0xFFFFFFFF, axis=1)
        rep = C.sizeof(nat.LapReport) * mine.get("lap_reports", 0)     # bytes of the report rows section (slot of "lap_reports")
        k = nat.SNAPSHOT_SECTIONS_NAMES.index("lap_reports")
        sect_bytes = np.ascontiguousarray(heads[:, 64 + 4 * nat.SNAPSHOT_SECTIONS:64 + 8 * nat.SNAPSHOT_SECTIONS]).view(np.int32)
        bad = np.nonzero(bad | (sect_bytes[:, k] != rep))[0]
        if bad.size:
            r = int(used[bad[0]])
            msg = nat.snapshot_layout_mismatch(nat.decode_snapshot_header(heads[bad[0]]), mine)
            raise ValueError("record %d: %s" % (r, msg or "header does not match this controller"))
        return dst, rec

    def clone(self, src, dst):
        """Controller ``dst[i]`` becomes a copy of controller ``src[i]`` (or of the single ``src`` for every ``dst``): packed into
        a temporary buffer first, so overlapping ``src`` / ``dst`` are safe (a permutation works)."""
        dst_i = nat.snapshot_indices(dst, self.B, "dst", unique=True)
        if dst_i is None:
            raise ValueError("dst: the controllers to overwrite are required")
        src_i = nat.snapshot_indices(src, self.B, "src")
        if src_i is None:
            raise ValueError("src: the controllers to copy are required")
        if src_i.size == 1 and dst_i.size > 1:
            rec_of = np.zeros(dst_i.size, np.int32)
        elif src_i.size == dst_i.size:
            rec_of = None
        else:
            raise ValueError("clone: one src, or one src per dst (%d), got %d" % (dst_i.size, src_i.size))
        self._snapshot_ready()
        recs = self.snapshot(src_i)
        self.restore(recs, dst_i, rec_of)

    @property
    def rollout_clock(self):
        """The simulator's step counter: the Philox noise of a step is keyed by (seed, stream, this counter), the stream being
        the controller's index unless ``set_noise_streams`` says otherwise."""
        v = C.c_ulonglong(0)
        nat.check(self._lib.lmpc_rollout_get_clock(self._h, C.byref(v)))
        return int(v.value)

    @rollout_clock.setter
    def rollout_clock(self, step):
        if int(step) < 0:
            raise ValueError("the rollout clock counts steps: >= 0")
        nat.check(self._lib.lmpc_rollout_set_clock(self._h, int(step)))

    def device_buffer(self, name):
        return int(self._lib.lmpc_device_buffer(self._h, name.encode()) or 0)

    def sync(self):
        nat.check(self._lib.lmpc_sync(self._h))

    @property
    def stream(self):
        return int(self._lib.lmpc_stream(self._h) or 0)
