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

    def set_param_sets(self, params, index=None, QterminalSlack=None):
        """Per-controller QP parameters (a parameter sweep in one batch): controller b solves with ``params[index[b]]`` (objects
        with the reference's MPCParams field names; every field but N and the constraint row counts may differ) and, for LMPC,
        ``QterminalSlack[index[b]]`` (None: the handle's).  ``index`` is required with ``params``.  ``params=None`` (no index)
        returns to the parameters the handle was created with.
        Waits for work already enqueued; warm-start records start over."""
        if params is None:
            if index is not None:
                raise ValueError("params=None reverts to the handle's own parameters and takes no index")
            nat.check(self._lib.lmpc_set_param_sets(self._h, None, 0, None))
            return
        sets, idx = nat.make_param_sets(self._p, params, index, self.B, self._p.numSS_Points, self.numSS_it, QterminalSlack)
        nat.check(self._lib.lmpc_set_param_sets(self._h, sets, len(sets), nat.ptr(idx)))

    def set_vehicles(self, vehicles, index=None):
        """Per-controller vehicles of the device simulator (a Monte-Carlo over the plant in one batch): controller b is driven
        with ``vehicles[index[b]]`` (objects with the reference's ten field names, e.g. reference_params.VehicleParams) by every
        later ``rollout_step`` and ``rollout_pid_step``.  ``index`` is required with ``vehicles``.  ``vehicles=None`` (no index)
        returns to the reference vehicle.  Independent of ``set_param_sets``.  Waits for work already enqueued."""
        if vehicles is None:
            if index is not None:
                raise ValueError("vehicles=None reverts to the reference vehicle and takes no index")
            nat.check(self._lib.lmpc_rollout_set_vehicles(self._h, None, 0, None))
            return
        sets, idx = nat.make_vehicle_sets(vehicles, index, self.B)
        nat.check(self._lib.lmpc_rollout_set_vehicles(self._h, sets, len(sets), nat.ptr(idx)))

    def set_tracks(self, tracks, index=None):
        """Per-controller tracks (several circuits in one batch): controller b drives ``tracks[index[b]]`` (objects with
        ``seg_table`` and ``TrackLength``, e.g. reference_params.TrackParams) in every later regression, safe-set selection,
        addPoint, lap cost, lap hand-over and simulator step.  ``index`` is required with ``tracks``.  ``tracks=None`` (no index)
        returns to the track the controller was created with.  Independent of ``set_param_sets`` and ``set_vehicles``.
        Only before the first lap is stored; while more than one track is installed the pooled exchange is refused.
        Waits for work already enqueued."""
        if tracks is None:
            if index is not None:
                raise ValueError("tracks=None reverts to the handle's own track and takes no index")
            nat.check(self._lib.lmpc_set_tracks(self._h, None, 0, None))
            return
        sets, idx = nat.make_track_sets(tracks, index, self.B)
        nat.check(self._lib.lmpc_set_tracks(self._h, sets, len(sets), nat.ptr(idx)))

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
        if pos < self.trToUse or len(laps) <= self.trToUse:
            if len(self.model_book[inst].slot_of) >= self.model_cap:          # evict the slowest stored lap not in usedIt
                stored = [ln for (_, ln) in laps if ln in self.model_book[inst].slot_of and ln != lapno]
                keep = {ln for (_, ln) in laps[:self.trToUse]}
                victims = [ln for ln in stored if ln not in keep]
                self.model_book[inst].drop(victims[-1] if victims else stored[-1])
            return self.model_book[inst].take(lapno)
        return -1

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
        """LMPC.addTrajectory bookkeeping (PC.py:425-428): new lap number = it; keep the numSS_it fastest + lap it-1."""
        lapno = self.it[inst]
        self.LapTime[inst].append(int(lap_time))
        self.own_laps[inst].append(lapno)
        book = self.ss_book[inst]
        if not book.free:
            order = list(np.argsort(np.array(self.LapTime[inst]), kind="stable"))
            keep = set(order[:self.numSS_it]) | {lapno}
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
        nit = max(self.numSS_it, 1)
        sel, isp, prev = self._sel, self._isp, self._prev
        rows = range(self.B) if self._sel_rows is None else self._sel_rows
        for b in rows:
            if not self.LapTime[b]:
                continue
            if len(self.LapTime[b]) < nit:
                # the reference indexes sortedLapTime[0:numSS_it] lap by lap and raises IndexError here (PC.py:402-403)
                raise IndexError("instance %d has %d stored laps, fewer than numSS_it = %d" % (b, len(self.LapTime[b]), nit))
            order = np.argsort(np.array(self.LapTime[b]), kind="stable")[:nit]     # PC.py:395,402
            for c, jj in enumerate(order):
                sel[b, c] = self.ss_book[b].slot_of[int(jj)]
                isp[b, c] = 0 if int(jj) < self.it[b] - 1 else 1                    # PC.py:506
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
        """Inspection: the slice of instance `inst` of a per-instance device buffer ("abc", "SS_sel", "Qfun_sel", ...)."""
        out = np.zeros(shape, dtype)
        nat.check(self._lib.lmpc_read_buffer(self._h, name.encode(), int(inst) * out.nbytes, nat.ptr(out), out.nbytes))
        return out

    def step_results(self):
        """status, iters, resid[B,3], flags of the most recent step_dev / rollout_step."""
        o = dict(status=np.zeros(self.B, np.int32), iters=np.zeros(self.B, np.int32), resid=np.zeros((self.B, 3)),
                 flags=np.zeros(self.B, np.int32))
        nat.check(self._lib.lmpc_step_results(self._h, nat.ptr(o["status"]), nat.ptr(o["iters"]), nat.ptr(o["resid"]), nat.ptr(o["flags"])))
        return o

    # ------------------------------------------------------------------ device-resident closed loop
    def enable_rollout(self, Tcl=512):
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

    def rollout_get_lap(self, inst):
        T = C.c_int(0)
        x, u = np.zeros((self.Tcl, 6)), np.zeros((self.Tcl, 2))
        nat.check(self._lib.lmpc_rollout_get_lap(self._h, int(inst), C.byref(T), nat.ptr(x), nat.ptr(u)))
        return x[:T.value].copy(), u[:T.value].copy()

    def rollout_finish_laps(self, done, cl_len, to_model=True):
        """main.py:113-119 for every instance whose lap just ended: lmpc.addTrajectory + predictiveModel.addTrajectory of the
        lap recorded on the device (no host copy of the lap), then the next lap starts from xF (SysModel.py:50)."""
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

    def rollout_export_laps(self, Tpad, rows_dev, lens_dev):
        """Pack the closed-loop records into caller-owned device tensors rows[B,Tpad,8], lens[B] (int32)."""
        nat.check(self._lib.lmpc_rollout_export_laps_dev(self._h, int(Tpad), nat.ptr(rows_dev), nat.ptr(lens_dev)))

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
        LMPC.addPoint extends, PC.py:466-476).  An instance for which the lap would not be among its numSS_it fastest is
        skipped.  Returns the instances that took a lap."""
        src = np.asarray(src, np.int32).reshape(self.B)
        n_src = int(lens_dev.shape[0])
        ss_slots = np.full(self.B, -1, np.int32); m_slots = np.full(self.B, -1, np.int32); use = np.full(self.B, -1, np.int32)
        for b in range(self.B):
            if src[b] < 0 or self.it[b] < 1:
                continue
            lt, last = int(lap_times[b]), self.it[b] - 1
            times = self.LapTime[b][:last] + [lt] + self.LapTime[b][last:]
            order = list(np.argsort(np.array(times), kind="stable"))[:self.numSS_it]
            if last not in order:
                continue                                  # never selected (PC.py:395) -> not stored
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
                book.drop(max(victims, key=lambda ln: times[ln]))
            ss_slots[b] = book.take(last)
            self.it[b] += 1
            use[b] = src[b]
            if to_model:
                m_slots[b] = self._model_slot_for(b, lt)
        took = np.nonzero(use >= 0)[0]
        if len(took):
            nat.check(self._lib.lmpc_ss_import_laps_dev(self._h, nat.ptr(ss_slots), nat.ptr(m_slots) if to_model else None,
                                                        nat.ptr(use), n_src, int(Tpad), nat.ptr(rows_dev), nat.ptr(lens_dev)))
            for b in took:
                self._touch(b, sel=True, used=to_model)
        return took

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

    def pool_export(self, kbest, Tpad, gid_base, rows_dev, meta_dev):
        """Send side of the pooled exchange: this rank's ``kbest`` fastest latest-own laps -> rows[kbest,Tpad,9], meta[kbest,4]."""
        nat.check(self._lib.lmpc_pool_export_dev(self._h, int(kbest), int(Tpad), int(gid_base), nat.ptr(rows_dev), nat.ptr(meta_dev)))

    def pool_import(self, n_src, share, Tpad, gid_base, rows_dev, meta_dev, count=False):
        """Receive side: every controller files the ``share`` globally fastest gathered laps it does not own."""
        took = np.zeros(1, np.int32) if count else None
        nat.check(self._lib.lmpc_pool_import_dev(self._h, int(n_src), int(share), int(Tpad), int(gid_base), nat.ptr(rows_dev),
                                                 nat.ptr(meta_dev), nat.ptr(took)))
        return int(took[0]) if count else None

    def device_buffer(self, name):
        return int(self._lib.lmpc_device_buffer(self._h, name.encode()) or 0)

    def sync(self):
        nat.check(self._lib.lmpc_sync(self._h))

    @property
    def stream(self):
        return int(self._lib.lmpc_stream(self._h) or 0)
