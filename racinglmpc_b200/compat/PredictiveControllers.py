"""Drop-in for src/fnc/controller/PredictiveControllers.py: same module name, same ``MPCParams`` / ``MPC`` /
``LMPC`` constructors, methods (solve, addTrajectory, addPoint) and result attributes, backed by
liblmpc_b200.so through racinglmpc_b200.controller (one instance of the batched engine).

Reference call sites this satisfies: Simulator.sim (SysModel.py:34-38: ``solve(x)``, ``uPred[0,:]``,
``addPoint(x,u)``), main.py:76-120 (parameter assignment, ``addTrajectory``, ``Qfun[it][0]``) and plot.py
(``SS, uSS, SS_glob, Qfun, LapTime, it, N, numSS_Points, xStoredPredTraj, SSStoredPredTraj``).
There is no CPU fallback: without the CUDA library / an H100 the constructors raise.
"""
import datetime
import os
import sys
from dataclasses import dataclass, field

import numpy as np

_PKG_PARENT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if _PKG_PARENT not in sys.path:
    sys.path.insert(0, _PKG_PARENT)

from racinglmpc_b200.batched import BatchedFTOCP, pack_abc           # noqa: E402
from racinglmpc_b200.controller import BatchedController             # noqa: E402


@dataclass
class PythonMsg:
    def __setattr__(self, key, value):
        if not hasattr(self, key):
            raise TypeError('Cannot add new field "%s" to frozen class %s' % (key, self))
        else:
            object.__setattr__(self, key, value)


@dataclass
class MPCParams(PythonMsg):
    # same fields as PredictiveControllers.py:24-51 (the ndarray default of `Q` there is not importable on
    # Python >= 3.11; None is used instead and every caller passes Q explicitly)
    n: int = field(default=None)
    d: int = field(default=None)
    N: int = field(default=None)
    A: np.array = field(default=None)
    B: np.array = field(default=None)
    Q: np.array = field(default=None)
    R: np.array = field(default=None)
    Qf: np.array = field(default=None)
    dR: np.array = field(default=None)
    Qslack: float = field(default=None)
    Fx: np.array = field(default=None)
    bx: np.array = field(default=None)
    Fu: np.array = field(default=None)
    bu: np.array = field(default=None)
    xRef: np.array = field(default=None)
    slacks: bool = field(default=True)
    timeVarying: bool = field(default=False)

    def __post_init__(self):
        if self.Qf is None: self.Qf = np.zeros((self.n, self.n))
        if self.dR is None: self.dR = np.zeros(self.d)
        if self.xRef is None: self.xRef = np.zeros(self.n)


def _zero_dt():
    t = datetime.datetime.now()
    return t - t


class MPC():
    """Model Predictive Controller (reference: PredictiveControllers.py:56-283)."""

    def __init__(self, mpcParameters, predictiveModel=[], device=0):
        p = mpcParameters
        self.N, self.n, self.d = p.N, p.n, p.d
        self.Qslack, self.Q, self.Qf, self.R, self.dR = p.Qslack, p.Q, p.Qf, p.R, p.dR
        self.A, self.B = p.A, p.B
        self.Fx, self.Fu, self.bx, self.bu, self.xRef = p.Fx, p.Fu, p.bx, p.bu, p.xRef
        self.slacks, self.timeVarying = p.slacks, p.timeVarying
        self.predictiveModel = predictiveModel
        self._params = p
        self._device = device
        self._engine = None
        self._model_seen = 0
        self._lmpc = False
        if self.timeVarying == True:
            self.xLin = self.predictiveModel.xStored[-1][0:self.N + 1, :]     # PC.py:89
            self.uLin = self.predictiveModel.uStored[-1][0:self.N, :]         # PC.py:90
        self.OldInput = np.zeros((1, 2))
        self.xPred = []
        self.uPred = None
        self.solverTime = _zero_dt()
        self.linearizationTime = _zero_dt()
        self.timeStep = 0
        self.feasible = 1
        self._state_dirty = True
        self._make_engine()

    # ------------------------------------------------------------------ engine plumbing
    def _make_engine(self):
        p = self._params
        if not self.timeVarying:
            self._engine = BatchedFTOCP(p, batch=1, device=self._device)
            self._abc = pack_abc(np.asarray(self.A, float), np.asarray(self.B, float))       # one LTI stage record
            return
        pm = self.predictiveModel
        self._engine = BatchedController(
            p, 1, pm.seg_table(), pm.map.TrackLength, trToUse=len(pm.usedIt),
            numSS_Points=getattr(self, "numSS_Points", 0), numSS_it=getattr(self, "numSS_it", 0),
            QterminalSlack=getattr(self, "QterminalSlack", None), device=self._device,
            model_kwargs=dict(MaxNumPoint=pm.MaxNumPoint, h=float(pm.h), lamb=float(pm.lamb), dt=float(pm.dt),
                              scaling=tuple(np.diag(pm.scaling))))
        self._out = self._engine.alloc_step_outputs()

    def _sync_model(self):
        pm = self.predictiveModel
        while self._model_seen < len(pm._added):
            x, u = pm._added[self._model_seen]
            self._engine.model_add_trajectory(0, x, u)
            self._model_seen += 1

    def _push_state(self):
        zt = getattr(self, "zt", np.zeros(6))
        self._engine.set_state(xLin=np.asarray(self.xLin, float), uLin=np.asarray(self.uLin, float), zt=np.asarray(zt, float),
                               OldInput=np.asarray(self.OldInput, float).ravel(), timeStep=[self.timeStep],
                               has_pred=[0 if isinstance(self.xPred, list) else 1],
                               xPred=None if isinstance(self.xPred, list) else self.xPred)
        self._state_dirty = False

    # ------------------------------------------------------------------ reference API
    def solve(self, x0):
        """Computes control action (PC.py:110-137)."""
        x0 = np.asarray(x0, dtype=float)
        startTimer = datetime.datetime.now()
        if not self.timeVarying:
            # LTI: the reference builds q once in __init__ (OldInput = 0) and never refreshes it (PC.py:116-119)
            o = self._engine.solve(x0.reshape(1, 6), np.zeros((1, 2)), self._abc)
            self.xPred, self.uPred = o["xPred"][0].copy(), o["uPred"][0].copy()
            self.feasible = 1 if o["status"][0] == 1 else 0
        else:
            self._sync_model()
            if self._state_dirty:
                self._push_state()      # before _pre_solve: the regression of this step reads the UNmodified xLin
            self._pre_solve(x0)         # (PC.py:117 runs before PC.py:121/394)
            o = self._engine.step(x0.reshape(1, 6), out=self._out)
            self.xPred, self.uPred = o["xPred"][0].copy(), o["uPred"][0].copy()
            self.feasible = 1 if (o["status"][0] == 1 and o["flags"][0] == 0) else 0
            self._post_solve(o)
        self.solverTime = datetime.datetime.now() - startTimer
        self.feasibleStateInput()
        if self.timeVarying == True:
            self.xLin = np.vstack((self.xPred[1:, :], self.zt))
            self.uLin = np.vstack((self.uPred[1:, :], self.zt_u))
        self.OldInput = self.uPred[0, :]
        self.timeStep += 1

    def _pre_solve(self, x0):
        pass

    def _post_solve(self, o):
        pass

    def feasibleStateInput(self):
        self.zt = self.xPred[-1, :]
        self.zt_u = self.uPred[-1, :]


class LMPC(MPC):
    """Learning MPC (reference: PredictiveControllers.py:286-514)."""

    def __init__(self, numSS_Points, numSS_it, QterminalSlack, mpcPrameters, predictiveModel, dt=0.1, device=0):
        self.numSS_Points = numSS_Points
        self.numSS_it = numSS_it
        self.QterminalSlack = QterminalSlack
        super().__init__(mpcPrameters, predictiveModel, device=device)
        self._lmpc = True
        self.OldInput = np.zeros((1, 2))
        self.xPred = []
        self.LapTime = []
        self.SS = []
        self.uSS = []
        self.Qfun = []
        self.SS_glob = []
        self.xStoredPredTraj = []
        self.xStoredPredTraj_it = []
        self.uStoredPredTraj = []
        self.uStoredPredTraj_it = []
        self.SSStoredPredTraj = []
        self.SSStoredPredTraj_it = []
        self.zt = np.array([0.0, 0.0, 0.0, 0.0, 10.0, 0.0])
        self.it = 0
        self._grow = None

    # ------------------------------------------------------------------ lap bookkeeping (host mirrors for main.py / plot.py)
    def addTrajectory(self, x, u, x_glob):
        """LMPC.addTrajectory (PC.py:418-445): the lap goes to the device store (which computes its own cost-to-go); the
        host lists the reference exposes (SS, uSS, SS_glob, Qfun, LapTime, *StoredPredTraj) are mirrors for main.py:120,127
        and plot.py."""
        lap = self.it
        for store, item in ((self.LapTime, x.shape[0]), (self.SS, x), (self.uSS, u), (self.SS_glob, x_glob),
                            (self.Qfun, self.computeCost(x, u))):
            store.append(item)
        self._grow = None                                   # addPoint now extends this lap
        self._engine.add_trajectory(0, x, u)
        if lap == 0:                                        # PC.py:431-433: views of the stored lap, as in the reference
            self.xLin, self.uLin = x[1:self.N + 2, :], u[1:self.N + 1, :]
        for hist, cur in (("xStoredPredTraj", "xStoredPredTraj_it"), ("uStoredPredTraj", "uStoredPredTraj_it"),
                          ("SSStoredPredTraj", "SSStoredPredTraj_it")):
            getattr(self, hist).append(getattr(self, cur))
            setattr(self, cur, [])
        self.it, self.timeStep = lap + 1, 0
        self._state_dirty = True

    def computeCost(self, x, u):
        """LMPC.computeCost (PC.py:447-464): steps until the finish line, counted backwards from the end of the lap and reset
        to 0 on every row at/after the line.  Closed form: Q[j] = r(j) - j with r(j) the first row >= j that is the last row
        or has s >= TrackLength -- the same rule the device uses (csrc/safeset.cuh lap_cost_block)."""
        s = np.asarray(x)[:, 4]
        T = s.shape[0]
        rows = np.arange(T)
        stop = ~(s < self.predictiveModel.map.TrackLength)
        stop[-1] = True
        nxt = np.minimum.accumulate(np.where(stop, rows, T)[::-1])[::-1]
        return (nxt - rows).astype(float)

    def addPoint(self, x, u):
        """LMPC.addPoint (PC.py:466-476): the current (x, u), one track length further, extends lap it-1; its cost-to-go keeps
        counting down past the finish line.  The device store appends in place; the host mirrors grow in amortised O(1)
        buffers and SS/uSS/Qfun[it-1] are re-pointed at views of them (the reference re-allocates the whole lap every step)."""
        j = self.it - 1
        g = self._grow
        if g is None or g["lap"] != j:
            n0 = self.SS[j].shape[0]
            cap = max(2 * n0, n0 + 256)
            g = self._grow = dict(lap=j, n=n0, x=np.empty((cap, self.n)), u=np.empty((cap, self.d)), q=np.empty(cap))
            g["x"][:n0], g["u"][:n0], g["q"][:n0] = self.SS[j], self.uSS[j], self.Qfun[j]
        n0 = g["n"]
        if n0 == g["q"].shape[0]:
            for k in ("x", "u", "q"):
                g[k] = np.concatenate((g[k], np.empty_like(g[k])), axis=0)
        g["x"][n0] = x
        g["x"][n0, 4] += self.predictiveModel.map.TrackLength
        g["u"][n0] = u
        g["q"][n0] = g["q"][n0 - 1] - 1
        g["n"] = n0 + 1
        self.SS[j], self.uSS[j], self.Qfun[j] = g["x"][:n0 + 1], g["u"][:n0 + 1], g["q"][:n0 + 1]
        self._engine.add_point(np.asarray(x, float), np.asarray(u, float))

    def _pre_solve(self, x0):
        # PC.py:392-394.  The device applies the zt part itself (ss_select_kernel); the xLin write only matters
        # while xLin is still a view of a stored lap (very first solve): mirror it into the device copies.
        L = self.predictiveModel.map.TrackLength
        if (self.zt[4] - x0[4] > L / 2):
            self.zt[4] = np.max([self.zt[4] - L, 0])
            self.xLin[4, -1] = self.xLin[4, -1] - L
            for j, lap in enumerate(self.SS):
                if np.shares_memory(lap, self.xLin) and j in self._engine.ss_book[0].slot_of:
                    self._engine.patch_row(0, j, 1 + 4, lap[1 + 4])
            # (the regression reads only vx,vy,wz of stored laps, so the model store needs no patch)

    def _post_solve(self, o):
        self.lambd = o["lambd"][0].copy()
        self.SS_PointSelectedTot = o["SS_sel"][0].copy()
        self._zt_dev, self._ztu_dev = o["zt"][0].copy(), o["zt_u"][0].copy()
        self.xStoredPredTraj_it.append(self.xPred)
        self.uStoredPredTraj_it.append(self.uPred)
        self.SSStoredPredTraj_it.append(self.SS_PointSelectedTot.T)

    # PC.py:382-384 (computed by the kernel epilogue: Succ_SS lam, Succ_uSS lam)
    def feasibleStateInput(self):
        self.zt = self._zt_dev
        self.zt_u = self._ztu_dev
