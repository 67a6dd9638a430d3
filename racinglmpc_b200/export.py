"""Presentation support for device-resident batches (SURVEY §8f rank 4): the data the reference's plot.py reads.

plot.py (src/fnc/plot.py:51-56,106-175) draws from attributes of one LMPC object -- SS, uSS, SS_glob, LapTime, it, N,
numSS_Points, xStoredPredTraj[it][i] ((N+1) x 6) and SSStoredPredTraj[it][i] (numSS_Points x 6) -- and from
Map.getGlobalPosition (Track.py:135-189).  A batched rollout keeps none of that on the host; ``RolloutTrace`` records it on the
device for a few chosen controllers and ``plot_view`` re-shapes one controller's trace into an object with exactly those
attributes, so that plot.py's functions can be pointed at it unchanged.
"""
import ctypes as C
from types import SimpleNamespace

import numpy as np

from . import _native as nat


def global_position(table6, track_length, s, ey, device=0):
    """Map.getGlobalPosition for arrays of points, on the device.  Returns xy[n,2], ok[n]."""
    table6 = np.ascontiguousarray(table6, float)
    s = np.ascontiguousarray(np.atleast_1d(s), float); ey = np.ascontiguousarray(np.atleast_1d(ey), float)
    xy = np.zeros((s.shape[0], 2)); ok = np.zeros(s.shape[0], np.int32)
    nat.check(nat.lib().lmpc_track_global_position(int(device), nat.ptr(table6), table6.shape[0], float(track_length), s.shape[0],
                                                   nat.ptr(s), nat.ptr(ey), nat.ptr(xy), nat.ptr(ok)))
    return xy, ok


class RolloutTrace:
    """Per-step record of chosen controllers of a BatchedController in rollout mode."""

    def __init__(self, ctrl, instances, cap_steps=1024):
        self.c = ctrl
        self.instances = [int(i) for i in instances]
        self.cap = int(cap_steps)
        inst = np.asarray(self.instances, np.int32)
        nat.check(ctrl._lib.lmpc_rollout_trace_create(ctrl._h, len(self.instances), nat.ptr(inst), self.cap))

    def get(self, tr):
        """Arrays of trace `tr` (index into `instances`): x[T,6], x_glob[T,6], u[T,2], xPred[T,N+1,6], SS_sel[T,6,M], lap[T]; for a
        controller with its own shape (BatchedController.set_shapes) N and M are its N_b and M_b."""
        c, N, M = self.c, self.c.N, max(self.c.M, 1)
        steps = C.c_int(0)
        o = dict(x=np.zeros((self.cap, 6)), x_glob=np.zeros((self.cap, 6)), u=np.zeros((self.cap, 2)), xPred=np.zeros((self.cap, N + 1, 6)),
                 SS_sel=np.zeros((self.cap, 6, M)), lap=np.zeros(self.cap, np.int32))
        nat.check(c._lib.lmpc_rollout_trace_get(c._h, int(tr), C.byref(steps), nat.ptr(o["x"]), nat.ptr(o["x_glob"]), nat.ptr(o["u"]),
                                                nat.ptr(o["xPred"]), nat.ptr(o["SS_sel"]), nat.ptr(o["lap"])))
        out = {k: v[:steps.value].copy() for k, v in o.items()}
        Nb, Mb = c.shape_of(self.instances[tr])
        if (Nb, Mb) != (c.N, c.M):      # the leading N_b + 1 rows and the row-major [6, M_b] block of the handle-sized regions
            out["xPred"] = out["xPred"][:, :Nb + 1].copy()
            out["SS_sel"] = out["SS_sel"].reshape(out["SS_sel"].shape[0], -1)[:, :6 * max(Mb, 1)].reshape(-1, 6, max(Mb, 1)).copy()
        return out

    def plot_view(self, tr, first_lap_number=0):
        """One traced controller as an object with the attributes plot.py reads (laps = the laps completed within the trace;
        lap numbers start at `first_lap_number`, e.g. 4 after main.py's four seed laps)."""
        t = self.get(tr)
        laps = sorted(set(int(l) for l in t["lap"]))
        Nb, Mb = self.c.shape_of(self.instances[tr])
        v = SimpleNamespace(N=Nb, numSS_Points=Mb, SS=[], uSS=[], SS_glob=[], LapTime=[], xStoredPredTraj=[],
                            SSStoredPredTraj=[], it=0)
        for l in laps[:-1] if len(laps) > 1 else laps:          # the last lap of the trace is usually still being driven
            m = t["lap"] == l
            v.SS.append(t["x"][m]); v.uSS.append(t["u"][m]); v.SS_glob.append(t["x_glob"][m]); v.LapTime.append(int(m.sum()))
            v.xStoredPredTraj.append([p for p in t["xPred"][m]])
            v.SSStoredPredTraj.append([s.T for s in t["SS_sel"][m]])             # numSS_Points x 6, as PC.py:379 stores it
        v.it = first_lap_number + len(v.SS)
        return v
