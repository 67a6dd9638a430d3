"""The per-lap report rule of the device closed loop (lmpc_rollout_enable_lap_reports, DESIGN.md "Per-lap reports") restated on the
host, one controller step at a time.

A caller feeds every step a controller drives (``step``), every lap hand-over (``file``) and every seeding (``restart``), and
``table`` returns what BatchedController.lap_reports returns.  A retired controller drives no step, so the caller feeds nothing for
it.  The lane rows are evaluated as the device does: d_i = (Fx[i][0] x[0] + Fx[i][1] x[1] + ... + Fx[i][5] x[5]) - bx[i], summed in
that order in float64 without fused multiply-adds (Python floats), a row is violated when d_i > 0, and viol_max takes np.fmax.
"""
import numpy as np

FIELDS = ("steps", "flags", "unsolved", "viol_steps", "ipm_iters", "ipm_iters_max", "viol_max")


def empty_row():
    return dict(steps=0, flags=0, unsolved=0, viol_steps=0, ipm_iters=0, ipm_iters_max=0, viol_max=-np.inf)


def lane_margins(Fx, bx, x):
    """d_i of every row i of Fx [ncx, 6], bx [ncx] at state x [6], in the device's operation order."""
    out = []
    for i in range(len(bx)):
        s = float(Fx[i][0]) * float(x[0])
        for j in range(1, 6):
            s = s + float(Fx[i][j]) * float(x[j])
        out.append(s - float(bx[i]))
    return out


class LapReportBook:
    """Report rows [B][L], counts n [B] and the running rows of B controllers."""

    def __init__(self, B, L):
        self.B, self.L = int(B), int(L)
        self.n = np.zeros(self.B, np.int64)
        self.rows = [[None] * self.L for _ in range(self.B)]
        self.run = [empty_row() for _ in range(self.B)]

    def step(self, b, x, Fx, bx, flags, status=None, iters=None):
        """One closed-loop step of controller b driven from plant state x: flags = the step flags | the simulator's bits; status /
        iters of its QP, None for a PID step."""
        r = self.run[b]
        x = [float(v) for v in np.asarray(x, np.float64).reshape(6)]
        if not all(np.isfinite(x)):
            viol = True
            r["viol_max"] = np.inf
        else:
            d = lane_margins(Fx, bx, x)
            viol = any(v > 0.0 for v in d)
            for v in d:
                r["viol_max"] = float(np.fmax(r["viol_max"], v))
        r["steps"] += 1
        r["flags"] |= int(flags)
        r["viol_steps"] += 1 if viol else 0
        if status is not None:
            r["unsolved"] += 1 if int(status) != 1 else 0
            r["ipm_iters"] += int(iters)
            r["ipm_iters_max"] = max(r["ipm_iters_max"], int(iters))

    def file(self, b):
        """A lap hand-over of controller b: the running row becomes report n (stored while n < L), n counts on, the row restarts."""
        n = int(self.n[b])
        if n < self.L:
            self.rows[b][n] = dict(self.run[b])
        self.n[b] = n + 1
        self.run[b] = empty_row()

    def restart(self, b):
        """The seeding of controller b: the record is consumed without a report and the table starts afresh."""
        self.n[b] = 0
        self.rows[b] = [None] * self.L
        self.run[b] = empty_row()

    def table(self):
        """{"n": [B], field: [B, L]} with unused rows zero, the form of BatchedController.lap_reports."""
        out = {"n": self.n.astype(np.int32)}
        for f in FIELDS:
            a = np.zeros((self.B, self.L), np.float64 if f == "viol_max" else np.int32)
            for b in range(self.B):
                for k in range(min(int(self.n[b]), self.L)):
                    a[b, k] = self.rows[b][k][f]
            out[f] = a
        return out


def assert_equal_tables(got, want, what=""):
    """Two report tables agree bit for bit (viol_max compared by its bits, so -inf, +inf and -0.0 count)."""
    assert np.array_equal(got["n"], want["n"]), (what, "n")
    for f in FIELDS:
        g, w = np.asarray(got[f]), np.asarray(want[f])
        if f == "viol_max":
            g, w = g.view(np.int64), w.view(np.int64)
        bad = np.argwhere(g != w)
        assert bad.size == 0, (what, f, bad[:5].tolist(), np.asarray(got[f])[tuple(bad[0])], np.asarray(want[f])[tuple(bad[0])])
