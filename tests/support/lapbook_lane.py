"""The lap lists of lapbook_window.WindowBooks under a per-controller lane rule (lmpc_set_lane_rules), for tests.

``LaneBooks(..., lane_mode=1, lane_tol=tol, Fx=Fx, bx=bx)`` judges every lap it files and ranks a lap by (unsafe, lap time): an
unsafe lap's safe-set key is its lap time + LANE_UNSAFE_KEY, which is what the device stores in ss_time.  Everything that ranks,
evicts or selects compares keys, so the lists of WindowBooks need no other change.  The model list and the lap history keep raw
lengths.  With lane_mode 0 every key is the lap time and the books are WindowBooks exactly.

Judged rows: an own lap's rows 0 .. Trec-1 (the record), an import's shipped rows 0 .. min(lt, rows, Tpad)-1 against the
importer's own Fx, bx and lane_tol."""
import numpy as np

from lapbook_window import WindowBooks
from plant_exact import compute_cost

LANE_UNSAFE_KEY = 1 << 24


def lane_unsafe(rows, Fx, bx, tol):
    """The device's judgement of the rows x[T, 6] (or more columns; the state is the first 6): True when an entry is not finite or
    for a lane row i, d_i = (Fx[i][0] x0 + Fx[i][1] x1 + ... + Fx[i][5] x5, separate fp64 multiplies and adds in this order) - bx[i]
    is > tol."""
    x = np.asarray(rows, np.float64)[:, :6]
    if x.size == 0:
        return False
    if not np.isfinite(x).all():
        return True
    Fx, bx = np.asarray(Fx, np.float64), np.asarray(bx, np.float64).reshape(-1)
    for i in range(Fx.shape[0]):
        s = Fx[i, 0] * x[:, 0]
        for j in range(1, 6):
            s = s + Fx[i, j] * x[:, j]
        if ((s - bx[i]) > tol).any():
            return True
    return False


def lane_key(T, unsafe):
    return T + LANE_UNSAFE_KEY if unsafe else T


class LaneBooks(WindowBooks):
    def __init__(self, numSS_it, ss_cap, trToUse, model_cap, Tmax, TrackLength=1.0, ss_window=0, md_window=0, lane_mode=0,
                 lane_tol=0.0, Fx=None, bx=None):
        super().__init__(numSS_it, ss_cap, trToUse, model_cap, Tmax, TrackLength, ss_window, md_window)
        self.lane_mode, self.lane_tol, self.Fx, self.bx = lane_mode, lane_tol, Fx, bx
        self.unsafe_hist = []          # the verdict of every own lap, in order

    def judge(self, rows):
        return self.lane_mode == 1 and rows is not None and lane_unsafe(rows, self.Fx, self.bx, self.lane_tol)

    def own(self, Trec, x=None, u=None, unsafe=None):
        """An own lap of Trec rows (x, u: its record, or None); ``unsafe`` overrides the judgement of x[:Trec]."""
        if unsafe is None:
            unsafe = self.judge(None if x is None else x[:Trec])
        self._prev_before = self.it - 1
        n = min(Trec, self.Tmax)
        ss = md = None
        if x is not None:
            ss = (x[:n], u[:n], compute_cost(x[:n, 4], self.TrackLength))
            md = (x[:n], u[:n])
        self.times.append(lane_key(Trec, unsafe))
        self.ss_rows.append(ss)
        self._after_ss_event(self.it - 1)
        self._md_add(Trec, md)
        self.lap_hist.append(Trec)
        self.unsafe_hist.append(bool(unsafe))

    def imp(self, lt, length=None, R=None, Tpad=None, unsafe=None):
        """An import with lap time lt and ``length`` shipped rows R[Tpad, 9] (or None); ``unsafe`` overrides the judgement of
        R[:min(lt, length, Tpad)].  Returns "none", "dropped" or "filed" as Books.imp."""
        if self.it < 1:
            return "none"
        if unsafe is None:
            unsafe = self.judge(None if R is None else R[:max(min(lt, length, Tpad), 0)])
        self._prev_before = self.it - 1
        ss = md = None
        if R is not None:
            n = min(length, Tpad, self.Tmax)
            ss = (R[:n, 0:6], R[:n, 6:8], R[:n, 8])
            m = min(lt, length, Tpad, self.Tmax)
            md = (R[:m, 0:6], R[:m, 6:8])
        pos = self.it - 1                                   # filed before the own latest lap
        times = self.times[:pos] + [lane_key(lt, unsafe)] + self.times[pos:]
        live = self._live(times) if self.ss_window else self._argsort(times)[:self.numSS_it]
        if pos not in live:
            self._md_add(lt, md)
            return "dropped"
        self.times = times
        self.ss_rows.insert(pos, ss)
        self._after_ss_event(self.it - 2, own_latest=self.it - 1)
        self._md_add(lt, md)
        return "filed"

    def unsafe(self):
        """The verdict of every safe-set lap, by lap number."""
        return [t >= LANE_UNSAFE_KEY for t in self.times]
