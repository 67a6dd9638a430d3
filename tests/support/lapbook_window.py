"""The unbounded lap lists of lapbook_exact.Books under per-controller lap windows (lmpc_set_lap_windows), for tests.

``WindowBooks(..., ss_window=W, md_window=Wm)`` keeps the lists of ``Books`` and changes only what a window changes; a window of 0
is unbounded and gives ``Books`` exactly.

Safe set: the selection is the stable argsort of the laps numbered [it - W, it), first numSS_it (the reference's order restricted
to the window).  A lap must stay resident while it is in the window and fewer than numSS_it NEWER laps rank ahead of it: older
laps leave the window before it does, newer ones stay as long as it does.  An import is dropped from the safe set when it is not
such a lap on arrival (its only newer lap is the own latest); flag 64 is due when those laps, the new one and for an import the
own latest outnumber ss_cap.

Model: usedIt is the first trToUse laps of the list among arrival numbers [seq - Wm, seq), the slowest repeating when there are
fewer; the slot table must hold every lap in the window with fewer than trToUse newer laps shorter."""
import numpy as np

from lapbook_exact import Books


def window_live(times, W, n):
    """Numbers of the laps `times` (indexed by lap or arrival number) a window of the W most recent keeps among the first n: in the
    window, fewer than n newer laps strictly faster (a newer lap of equal time sorts after)."""
    m = len(times)
    return {j for j in range(max(m - W, 0), m) if sum(1 for i in range(j + 1, m) if times[i] < times[j]) < n}


class WindowBooks(Books):
    def __init__(self, numSS_it, ss_cap, trToUse, model_cap, Tmax, TrackLength=1.0, ss_window=0, md_window=0):
        super().__init__(numSS_it, ss_cap, trToUse, model_cap, Tmax, TrackLength)
        self.ss_window, self.md_window = ss_window, md_window

    def _live(self, times):
        return window_live(times, self.ss_window, self.numSS_it)

    def _after_ss_event(self, new, own_latest=None):
        if not self.ss_window:
            return super()._after_ss_event(new, own_latest)
        resident = self._live(self.times) | {new}
        if own_latest is not None:
            resident.add(own_latest)
        if len(resident) > self.ss_cap:
            self.flag |= 64
            self.dead = True

    def imp(self, lt, length=None, R=None, Tpad=None):
        if not self.ss_window or self.it < 1:
            return super().imp(lt, length, R, Tpad)
        self._prev_before = self.it - 1
        ss = md = None
        if R is not None:
            n = min(length, Tpad, self.Tmax)
            ss = (R[:n, 0:6], R[:n, 6:8], R[:n, 8])
            m = min(lt, length, Tpad, self.Tmax)
            md = (R[:m, 0:6], R[:m, 6:8])
        pos = self.it - 1                                   # filed before the own latest lap, as without a window
        times = self.times[:pos] + [lt] + self.times[pos:]
        if pos not in self._live(times):
            self._md_add(lt, md)
            return "dropped"
        self.times = times
        self.ss_rows.insert(pos, ss)
        self._after_ss_event(self.it - 2, own_latest=self.it - 1)
        self._md_add(lt, md)
        return "filed"

    def sel(self):
        if not self.ss_window:
            return super().sel()
        lo = max(self.it - self.ss_window, 0)
        order = [lo + k for k in np.argsort(np.array(self.times[lo:], dtype=np.int64), kind="stable")][:self.numSS_it]
        if len(order) < self.numSS_it:
            return order + [order[-1]] * (self.numSS_it - len(order)) if order else [], 8
        return order, 0

    def used(self):
        if not self.md_window:
            return super().used()
        u = [s for (_, s, _) in self.md if s >= self.seq - self.md_window][:self.trToUse]
        return u + [u[-1]] * (self.trToUse - len(u)) if u else []

    def resident(self):
        if not self.ss_window:
            return super().resident()
        r = self._live(self.times)
        if self.it >= 1:
            r.add(self.it - 1)
        return r

    def md_resident(self):
        """Arrival numbers the model slot table must hold: usedIt without a window, else every lap in the window with fewer than
        trToUse newer laps shorter."""
        if not self.md_window:
            return set(self.used())
        t = {s: tm for (tm, s, _) in self.md}
        return window_live([t[s] for s in range(self.seq)], self.md_window, self.trToUse)
