"""The reference's per-controller lap bookkeeping as unbounded lists, for tests: no slots, no capacity, no eviction.

LMPC keeps a list of laps (LapTime, SS, uSS, Qfun) and decides from it, once per lap, which stored laps the next lap uses
(PC.py:395-445); PredictiveModel keeps its laps ordered by length (PredictiveModel.py:35-46).  ``Books`` restates both lists for
one controller in this project's words.  The device (csrc/lapbooks.cuh) and the host books (racinglmpc_b200/controller.py)
keep only the laps that can still be read, in fixed-capacity slot tables; the tests compare what those tables select with
what these lists select.

Safe-set list: an own lap is appended as lap number ``it`` with its lap time Trec (the reference's x.shape[0]); the slot
tables store at most Tmax of its rows, which does not change its place in the order.  Selection is the stable argsort of the
lap times, first numSS_it (PC.py:395,402); lap it-1 is the one addPoint extends (PC.py:466-476) and the only one with
is_prev = 1 (PC.py:506).  Fewer than numSS_it laps is flag 8 (the reference raises IndexError); the device then repeats the
slowest lap it has.

Project rules that are not the reference's (the reference has no exchange):
  - an imported lap is filed BEFORE the controller's own latest lap: it takes lap number it-1, the own latest becomes it;
  - an import that would not be among the numSS_it fastest on arrival is dropped from the safe set (it stays unchanged) --
    faster laps only push it further down, so it could never be selected;
  - every import still reaches the model list, as every lap in main.py:117-119 reaches both lists: with trToUse > numSS_it a
    lap the safe set drops can be among the trToUse shortest;
  - an import is ordered by its shipped lap time lt in both lists, as an own lap by Trec: a lap longer than Tmax stays as
    slow as it was, even though only Tmax of its rows (Tpad of an import's) are stored;
  - a controller with no lap of its own (it = 0) takes no import.

Model list: the reference's append-or-insert loop (equal lengths go after the laps already there); usedIt is the first trToUse
laps, identified by arrival number; with fewer laps than trToUse the slowest repeats (the device's stand-in where the
reference would raise).

Flag 64 (safe-set pool too small) is due exactly when the laps that must stay resident -- the numSS_it fastest after the event,
the new lap, and for an import the own latest lap -- outnumber ss_cap.  After it the slot tables no longer follow the lists
(``dead``).

``variant`` selects the known-wrong restatements the tests must reject: "unstable" (ties of the argsort in reverse lap order),
"bisect_left" (a model lap goes before equal lengths), "import_after" (an import numbered after the own latest lap),
"evict_fastest" (a capacity-bound list that evicts its fastest lap), "stale_prev" (the addPoint target not moved by the event).
"""
import numpy as np

from plant_exact import compute_cost

VARIANTS = ("unstable", "bisect_left", "import_after", "evict_fastest", "stale_prev")


class Books:
    def __init__(self, numSS_it, ss_cap, trToUse, model_cap, Tmax, TrackLength=1.0, variant=None):
        assert variant is None or variant in VARIANTS
        self.numSS_it, self.ss_cap, self.trToUse, self.model_cap, self.Tmax = numSS_it, ss_cap, trToUse, model_cap, Tmax
        self.TrackLength = TrackLength
        self.variant = variant
        self.times = []        # LapTime, index = lap number
        self.ss_rows = []      # (x, u, q) of each safe-set lap, or None
        self.md = []           # [(time, arrival, (x, u) or None)] in PredictiveModel order
        self.seq = 0           # model laps filed so far (md_cnt)
        self.lap_hist = []     # Trec of every own lap
        self.flag = 0          # OR of the hand-over flags (8, 64)
        self.dead = False
        self.gone = set()      # "evict_fastest" only
        self._prev_before = -1

    @property
    def it(self):
        return len(self.times)

    # ---- the lists ---------------------------------------------------------------------------------------------------
    def _argsort(self, times):
        idx = [j for j in range(len(times)) if j not in self.gone]
        if self.variant == "unstable":
            return sorted(idx, key=lambda j: (times[j], -j))
        return [idx[k] for k in np.argsort(np.array([times[j] for j in idx], dtype=np.int64), kind="stable")]

    def _md_add(self, T, rows):
        md = self.md
        entry = (T, self.seq, rows)
        self.seq += 1
        if self.variant == "bisect_left":
            if not md or T > md[-1][0]:
                md.append(entry)
            else:
                for i in range(len(md)):
                    if T <= md[i][0]:
                        md.insert(i, entry)
                        break
            return
        if not md or T >= md[-1][0]:                     # PredictiveModel.py:36-40
            md.append(entry)
        else:
            for i in range(len(md)):                     # PredictiveModel.py:41-46
                if T < md[i][0]:
                    md.insert(i, entry)
                    break

    def _after_ss_event(self, new, own_latest=None):
        resident = set(self._argsort(self.times)[:self.numSS_it]) | {new}
        if own_latest is not None:
            resident.add(own_latest)
        if len(resident) > self.ss_cap:
            self.flag |= 64
            self.dead = True
        if self.variant == "evict_fastest":
            live = [j for j in range(self.it) if j not in self.gone]
            while len(live) > self.ss_cap:
                j = min((j for j in live if j not in (new, own_latest)), key=lambda j: (self.times[j], j))
                self.gone.add(j)
                live.remove(j)

    def own(self, Trec, x=None, u=None):
        """The controller's own lap of Trec rows (x[Trec, 6], u[Trec, 2]: its record, or None)."""
        self._prev_before = self.it - 1
        n = min(Trec, self.Tmax)                         # rows stored
        ss = md = None
        if x is not None:
            ss = (x[:n], u[:n], compute_cost(x[:n, 4], self.TrackLength))
            md = (x[:n], u[:n])
        self.times.append(Trec)
        self.ss_rows.append(ss)
        self._after_ss_event(self.it - 1)
        self._md_add(Trec, md)
        self.lap_hist.append(Trec)

    def imp(self, lt, length=None, R=None, Tpad=None):
        """A lap another controller drove, with lap time lt and `length` shipped rows R[Tpad, 9] (or None).  Returns "none"
        (it = 0: nothing taken), "dropped" (only the model list took it) or "filed"."""
        if self.it < 1:
            return "none"
        self._prev_before = self.it - 1
        T = lt
        ss = md = None
        if R is not None:
            n = min(length, Tpad, self.Tmax)
            ss = (R[:n, 0:6], R[:n, 6:8], R[:n, 8])
            m = min(lt, length, Tpad, self.Tmax)
            md = (R[:m, 0:6], R[:m, 6:8])
        if self.variant == "import_after":
            pos = self.it
        else:
            pos = self.it - 1
        times = self.times[:pos] + [T] + self.times[pos:]
        if pos not in self._argsort(times)[:self.numSS_it]:
            self._md_add(T, md)
            return "dropped"
        self.times = times
        self.ss_rows.insert(pos, ss)
        if self.variant == "import_after":
            self._after_ss_event(self.it - 1)
        else:
            self._after_ss_event(self.it - 2, own_latest=self.it - 1)
        self._md_add(T, md)
        return "filed"

    # ---- what the next lap reads -----------------------------------------------------------------------------------------
    def sel(self):
        """Lap numbers of the numSS_it laps K2 selects, in order, and the flag (8: fewer laps than numSS_it)."""
        order = self._argsort(self.times)[:self.numSS_it]
        if len(order) < self.numSS_it:
            return order + [order[-1]] * (self.numSS_it - len(order)) if order else [], 8
        return order, 0

    def is_prev(self):
        return [1 if j == self.it - 1 else 0 for j in self.sel()[0]]

    def prev(self):
        """The lap addPoint extends (and the exchange ships): lap it-1, -1 = none."""
        if self.variant == "stale_prev":
            return self._prev_before
        return self.it - 1

    def used(self):
        """Arrival numbers of usedIt, the first trToUse model laps; the slowest repeats when there are fewer."""
        u = [s for (_, s, _) in self.md[:self.trToUse]]
        return u + [u[-1]] * (self.trToUse - len(u)) if u else []

    def resident(self):
        """Safe-set lap numbers the slot table must hold: the numSS_it fastest and lap it-1."""
        r = set(self._argsort(self.times)[:self.numSS_it])
        if self.it >= 1:
            r.add(self.it - 1)
        return r

    def md_by_seq(self):
        return {s: (t, rows) for (t, s, rows) in self.md}


# ---- the pooled exchange -------------------------------------------------------------------------------------------------
POOL_MAXSRC = 64


def pool_local_best(cands, kbest, Tpad, min_over):
    """cands: [(lap time, controller, rows stored)] of the latest own laps of one group.  The kbest fastest, ascending (lap
    time, controller), that ship at least min_over rows past the finish line; -1 pads."""
    ok = [(t, b) for (t, b, n) in cands if not (min_over > 0 and min(n, Tpad) - t < min_over)]
    ok.sort()
    best = [b for (_, b) in ok[:kbest]]
    return best + [-1] * (kbest - len(best))


def pool_rank(meta, G):
    """Per group g in [0, G): indices of the gathered rows of g, valid rows (gid >= 0, len >= 2) first, then ascending (lap
    time, gid), then row index; at most POOL_MAXSRC."""
    out = []
    for g in range(G):
        rows = [i for i in range(len(meta)) if int(meta[i][3]) == g]
        rows.sort(key=lambda i: (not (meta[i][2] >= 0 and meta[i][0] >= 2), int(meta[i][1]), int(meta[i][2]), i))
        out.append(rows[:POOL_MAXSRC])
    return out


def pool_pick(order, meta, gid, share):
    """The rows a controller with global id `gid` takes from its group's ranking: skip its own, stop at the first invalid
    row, at most `share`."""
    got = []
    for i in order:
        if len(got) >= share:
            break
        ln, _, g, _ = (int(v) for v in meta[i])
        if g < 0 or ln < 2:
            break
        if g == gid:
            continue
        got.append(i)
    return got
