"""CPU tier: the host lap books of racinglmpc_b200.controller.BatchedController against the unbounded lists of
tests/support/lapbook_exact.py (the reference's LapTime / PredictiveModel lists restated), on seeded random sequences of own laps
and imported laps over the capacity grid of the GPU tier, behind a recording stub in place of liblmpc_b200.  After every event the
full lap lists, which laps are stored, the selection mapped to lap numbers, is_prev, the addPoint target and usedIt mapped to
arrival numbers must agree; flag 64 (pool too small) must be raised exactly when the model expects it.  Each known-wrong
variant of the model must fail the same comparisons."""
import ctypes as C

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat, reference_params as rp
from racinglmpc_b200.controller import BatchedController
import lapbook_exact as lx

# (numSS_it, ss_cap, trToUse, model_cap): library default, test/benchmark default, tightest (flag 64), import edge, smallest
# tables, trToUse > numSS_it, largest tables
GRID = [(4, 6, 4, 5), (4, 7, 4, 5), (4, 4, 4, 4), (4, 5, 4, 4), (1, 2, 1, 1), (2, 4, 8, 8), (8, 10, 8, 9)]
TMAX = 64
SEQS = 300          # random sequences per grid row
LAPS = (20, 48)     # events per sequence


class _Stub:
    def __getattr__(self, name):
        if not name.startswith("lmpc_"):
            raise AttributeError(name)
        return lambda *a: 0


@pytest.fixture
def stubbed(monkeypatch):
    monkeypatch.setattr(nat, "lib", lambda: _Stub())


def _host(cfg):
    numSS_it, ss_cap, trToUse, model_cap = cfg
    _, _, _, _, Qts, par = rp.lmpc_params(12)
    c = BatchedController(par, 1, np.array([[0.0, 19.3, 0.0]]), 19.3, trToUse=trToUse, numSS_Points=2 * numSS_it,
                          numSS_it=numSS_it, QterminalSlack=Qts, Tmax=TMAX, ss_cap=ss_cap, model_cap=model_cap)
    c._h = C.c_void_p(1)
    return c


def _times(rng, n):
    """Lap lengths of one sequence: ties from {k, k+1}, strictly decreasing, strictly increasing, T in {1, 2}, around and above
    Tmax, or uniform."""
    kind = int(rng.integers(6))
    k = int(rng.integers(3, TMAX - 4))
    if kind == 0:
        return list(k + rng.integers(0, 2, n))
    if kind == 1:
        return [TMAX + 10 - i for i in range(n)]
    if kind == 2:
        return [1 + i for i in range(n)]
    if kind == 3:
        return list(rng.integers(1, 3, n))
    if kind == 4:
        return list(rng.integers(TMAX - 3, TMAX + 20, n))
    return list(rng.integers(1, TMAX + 10, n))


def sequence(rng):
    """[("own", T) | ("imp", lt)]: own laps with the first at least one, imports tying the own latest lap and stored laps."""
    n = int(rng.integers(*LAPS))
    ts = _times(rng, 2 * n)
    p_imp = float(rng.choice([0.0, 0.25, 0.5]))
    ev, own = [], []
    for i in range(n):
        if own and rng.random() < p_imp:
            r = rng.random()
            lt = own[-1] if r < 0.3 else (int(rng.choice(own)) if r < 0.6 else int(ts[n + i]))
            ev.append(("imp", int(lt)))
        else:
            own.append(int(ts[i]))
            ev.append(("own", int(ts[i])))
    return ev


def _agree(c, m):
    """The host books of controller 0 agree with model m after an event (see the module docstring); raises AssertionError."""
    assert c.it[0] == m.it
    assert c.LapTime[0] == m.times
    assert c.model_laps[0] == [(t, s) for (t, s, _) in m.md]
    stored = c.ss_book[0].slot_of
    assert len(stored) <= m.ss_cap and m.resident() <= set(stored)
    mstored = c.model_book[0].slot_of
    assert len(mstored) <= m.model_cap and set(m.used()) <= set(mstored)
    sel, flag = m.sel()
    try:
        c._flush()
    except IndexError:
        assert flag == 8
        return
    assert flag == 0
    inv = {s: ln for ln, s in stored.items()}
    assert [inv[int(s)] for s in c._sel[0]] == sel
    assert list(c._isp[0]) == m.is_prev()
    assert inv.get(int(c._prev[0]), -1) == m.prev()
    minv = {s: ln for ln, s in mstored.items()}
    assert [minv[int(u)] for u in c._used[0]] == m.used()


def run_sequence(cfg, ev, variant=None):
    """Drive the host books and the model through one event list; returns the index of the first disagreement or None."""
    c = _host(cfg)
    m = lx.Books(*cfg, Tmax=TMAX, variant=variant)
    rows, lens = np.zeros((1, 4, 9)), np.zeros(1, np.int32)
    try:
        for i, (kind, T) in enumerate(ev):
            try:
                if kind == "own":
                    m.own(T)
                    c.rollout_finish_laps(np.array([1], np.int32), np.array([T], np.int32))
                else:
                    m.imp(T)
                    c.import_laps(np.array([0]), np.array([T]), 4, rows, lens)
            except RuntimeError as e:
                assert "pool too small" in str(e)
                if not m.dead:
                    return i
                return None
            if m.dead:
                return i
            try:
                _agree(c, m)
            except AssertionError:
                return i
        return None
    finally:
        c._h = None


def test_host_books_equal_the_unbounded_lists(stubbed):
    rng = np.random.default_rng(20261016)
    flagged = dropped = 0
    for cfg in GRID:
        for _ in range(SEQS):
            ev = sequence(rng)
            bad = run_sequence(cfg, ev)
            assert bad is None, (cfg, ev[:bad + 1])
            m = lx.Books(*cfg, Tmax=TMAX)
            for kind, T in ev:
                if m.dead:
                    break
                if kind == "own":
                    m.own(T)
                else:
                    dropped += m.imp(T) == "dropped"
            flagged += m.dead
    assert flagged > 0 and dropped > 0            # the sequences reach flag 64 and dropped imports


@pytest.mark.parametrize("variant", lx.VARIANTS)
def test_each_wrong_variant_of_the_lists_is_caught(stubbed, variant):
    rng = np.random.default_rng(7)
    caught = 0
    for cfg in GRID:
        for _ in range(40):
            caught += run_sequence(cfg, sequence(rng), variant) is not None
    assert caught > 0, variant


def test_an_import_the_safe_set_drops_still_reaches_the_regression_model(stubbed):
    """trToUse = 8 > numSS_it = 2: an import slower than the two fastest laps is among the eight shortest model laps."""
    cfg = (2, 4, 8, 8)
    c, m = _host(cfg), lx.Books(*cfg, Tmax=TMAX)
    rows, lens = np.zeros((1, 4, 9)), np.zeros(1, np.int32)
    for T in (30, 20, 25):
        m.own(T)
        c.rollout_finish_laps(np.array([1], np.int32), np.array([T], np.int32))
    assert m.imp(27) == "dropped"
    took = c.import_laps(np.array([0]), np.array([27]), 4, rows, lens)
    assert len(took) == 0 and c.it[0] == 3
    assert (27, 3) in c.model_laps[0] and 3 in c.model_book[0].slot_of
    _agree(c, m)
    assert m.used()[:4] == [1, 2, 3, 0]
    c._h = None


def test_a_lap_longer_than_tmax_keeps_its_lap_time(stubbed):
    """Only Tmax rows of a lap fit a slot, but the lap is ordered by its lap time, own or imported: a slow lap stays slow."""
    cfg = (1, 2, 1, 1)
    c, m = _host(cfg), lx.Books(*cfg, Tmax=TMAX)
    rows, lens = np.zeros((1, 4, 9)), np.zeros(1, np.int32)
    m.own(TMAX + 9)
    c.rollout_finish_laps(np.array([1], np.int32), np.array([TMAX + 9], np.int32))
    assert c.LapTime[0] == [TMAX + 9] and c.model_laps[0] == [(TMAX + 9, 0)]
    assert m.imp(TMAX + 20) == "dropped"          # slower than the own lap: clamped to Tmax it would tie and be filed first
    c.import_laps(np.array([0]), np.array([TMAX + 20]), 4, rows, lens)
    assert c.LapTime[0] == [TMAX + 9] and c.model_laps[0] == [(TMAX + 9, 0), (TMAX + 20, 1)]
    _agree(c, m)
    assert m.imp(TMAX + 3) == "filed"             # faster than the own lap, though both are cut at Tmax rows
    c.import_laps(np.array([0]), np.array([TMAX + 3]), 4, rows, lens)
    assert c.LapTime[0] == [TMAX + 3, TMAX + 9]
    _agree(c, m)
    c._h = None
