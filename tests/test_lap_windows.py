"""CPU tier: per-controller lap windows (lmpc_set_lap_windows).

The struct and the exported symbols, _native.make_lap_window_sets and its refusals, the cross-check with per-controller lap
counts in both install orders, the host lap books of a batch with mixed windows against tests/support/lapbook_window.py (one
unbounded list per controller, each with its own windows) after every own lap and import, and the argument checks of
rollout_mc.run(lap_window_sets=...), all raised before any device work."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat, reference_params as rp
from racinglmpc_b200.controller import BatchedController
import lapbook_exact as lx
from lapbook_window import WindowBooks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
import rollout_mc                                                  # noqa: E402

B = 16
NIT = 4
W = rp.LapWindowParams


def _pack(windows, index=None, laps=None, ss_cap=7, trToUse=4, model_cap=5, lmpc=True):
    index = np.arange(B) % len(windows) if index is None else index
    return nat.make_lap_window_sets(windows, index, B, [NIT] * B if laps is None else laps, ss_cap, trToUse, model_cap, lmpc)


def test_library_exports_the_call_and_the_struct_size_matches():
    assert {"lmpc_set_lap_windows", "lmpc_sizeof_lap_window_params"} <= set(nat.exported_symbols())
    L = nat.lib()                                 # asserts lmpc_sizeof_lap_window_params() == sizeof(LapWindowParams)
    assert L.lmpc_sizeof_lap_window_params() == C.sizeof(nat.LapWindowParams) == 8
    assert L.lmpc_set_lap_windows(None, None, 0, None) != 0 and b"null handle" in L.lmpc_last_error()


def test_valid_windows_pack_in_order():
    packed, idx = _pack([W(0, 0), W(4, 4), W(7, 5), W(5, 0)])
    assert [(p.ss_window, p.model_window) for p in packed] == [(0, 0), (4, 4), (7, 5), (5, 0)]
    assert idx.dtype == np.int32 and np.array_equal(idx, np.arange(B) % 4)
    assert W.unbounded() == W(0, 0)
    packed, _ = _pack([W(np.int64(6), np.int32(4))])
    assert (packed[0].ss_window, packed[0].model_window) == (6, 4)


@pytest.mark.parametrize("ss", [-1, 8, 100])
def test_ss_window_outside_zero_or_up_to_ss_cap_is_refused(ss):
    with pytest.raises(ValueError, match=r"ss_window must be 0 or numSS_it \.\. ss_cap \(7\)"):
        _pack([W(0, 0), W(ss, 0)])


@pytest.mark.parametrize("ss, laps", [(3, NIT), (1, 2), (2, 3)])
def test_ss_window_below_the_controllers_numSS_it_is_refused(ss, laps):
    lap = [NIT] * B
    lap[5] = laps
    with pytest.raises(ValueError, match=r"controller 5: ss_window %d is below its numSS_it \(%d\)" % (ss, laps)):
        _pack([W(0, 0), W(ss, 0)], (np.arange(B) == 5).astype(int), laps=lap)
    lap[5] = 1                                                      # the controller's own numSS_it 1 admits any window
    _pack([W(0, 0), W(ss, 0)], (np.arange(B) == 5).astype(int), laps=lap)


@pytest.mark.parametrize("mw", [-1, 1, 3, 6])
def test_model_window_outside_zero_or_trToUse_to_model_cap_is_refused(mw):
    with pytest.raises(ValueError, match=r"model_window must be 0 or trToUse \(4\) \.\. model_cap \(5\)"):
        _pack([W(0, mw)])


@pytest.mark.parametrize("field", ["ss_window", "model_window"])
@pytest.mark.parametrize("value", [4.0, "4", None, True])
def test_window_that_is_not_an_integer_is_refused(field, value):
    kw = {"ss_window": 4, "model_window": 4}
    kw[field] = value
    with pytest.raises(ValueError, match="%s must be an integer" % field):
        _pack([W(**kw)])


def test_ss_window_on_an_mpc_handle_is_refused():
    with pytest.raises(ValueError, match="no safe set"):
        _pack([W(4, 0)], lmpc=False)
    _pack([W(0, 4)], lmpc=False)                                    # the model window alone is fine


@pytest.mark.parametrize("index", [None, np.zeros(B - 1, int), np.full(B, 2), np.full(B, -1), np.full(B, 0.5)])
def test_bad_index_is_refused(index):
    with pytest.raises(ValueError):
        nat.make_lap_window_sets([W(0, 0), W(4, 4)], index, B, [NIT] * B, 7, 4, 5)


class _Stub:
    def __getattr__(self, name):
        if not name.startswith("lmpc_"):
            raise AttributeError(name)
        return lambda *a: 0


class _Counting(_Stub):
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        f = super().__getattr__(name)
        return lambda *a: (self.calls.append(name), f(*a))[1]


@pytest.fixture
def stubbed(monkeypatch):
    monkeypatch.setattr(nat, "lib", lambda: _Stub())


TMAX = 64


def _host(batch, ss_cap, trToUse, model_cap, M=24, N=14, nit=NIT):
    _, _, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, batch, np.array([[0.0, 19.3, 0.0]]), 19.3, trToUse=trToUse, numSS_Points=M, numSS_it=nit,
                          QterminalSlack=Qts, Tmax=TMAX, ss_cap=ss_cap, model_cap=model_cap)
    c._h = C.c_void_p(1)
    return c


def test_controller_refuses_bad_windows_before_any_native_call(monkeypatch):
    lib = _Counting()
    monkeypatch.setattr(nat, "lib", lambda: lib)
    c = _host(4, 7, 4, 5)
    lib.calls.clear()
    for bad in ([W(8, 0)], [W(3, 0)], [W(0, 6)], [W(4.0, 0)]):
        with pytest.raises(ValueError):
            c.set_lap_windows(bad, [0] * 4)
    with pytest.raises(ValueError, match="index"):
        c.set_lap_windows([W(4, 4)], [0] * 3)
    with pytest.raises(ValueError, match="takes no index"):
        c.set_lap_windows(None, [0] * 4)
    assert "lmpc_set_lap_windows" not in lib.calls
    assert [c.lap_windows_of(b) for b in range(4)] == [(0, 0)] * 4
    c.set_lap_windows([W(0, 0), W(5, 4)], [0, 1, 1, 0])
    assert lib.calls[-1] == "lmpc_set_lap_windows"
    assert [c.lap_windows_of(b) for b in range(4)] == [(0, 0), (5, 4), (5, 4), (0, 0)]
    c.set_lap_windows(None)
    assert [c.lap_windows_of(b) for b in range(4)] == [(0, 0)] * 4
    c._h = None


def test_both_install_orders_against_the_lap_counts(stubbed):
    c = _host(4, 7, 4, 5, M=24)
    c.set_ss_laps([2, 4], [0, 1, 0, 0])
    with pytest.raises(ValueError, match=r"controller 1: ss_window 3 is below its numSS_it \(4\)"):
        c.set_lap_windows([W(3, 0)], [0] * 4)
    c.set_lap_windows([W(3, 0), W(4, 0)], [0, 1, 0, 0])             # controller 1 (numSS_it 4) has a window of 4
    c.set_ss_laps([2, 3], [0, 1, 0, 0])                             # a value at or below the window is fine
    with pytest.raises(ValueError, match=r"controller 0: numSS_it 4 exceeds its ss_window \(3\)"):
        c.set_ss_laps([4], [0] * 4)
    with pytest.raises(ValueError, match=r"controller 0: numSS_it 4 exceeds its ss_window \(3\)"):
        c.set_ss_laps(None)                                        # the handle's numSS_it 4 against the window 3
    c.set_lap_windows(None)
    c.set_ss_laps(None)
    c._h = None


def _agree(c, b, m):
    """The host books of controller b agree with its windowed list m; raises AssertionError.  False when the selection flags 8."""
    nit = c.ss_laps_of(b)
    assert c.it[b] == m.it and c.LapTime[b] == m.times
    assert c.model_laps[b] == [(t, s) for (t, s, _) in m.md]
    stored = c.ss_book[b].slot_of
    assert len(stored) <= m.ss_cap and m.resident() <= set(stored)
    mstored = c.model_book[b].slot_of
    assert len(mstored) <= m.model_cap and m.md_resident() <= set(mstored)
    c._flush()
    minv = {s: ln for ln, s in mstored.items()}
    assert [minv[int(s)] for s in c._used[b]] == m.used()
    sel, flag = m.sel()
    if flag:
        return False
    inv = {s: ln for ln, s in stored.items()}
    assert [inv[int(s)] for s in c._sel[b, :nit]] == sel
    assert list(c._isp[b, :nit]) == m.is_prev()
    assert inv.get(int(c._prev[b]), -1) == m.prev()
    return True


# (ss_cap, trToUse, model_cap, numSS_it, windows): each batch interleaves its windows; ss_cap = W and model_cap = Wm appear in
# every configuration, numSS_it = 1 gives imports that are dropped on arrival, model_window = trToUse
CASES = [(7, 4, 5, 4, [(0, 0), (4, 4), (7, 5), (5, 0), (6, 4)]),
         (5, 3, 4, 2, [(5, 4), (2, 3), (3, 0), (0, 3), (4, 4)]),
         (4, 2, 3, 1, [(1, 2), (2, 3), (4, 0), (3, 2), (0, 3)]),
         (3, 1, 2, 1, [(3, 2), (1, 1), (2, 0), (0, 2)])]


@pytest.mark.parametrize("cfg", CASES, ids=["nit4", "nit2", "nit1", "nit1-small"])
def test_host_books_with_lap_windows_equal_the_window_aware_lists(monkeypatch, cfg):
    """Controllers with mixed windows, each on its own seeded sequence of own laps and imports: after every event the host books
    equal the exact list created with the controller's windows -- stored laps, selection, is_prev, prev_slot, usedIt -- and a
    window within the capacities never makes the pool too small."""
    monkeypatch.setattr(nat, "lib", lambda: _Stub())
    ss_cap, trToUse, model_cap, nit, wins = cfg
    rng = np.random.default_rng(20261018 + ss_cap)
    nb = 2 * len(wins)
    checked = dropped = 0
    for _ in range(24):
        c = _host(nb, ss_cap, trToUse, model_cap, M=24, nit=nit)
        c.set_lap_windows([W(*w) for w in wins], np.arange(nb) % len(wins))
        models = [WindowBooks(nit, ss_cap, trToUse, model_cap, Tmax=TMAX, ss_window=c.lap_windows_of(b)[0],
                           md_window=c.lap_windows_of(b)[1]) for b in range(nb)]
        own = [[] for _ in range(nb)]
        live = [True] * nb
        rows, lens = np.zeros((1, 4, 9)), np.zeros(1, np.int32)
        for step in range(int(rng.integers(14, 30))):
            for b in range(nb):
                if not live[b]:
                    continue
                m = models[b]
                imp = step >= nit and rng.random() < 0.45
                T = int(own[b][-1]) if imp and rng.random() < 0.3 else int(rng.integers(1, 40))
                try:
                    if imp:
                        got = m.imp(T)
                        dropped += got == "dropped"
                        src = np.full(nb, -1); src[b] = 0
                        took = c.import_laps(src, np.full(nb, T), 4, rows, lens)
                        assert (b in took) == (got == "filed"), (b, got)
                    else:
                        own[b].append(T)
                        m.own(T)
                        done = np.zeros(nb, np.int32); done[b] = 1
                        c.rollout_finish_laps(done, np.full(nb, T, np.int32))
                except RuntimeError as e:                            # only an unbounded window can outgrow the pool
                    assert "pool too small" in str(e) and m.dead and c.lap_windows_of(b)[0] == 0, (b, T)
                    live[b] = False
                    continue
                assert not m.dead, "controller %d: flag 64 expected" % b
                if step >= nit:
                    checked += _agree(c, b, m)
        c._h = None
    assert checked > 0
    if nit == 1:
        assert dropped > 0                                          # imports the own latest lap keeps out for good


def test_exact_lists_with_a_window_covering_every_lap_equal_the_unbounded_ones():
    """A window that covers every lap selects the laps no window selects: by lap number while every import is filed, by lap
    time always (a window stores an import the unbounded list drops, which takes a lap number but is never selected)."""
    rng = np.random.default_rng(7)
    differed = 0
    for _ in range(60):
        a = lx.Books(3, 64, 2, 64, Tmax=TMAX)
        w = WindowBooks(3, 64, 2, 64, Tmax=TMAX, ss_window=60, md_window=60)
        for _ in range(int(rng.integers(3, 24))):
            T = int(rng.integers(1, 30))
            if a.it >= 1 and rng.random() < 0.4:
                ga, gw = a.imp(T), w.imp(T)
                assert gw == "filed" and ga in ("filed", "dropped")
            else:
                a.own(T); w.own(T)
            assert a.used() == w.used() and a.is_prev() == w.is_prev() and a.sel()[1] == w.sel()[1]
            assert [a.times[j] for j in a.sel()[0]] == [w.times[j] for j in w.sel()[0]]
            if a.it == w.it:
                assert a.sel() == w.sel() and a.prev() == w.prev()
            differed += a.it != w.it
    assert differed > 0


def test_windows_of_the_recent_laps_select_the_last_laps():
    """ss_window = numSS_it selects exactly the last numSS_it laps; model_window = trToUse uses exactly the last trToUse."""
    rng = np.random.default_rng(11)
    m = WindowBooks(3, 3, 2, 2, Tmax=TMAX, ss_window=3, md_window=2)
    for _ in range(3):
        m.own(int(rng.integers(1, 30)))
    for _ in range(20):
        m.own(int(rng.integers(1, 30)))
        assert sorted(m.sel()[0]) == [m.it - 3, m.it - 2, m.it - 1]
        assert sorted(m.used()) == [m.seq - 2, m.seq - 1]
        assert not m.dead


def test_driver_refuses_bad_windows_and_other_window_rows():
    with pytest.raises(ValueError, match=r"ss_window must be 0 or numSS_it \.\. ss_cap \(7\)"):
        rollout_mc.run(batch=8, lap_window_sets=([W(0, 0), W(8, 0)], np.arange(8) % 2))
    with pytest.raises(ValueError, match=r"controller 1: ss_window 3 is below its numSS_it \(4\)"):
        rollout_mc.run(batch=8, lap_window_sets=([W(0, 0), W(3, 0)], np.arange(8) % 2))
    with pytest.raises(ValueError, match=r"model_window must be 0 or trToUse \(4\) \.\. model_cap \(5\)"):
        rollout_mc.run(batch=8, lap_window_sets=([W(4, 6)], np.zeros(8, int)))
    with pytest.raises(ValueError, match="index"):
        rollout_mc.run(batch=8, lap_window_sets=([W(4, 4)], np.zeros(7, int)))
    # with lap counts the window is checked against each controller's own value: 3 is fine for numSS_it 2
    with pytest.raises(ValueError, match=r"controller 0: ss_window 3 is below its numSS_it \(4\)"):
        rollout_mc.run(batch=8, ss_laps_sets=([4, 2], np.arange(8) % 2), lap_window_sets=([W(3, 0)], np.zeros(8, int)))
    def rows(*windows):
        return rollout_mc.table_rows(rollout_mc.pack_tables(8, lap_window_sets=(list(windows), np.zeros(8, int)))[0])
    w = rows(W(4, 4))
    rollout_mc.check_start_tables({}, {})
    rollout_mc.check_start_tables(w, rows(W(4, 4)))
    for had, mine in (({}, w), (w, {}), (w, rows(W(0, 0)))):
        with pytest.raises(ValueError, match="other lap windows"):
            rollout_mc.check_start_tables(had, mine)


def test_window_lists_with_unbounded_windows_are_the_unbounded_lists():
    """WindowBooks with both windows 0 files, drops, selects and flags exactly as lapbook_exact.Books."""
    rng = np.random.default_rng(13)
    for cfg in ((4, 6, 4, 5), (1, 2, 1, 1), (2, 3, 3, 4)):
        for _ in range(30):
            a, w = lx.Books(*cfg, Tmax=TMAX), WindowBooks(*cfg, Tmax=TMAX)
            for _ in range(int(rng.integers(3, 24))):
                T = int(rng.integers(1, 30))
                if a.it >= 1 and rng.random() < 0.4:
                    assert a.imp(T) == w.imp(T)
                else:
                    a.own(T); w.own(T)
                assert (a.times, a.sel(), a.used(), a.resident(), a.prev(), a.flag, a.dead) == \
                       (w.times, w.sel(), w.used(), w.resident(), w.prev(), w.flag, w.dead)
                assert w.md_resident() == set(a.used())
