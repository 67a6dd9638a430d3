"""CPU tier: per-controller safe-set lap counts (lmpc_set_ss_laps).

The struct and the exported symbols, _native.make_ss_laps_sets and its refusals, the cross-check with per-controller shapes in
both install orders, the host lap books of a batch with interleaved lap counts against tests/support/lapbook_exact.py (one
unbounded list per controller, each with its own numSS_it) at capacity, and the argument checks of rollout_mc.run(ss_laps_sets=...),
all raised before any device work."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat, reference_params as rp
from racinglmpc_b200.controller import BatchedController
import lapbook_exact as lx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
import rollout_mc                                                  # noqa: E402

B = 16
NIT = 4                                                            # the handle's numSS_it (the reference's)


def test_library_exports_the_call_and_the_struct_size_matches():
    assert {"lmpc_set_ss_laps", "lmpc_sizeof_ss_laps_params"} <= set(nat.exported_symbols())
    L = nat.lib()                                 # asserts lmpc_sizeof_ss_laps_params() == sizeof(SsLapsParams)
    assert L.lmpc_sizeof_ss_laps_params() == C.sizeof(nat.SsLapsParams) == 4
    assert L.lmpc_set_ss_laps(None, None, 0, None) != 0 and b"null handle" in L.lmpc_last_error()


def test_valid_sets_pack_in_order():
    idx = np.arange(B) % 4
    packed, pidx = nat.make_ss_laps_sets([3, 1, 4, 2], idx, B, NIT, [48] * B)
    assert [p.numSS_it for p in packed] == [3, 1, 4, 2]
    assert pidx.dtype == np.int32 and np.array_equal(pidx, idx)
    packed, _ = nat.make_ss_laps_sets([np.int64(2)], np.zeros(B, int), B, NIT, [24] * B)
    assert [p.numSS_it for p in packed] == [2]


@pytest.mark.parametrize("value", [0, -1, NIT + 1, 8])
def test_value_outside_one_to_the_handles_is_refused(value):
    with pytest.raises(ValueError, match=r"1 \.\. the handle's 4"):
        nat.make_ss_laps_sets([2, value], np.arange(B) % 2, B, NIT, [48] * B)


@pytest.mark.parametrize("value", [2.0, "2", None, True])
def test_value_that_is_not_an_integer_is_refused(value):
    with pytest.raises(ValueError, match="integer"):
        nat.make_ss_laps_sets([value], np.zeros(B, int), B, NIT, [48] * B)


@pytest.mark.parametrize("points, value", [(18, 2), (30, 2), (32, 3), (64, 3), (20, 3)])
def test_odd_or_fractional_points_per_lap_are_refused(points, value):
    pts = [48] * B
    pts[5] = points
    with pytest.raises(ValueError, match="controller 5: numSS_Points %d is not numSS_it \\(%d\\)" % (points, value)):
        nat.make_ss_laps_sets([1, value], (np.arange(B) == 5).astype(int), B, NIT, pts)


def test_mpc_handle_is_refused():
    with pytest.raises(ValueError, match="LMPC handle"):
        nat.make_ss_laps_sets([1], np.zeros(B, int), B, 0, [0] * B)
    with pytest.raises(ValueError, match="LMPC handle"):
        nat.make_ss_laps_sets([1], np.zeros(B, int), B, NIT, [0] * B)


@pytest.mark.parametrize("index", [None, np.zeros(B - 1, int), np.full(B, 2), np.full(B, -1), np.full(B, 0.5)])
def test_bad_index_is_refused(index):
    with pytest.raises(ValueError):
        nat.make_ss_laps_sets([1, 2], index, B, NIT, [48] * B)


def test_empty_or_too_many_sets_are_refused():
    with pytest.raises(ValueError, match="need 1 .. batch"):
        nat.make_ss_laps_sets([], np.zeros(B, int), B, NIT, [48] * B)
    with pytest.raises(ValueError, match="need 1 .. batch"):
        nat.make_ss_laps_sets([1] * (B + 1), np.zeros(B, int), B, NIT, [48] * B)


def test_shapes_are_checked_against_the_lap_counts():
    """The other install order: make_shape_sets with the controllers' lap counts checks every controller's pair."""
    laps = np.where(np.arange(B) == 3, 3, 4)
    shapes, idx = [(14, 96), (14, 32)], (np.arange(B) == 3).astype(int)
    with pytest.raises(ValueError, match=r"controller 3: numSS_Points 32 is not its numSS_it \(3\)"):
        nat.make_shape_sets(shapes, idx, B, 14, 96, NIT, ss_laps=laps)
    nat.make_shape_sets(shapes, idx, B, 14, 96, NIT)                         # without lap counts 32 / 4 is fine
    nat.make_shape_sets([(14, 32), (14, 96)], idx, B, 14, 96, NIT, ss_laps=laps)   # controller 3 (96 / 3 = 32) is fine


class _Stub:
    def __getattr__(self, name):
        if not name.startswith("lmpc_"):
            raise AttributeError(name)
        return lambda *a: 0


@pytest.fixture
def stubbed(monkeypatch):
    monkeypatch.setattr(nat, "lib", lambda: _Stub())


TMAX = 64


def _host(batch, ss_cap, trToUse, model_cap, M=24, N=14):
    _, _, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, batch, np.array([[0.0, 19.3, 0.0]]), 19.3, trToUse=trToUse, numSS_Points=M, numSS_it=NIT,
                          QterminalSlack=Qts, Tmax=TMAX, ss_cap=ss_cap, model_cap=model_cap)
    c._h = C.c_void_p(1)
    return c


def test_controller_refuses_a_bad_pair_in_either_install_order(stubbed):
    c = _host(4, 6, 4, 5, M=96)
    c.set_shapes([(14, 96), (14, 32)], [0, 1, 0, 0])
    with pytest.raises(ValueError, match=r"controller 1: numSS_Points 32 is not numSS_it \(3\)"):
        c.set_ss_laps([4, 3], [0, 1, 0, 0])
    c.set_ss_laps([4, 3], [0, 0, 1, 0])                       # 96 / 3 = 32 points per lap
    assert [c.ss_laps_of(b) for b in range(4)] == [4, 4, 3, 4]
    with pytest.raises(ValueError, match=r"controller 2: numSS_Points 32 is not its numSS_it \(3\)"):
        c.set_shapes([(14, 96), (14, 32)], [0, 0, 1, 0])
    c.set_ss_laps(None)
    assert [c.ss_laps_of(b) for b in range(4)] == [4] * 4
    c._h = None


def _agree(c, b, m):
    """The host books of controller b agree with its unbounded list m (numSS_it of the controller); raises AssertionError."""
    nit = c.ss_laps_of(b)
    assert m.numSS_it == nit
    assert c.it[b] == m.it and c.LapTime[b] == m.times
    assert c.model_laps[b] == [(t, s) for (t, s, _) in m.md]
    stored = c.ss_book[b].slot_of
    assert len(stored) <= m.ss_cap and m.resident() <= set(stored)
    sel, flag = m.sel()
    try:
        c._flush()
    except IndexError:
        assert flag == 8
        return False
    assert flag == 0
    inv = {s: ln for ln, s in stored.items()}
    assert [inv[int(s)] for s in c._sel[b, :nit]] == sel
    assert list(c._isp[b, :nit]) == m.is_prev()
    assert np.all(c._sel[b, nit:] == c._sel[b, nit - 1]) and np.all(c._isp[b, nit:] == 0)   # what the device books write
    assert inv.get(int(c._prev[b]), -1) == m.prev()
    return True


@pytest.mark.parametrize("cfg", [(6, 4, 5), (5, 4, 4), (4, 4, 4), (7, 8, 9)])
def test_host_books_with_per_controller_lap_counts_equal_the_unbounded_lists(stubbed, cfg):
    """Eight controllers with lap counts 1, 2, 3, 4 interleaved, each on its own seeded sequence of own laps and imports (the
    first four own laps stand for the seeding's copies, so that no controller of the batch has fewer laps than its value when
    the books are flushed): after every event the controller's books equal the unbounded list created with its own numSS_it
    and the same ss_cap (flag 64 where the list says the pool is too small)."""
    ss_cap, trToUse, model_cap = cfg
    rng = np.random.default_rng(20261017 + ss_cap)
    nb = 8
    values = [1, 2, 3, 4]
    checked = flagged = 0
    for _ in range(40):
        c = _host(nb, ss_cap, trToUse, model_cap)
        c.set_ss_laps(values, np.arange(nb) % 4)
        models = [lx.Books(c.ss_laps_of(b), ss_cap, trToUse, model_cap, Tmax=TMAX) for b in range(nb)]
        live = [True] * nb
        own = [[] for _ in range(nb)]
        rows, lens = np.zeros((1, 4, 9)), np.zeros(1, np.int32)
        for step in range(int(rng.integers(16, 34))):
            for b in range(nb):
                if not live[b]:
                    continue
                m = models[b]
                imp = step >= NIT and rng.random() < 0.4         # the first NIT laps are own laps, as the seeding's copies
                T = int(own[b][-1]) if imp and rng.random() < 0.3 else int(rng.integers(1, TMAX + 10))
                try:
                    if imp:
                        m.imp(T)
                        src = np.full(nb, -1); src[b] = 0
                        c.import_laps(src, np.full(nb, T), 4, rows, lens)
                    else:
                        own[b].append(T)
                        m.own(T)
                        done = np.zeros(nb, np.int32); done[b] = 1
                        c.rollout_finish_laps(done, np.full(nb, T, np.int32))
                except RuntimeError as e:
                    assert "pool too small" in str(e) and m.dead, (b, T)
                    live[b] = False
                    flagged += 1
                    continue
                if m.dead:                                # the list says flag 64 where the slot tables still found room
                    raise AssertionError("controller %d: flag 64 expected" % b)
                if step >= NIT:                           # every controller has its laps: a flush raises for none
                    checked += _agree(c, b, m)
        c._h = None
    assert checked > 0
    if ss_cap == 4:
        assert flagged > 0                                # the tightest pool reaches flag 64


def test_driver_refuses_bad_lap_counts_before_any_device_work():
    with pytest.raises(ValueError, match=r"1 \.\. the handle's 4"):
        rollout_mc.run(batch=8, ss_laps_sets=([2, 5], np.arange(8) % 2))
    with pytest.raises(ValueError, match="index"):
        rollout_mc.run(batch=8, ss_laps_sets=([2, 3], np.arange(7) % 2))
    # (12, 32) splits into 4 laps of 8 but not into 3 laps
    with pytest.raises(ValueError, match=r"controller 1: numSS_Points 32 is not numSS_it \(3\)"):
        rollout_mc.run(batch=8, shape_sets=([(12, 48), (12, 32)], np.arange(8) % 2), ss_laps_sets=([4, 3], np.arange(8) % 2))
