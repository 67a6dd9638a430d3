"""CPU tier: lane-safe safe sets (lmpc_set_lane_rules) -- the ABI record, packing and every refusal in both install orders, the
driver's refusals, the judgement of tests/support/lapbook_lane.py at its edges, LaneBooks against hand-built lists (with lap
windows) and against WindowBooks with every rule off, and split_lane_key."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat
from racinglmpc_b200.reference_params import LaneRuleParams as R
from lapbook_lane import LaneBooks, lane_unsafe, LANE_UNSAFE_KEY
from lapbook_window import WindowBooks

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "benchmarks"))
import rollout_mc                                                      # noqa: E402

FX = np.array([[0., 0., 0., 0., 0., 1.], [0., 0., 0., 0., 0., -1.]])
BX = np.array([0.4, 0.4])


def test_abi_record_and_constants():
    assert C.sizeof(nat.LaneRuleParams) == 16
    assert nat.LaneRuleParams.lane_tol.offset == 8
    assert nat.LANE_UNSAFE_KEY == LANE_UNSAFE_KEY == 1 << 24
    hdr = open(nat.__file__.replace("racinglmpc_b200/_native.py", "include/lmpc_b200.h")).read()
    assert "#define LMPC_LANE_UNSAFE_KEY (1 << 24)" in hdr and "#define LMPC_REPORT_LANE_UNSAFE (1 << 16)" in hdr
    assert nat.REPORT_LANE_UNSAFE == 1 << 16
    assert "lmpc_set_lane_rules" in nat.exported_symbols() and "lmpc_sizeof_lane_rule_params" in nat.exported_symbols()


def test_packing():
    rows, idx = nat.make_lane_rule_sets([R(0, 0.0), R(1, 0.02), R(1, 0)], [2, 0, 1, 1], 4)
    assert [(r.mode, r.pad, r.lane_tol) for r in rows] == [(0, 0, 0.0), (1, 0, 0.02), (1, 0, 0.0)]
    assert idx.dtype == np.int32 and list(idx) == [2, 0, 1, 1]
    rows, _ = nat.make_lane_rule_sets([R(1, 1e300)], np.zeros(3, int), 3, Tcl=(1 << 24) - 1)
    assert rows[0].lane_tol == 1e300


@pytest.mark.parametrize("rule", [R(2, 0.0), R(-1, 0.0), R(True, 0.0), R(1.0, 0.0), R(1, -1e-300), R(1, math.nan), R(1, math.inf),
                                  R(0, -math.inf), R(1, "0.1"), R(1, None)])
def test_refused_rows(rule):
    with pytest.raises(ValueError):
        nat.make_lane_rule_sets([rule], np.zeros(2, int), 2)


def test_refused_index_handle_and_record_length():
    with pytest.raises(ValueError):
        nat.make_lane_rule_sets([R(1, 0.0)], [0, 1], 2)                    # index out of range
    with pytest.raises(ValueError):
        nat.make_lane_rule_sets([R(1, 0.0)], [0], 2)                       # one index per controller
    with pytest.raises(ValueError):
        nat.make_lane_rule_sets([R(1, 0.0)], [0, 0], 2, lmpc=False)        # no safe set
    with pytest.raises(ValueError):
        nat.make_lane_rule_sets([R(1, 0.0)], [0, 0], 2, Tcl=1 << 24)      # a lap time could reach the key
    nat.make_lane_rule_sets([R(0, 0.0)], [0, 0], 2, Tcl=1 << 24)          # mode 0 never keys a lap


class _Stub:
    """What BatchedController's lane-rule methods read, without a GPU handle."""
    from racinglmpc_b200.controller import BatchedController as _BC
    set_lane_rules = _BC.set_lane_rules
    lane_rules_of = _BC.lane_rules_of
    _no_lane_rule = _BC._no_lane_rule
    enable_rollout = _BC.enable_rollout
    _install = _BC._install

    def __init__(self, B=4, lmpc=True):
        self.B, self.lmpc, self._lane, self.calls = B, lmpc, None, []

        class L:
            def lmpc_set_lane_rules(_, h, rows, n, idx):
                self.calls.append(n)
                return 0

            def lmpc_rollout_create(_, h, Tcl):
                self.calls.append(("create", Tcl))
                return 0
        self._lib, self._h = L(), None


def test_both_install_orders():
    s = _Stub()
    s.enable_rollout(Tcl=1 << 24)                                          # no rule yet: any Tcl the library takes
    with pytest.raises(ValueError):
        s.set_lane_rules([R(1, 0.0)], np.zeros(4, int))                    # the rollout's Tcl reaches the key
    assert s.calls == [("create", 1 << 24)] and s._lane is None
    s = _Stub()
    s.set_lane_rules([R(0, 0.0), R(1, 0.05)], [0, 1, 1, 0])
    assert [s.lane_rules_of(b) for b in range(4)] == [(0, 0.0), (1, 0.05), (1, 0.05), (0, 0.0)]
    with pytest.raises(ValueError):
        s.enable_rollout(Tcl=1 << 24)                                      # the other order
    with pytest.raises(ValueError):
        s._no_lane_rule("rollout_finish_laps")                             # host-slot paths
    s.set_lane_rules(None)
    assert s.lane_rules_of(2) == (0, 0.0) and s.calls[-1] == 0
    s._no_lane_rule("rollout_finish_laps")
    with pytest.raises(ValueError):
        s.set_lane_rules(None, [0, 0, 0, 0])                               # removal takes no index
    with pytest.raises(ValueError):
        _Stub(lmpc=False).set_lane_rules([R(0, 0.0)], np.zeros(4, int))


def test_driver_refusals_and_start_rule_rows():
    rmc = rollout_mc
    for bad in (([R(2, 0.0)], np.zeros(8, int)), ([R(1, -1.0)], np.zeros(8, int)), ([R(1, 0.0)], np.ones(8, int)),
                ([R(1, 0.0)], np.zeros(7, int))):
        with pytest.raises(ValueError):
            rmc.run(batch=8, laps=1, lane_rule_sets=bad)
    rule, none = rmc.table_rows(rmc.pack_tables(8, lane_rule_sets=([R(1, 0.0)], np.zeros(8, int)))[0]), {}
    other = rmc.table_rows(rmc.pack_tables(8, lane_rule_sets=([R(1, 0.01)], np.zeros(8, int)))[0])
    for had, mine in ((rule, none), (none, rule), (rule, other)):
        with pytest.raises(ValueError, match="other lane rules"):
            rmc.check_start_tables(had, mine)
    rmc.check_start_tables(rule, rule)
    rmc.check_start_tables(none, none)


def _row(ey):
    return np.array([[1.0, 0.0, 0.0, 0.0, 3.0, ey]])


def test_lane_unsafe_at_its_edges():
    w = 0.4
    assert not lane_unsafe(_row(w), FX, BX, 0.0)                           # exactly on the lane edge: d = 0 is not > 0
    assert lane_unsafe(_row(np.nextafter(w, 1.0)), FX, BX, 0.0)             # one ulp outside
    assert not lane_unsafe(_row(-w), FX, BX, 0.0)
    assert lane_unsafe(_row(-np.nextafter(w, 1.0)), FX, BX, 0.0)
    tol = 0.02
    edge = (w + tol)
    d = edge - w                                                           # the margin the device computes at ey = edge
    assert not lane_unsafe(_row(edge), FX, BX, d)
    assert lane_unsafe(_row(np.nextafter(edge, 1.0)), FX, BX, d) == ((np.nextafter(edge, 1.0) - w) > d)
    for bad in (np.nan, np.inf, -np.inf):
        x = _row(0.0)
        x[0, 2] = bad                                                      # a non-finite entry outside the lane rows too
        assert lane_unsafe(x, FX, BX, 1e300)
    assert not lane_unsafe(np.zeros((0, 6)), FX, BX, 0.0)
    # in order, separate multiplies and adds: 0 * inf would be nan, but only finite rows get there
    x = np.array([[1e308, 0, 0, 0, 0, 0.1]])
    assert not lane_unsafe(x, FX, BX, 0.0)
    assert lane_unsafe(x, FX * 2.0, BX, 0.0) == (((0.0 * 1e308 + 0.0) + 0.0 + 0.0 + 0.0 + 0.2) - 0.4 > 0)


def _own(m, times, unsafe):
    for t, u in zip(times, unsafe):
        m.own(t, unsafe=u)


def test_lane_books_rank_unsafe_laps_behind_safe_ones():
    m = LaneBooks(2, 4, 1, 2, 100, lane_mode=1, lane_tol=0.0, Fx=FX, bx=BX)
    _own(m, [50, 40, 45, 30], [False, True, False, True])
    assert m.times == [50, 40 + LANE_UNSAFE_KEY, 45, 30 + LANE_UNSAFE_KEY]
    assert m.sel() == ([2, 0], 0)                                          # the safe laps, fastest first
    assert m.lap_hist == [50, 40, 45, 30] and [t for t, _, _ in m.md] == [30, 40, 45, 50]   # raw lengths
    assert m.prev() == 3 and 3 in m.resident()                             # an unsafe own latest lap stays lap it-1
    m2 = LaneBooks(3, 5, 1, 2, 100, lane_mode=1, Fx=FX, bx=BX)
    _own(m2, [50, 40, 30], [True, False, True])
    assert m2.sel() == ([1, 2, 0], 0)                                      # unsafe laps fill the selection, by lap time
    m3 = LaneBooks(3, 5, 1, 2, 100, lane_mode=1, Fx=FX, bx=BX)
    _own(m3, [50, 40], [True, False])
    assert m3.sel() == ([1, 0, 0], 8)                                      # flag 8 is unchanged


def test_lane_books_with_windows_against_hand_built_lists():
    m = LaneBooks(2, 4, 1, 2, 100, ss_window=3, lane_mode=1, Fx=FX, bx=BX)
    _own(m, [30, 50, 60, 40, 55], [False, False, True, True, False])
    # the window is laps 2, 3, 4: keys 60+K, 40+K, 55 -> lap 4 (safe), then lap 3 (unsafe, faster than lap 2)
    assert m.sel() == ([4, 3], 0)
    assert m.resident() == {3, 4}
    # an import is filed as lap it-1 and judged by the importer: unsafe, it ranks behind the safe own latest
    R_ = np.zeros((20, 9))
    R_[:, 5] = 0.5                                                         # outside the 0.4 lane
    assert m.imp(10, 20, R_, 32) == "filed"
    assert m.times[4] == 10 + LANE_UNSAFE_KEY and m.times[5] == 55
    assert m.sel() == ([5, 4], 0)
    R_[:, 5] = 0.1
    assert m.imp(12, 20, R_, 32) == "filed"                                # safe: the fastest
    assert m.times[4:] == [10 + LANE_UNSAFE_KEY, 12, 55]
    assert m.sel() == ([5, 6], 0)                                          # the window is laps 4, 5, 6: 12, 55, then 10 + K
    R_[:12, 5] = 0.1
    R_[12:, 5] = 9.0                                                       # rows past min(lt, rows, Tpad) are not judged
    m4 = LaneBooks(2, 4, 1, 2, 100, lane_mode=1, Fx=FX, bx=BX)
    m4.own(30, unsafe=False)
    assert m4.imp(12, 20, R_, 32) == "filed" and m4.times[0] == 12


def test_every_rule_off_is_window_books_exactly():
    rng = np.random.default_rng(7)
    for mode, win in ((0, (0, 0)), (0, (3, 2)), (None, (4, 0))):
        a = WindowBooks(2, 4, 2, 3, 40, ss_window=win[0], md_window=win[1])
        b = LaneBooks(2, 4, 2, 3, 40, ss_window=win[0], md_window=win[1], lane_mode=mode or 0, lane_tol=0.0, Fx=FX, bx=BX)
        for _ in range(60):
            if rng.random() < 0.3 and a.it >= 1:
                lt, ln = int(rng.integers(1, 50)), int(rng.integers(2, 60))
                Rr = rng.standard_normal((32, 9))
                assert a.imp(lt, ln, Rr, 32) == b.imp(lt, ln, Rr, 32)
            else:
                T = int(rng.integers(1, 50))
                x, u = rng.standard_normal((T, 6)), rng.standard_normal((T, 2))
                a.own(T, x, u)
                b.own(T, x, u)
            assert a.times == b.times and a.sel() == b.sel() and a.used() == b.used() and a.flag == b.flag
            assert a.resident() == b.resident() and [e[:2] for e in a.md] == [e[:2] for e in b.md]


def test_split_lane_key():
    assert nat.split_lane_key(57) == (57, False)
    assert nat.split_lane_key(57 + (1 << 24)) == (57, True)
    assert nat.split_lane_key(0x7FFFFFFF) == (0x7FFFFFFF, False)           # a free slot
    t, u = nat.split_lane_key(np.array([[3, (1 << 24) + 3], [-1, 0x7FFFFFFF]], np.int32))
    assert t.dtype == np.int32 and t.tolist() == [[3, 3], [-1, 0x7FFFFFFF]]
    assert u.tolist() == [[False, True], [False, False]]
