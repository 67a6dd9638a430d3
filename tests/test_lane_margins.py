"""CPU tier: lane margins (lmpc_set_lane_margins) -- the ABI record, packing, every refusal (the margin against the QP row in both
install orders with parameter sets), the driver's refusals, the host restatement of the update rule at its edges
(tests/support/lane_margin.py) and the snapshot decoder's name for section 39."""
import ctypes as C
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat
from racinglmpc_b200 import reference_params as rp
from racinglmpc_b200.reference_params import LaneMarginParams as G
import lane_margin as lm

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "benchmarks"))
import rollout_mc                                                      # noqa: E402

FX = np.array([[0., 0., 0., 0., 0., 1.], [0., 0., 0., 0., 0., -1.]])
BX = np.array([0.4, 0.4])


def test_abi_record_and_symbols():
    assert C.sizeof(nat.LaneMarginParams) == 40
    assert [getattr(nat.LaneMarginParams, f).offset for f in ("mode", "pad", "margin0", "margin_max", "step_up", "step_down")] == \
        [0, 4, 8, 16, 24, 32]
    syms = nat.exported_symbols()
    for s in ("lmpc_set_lane_margins", "lmpc_get_lane_margins", "lmpc_sizeof_lane_margin_params"):
        assert s in syms
    assert G.reference() == G(0, 0.0, 0.0, 0.0, 0.0)


def test_packing():
    rows, idx = nat.make_lane_margin_sets([G(0), G(1, 0.05, 0.05), G(2, 0.0, 0.1, 0.01, 0.0025)], [2, 0, 1, 1], 4, np.full(4, 0.4))
    assert [(r.mode, r.pad, r.margin0, r.margin_max, r.step_up, r.step_down) for r in rows] == \
        [(0, 0, 0.0, 0.0, 0.0, 0.0), (1, 0, 0.05, 0.05, 0.0, 0.0), (2, 0, 0.0, 0.1, 0.01, 0.0025)]
    assert idx.dtype == np.int32 and list(idx) == [2, 0, 1, 1]


@pytest.mark.parametrize("row", [G(3), G(-1), G(True), G(1.0), G(1, -1e-300), G(1, math.nan), G(2, 0.0, math.inf),
                                 G(2, 0.0, 0.1, -0.01), G(2, 0.0, 0.1, 0.01, math.nan), G(2, 0.05, 0.01), G(1, "0.1"),
                                 G(1, None)])
def test_refused_rows(row):
    with pytest.raises(ValueError):
        nat.make_lane_margin_sets([row], np.zeros(2, int), 2, np.full(2, 0.4))


def test_a_margin_must_leave_a_lane():
    bx = np.array([0.4, 0.1])
    nat.make_lane_margin_sets([G(1, 0.05, 0.05)], [0, 0], 2, bx)
    nat.make_lane_margin_sets([G(1, 0.3, 0.3), G(0)], [0, 1], 2, bx)             # mode 0 on the narrow lane
    nat.make_lane_margin_sets([G(2, 0.0, 0.0999)], [0, 0], 2, bx)
    for rows in ([G(1, 0.1, 0.1)], [G(2, 0.0, 0.1)], [G(2, 0.0, 0.2, 0.01)], [G(1, 0.5, 0.5)]):
        with pytest.raises(ValueError, match="does not leave a lane"):
            nat.make_lane_margin_sets(rows, [0, 0], 2, bx)
    with pytest.raises(ValueError):
        nat.make_lane_margin_sets([G(1, 0.0)], [0, 1], 2, bx)              # index out of range
    with pytest.raises(ValueError):
        nat.make_lane_margin_sets([G(1, 0.0)], [0], 2, bx)                 # one index per controller


class _Stub:
    """What BatchedController's parameter-set and lane-margin methods read, without a GPU handle."""
    from racinglmpc_b200.controller import BatchedController as _BC
    set_param_sets = _BC.set_param_sets
    set_lane_margins = _BC.set_lane_margins
    lane_margins_of = _BC.lane_margins_of
    lane_margin_values = _BC.lane_margin_values
    rollout_finish_laps = _BC.rollout_finish_laps
    _row_bx_min = staticmethod(_BC._row_bx_min)
    _no_lane_rule = _BC._no_lane_rule
    _install = _BC._install

    def __init__(self, B=4):
        _, _, _, _, Qts, par = rp.lmpc_params(12)
        self.B, self.numSS_it, self._lane, self._margins, self.calls = B, 4, None, None, []
        self._p = nat.make_params(par, 48, 4, Qts)
        self._bx_min = np.full(B, self._row_bx_min(self._p))

        class L:
            def lmpc_set_lane_margins(_, h, rows, n, idx):
                self.calls.append(("margins", n))
                return 0

            def lmpc_set_param_sets(_, h, rows, n, idx):
                self.calls.append(("params", n))
                return 0
        self._lib, self._h = L(), None


def _par(width):
    p = rp.lmpc_params(12)[5]
    return SimpleNamespace(**{**vars(p), "bx": np.array([width, width])})


def test_both_install_orders_against_parameter_sets():
    s = _Stub()
    s.set_param_sets([_par(0.4), _par(0.05)], [0, 1, 0, 1])
    with pytest.raises(ValueError, match="does not leave a lane"):
        s.set_lane_margins([G(1, 0.05, 0.05)], np.zeros(4, int))                 # the narrow set's lane would be gone
    assert s._margins is None and ("margins", 1) not in s.calls
    s.set_lane_margins([G(1, 0.2, 0.2), G(2, 0.0, 0.04, 0.01)], [0, 1, 0, 1])
    assert s.lane_margins_of(1) == (2, 0.0, 0.04, 0.01, 0.0) and s.lane_margins_of(0) == (1, 0.2, 0.2, 0.0, 0.0)
    n = len(s.calls)
    with pytest.raises(ValueError, match="does not leave a lane"):
        s.set_param_sets([_par(0.2), _par(0.05)], [0, 1, 0, 1])           # the other order: controller 0's margin 0.2
    with pytest.raises(ValueError, match="does not leave a lane"):
        s.set_param_sets([_par(0.4), _par(0.04)], [0, 1, 0, 1])           # controller 1's margin_max 0.04
    assert len(s.calls) == n
    s.set_param_sets([_par(0.3), _par(0.05)], [0, 1, 0, 1])
    s.set_param_sets(None)                                                 # back to the handle's 0.4
    assert np.array_equal(s._bx_min, np.full(4, 0.4))
    with pytest.raises(ValueError):
        s.rollout_finish_laps(np.ones(4, int), np.full(4, 10))            # adaptive rows need the device hand-over
    s.set_lane_margins(None)
    assert s._margins is None and s.lane_margins_of(0) is None and s.calls[-1] == ("margins", 0)
    with pytest.raises(ValueError):
        s.lane_margin_values()
    with pytest.raises(ValueError):
        s.set_lane_margins(None, [0, 0, 0, 0])                             # removal takes no index


def test_driver_refusals_and_start_margin_rows():
    rmc = rollout_mc
    for bad in (([G(3)], np.zeros(8, int)), ([G(1, -1.0)], np.zeros(8, int)), ([G(1, 0.0)], np.ones(8, int)),
                ([G(1, 0.0)], np.zeros(7, int)), ([G(1, 0.4, 0.4)], np.zeros(8, int)), ([G(2, 0.0, 0.5, 0.01)], np.zeros(8, int))):
        with pytest.raises(ValueError):
            rmc.run(batch=8, laps=1, lane_margin_sets=bad)
    with pytest.raises(ValueError, match="does not leave a lane"):
        rmc.run(batch=8, laps=1, param_sets=([_par(0.4), _par(0.1)], np.arange(8) % 2),
                lane_margin_sets=([G(1, 0.1, 0.1)], np.zeros(8, int)))
    row, none = rmc.table_rows(rmc.pack_tables(8, lane_margin_sets=([G(2, 0.0, 0.1, 0.01, 0.0025)], np.zeros(8, int)))[0]), {}
    other = rmc.table_rows(rmc.pack_tables(8, lane_margin_sets=([G(2, 0.0, 0.1, 0.01, 0.0)], np.zeros(8, int)))[0])
    for had, mine in ((row, none), (none, row), (row, other)):
        with pytest.raises(ValueError, match="other lane margins"):
            rmc.check_start_tables(had, mine)
    rmc.check_start_tables(row, row)
    rmc.check_start_tables(none, none)


def _x(ey):
    return np.array([[1.0, 0.0, 0.0, 0.0, 3.0, 0.0], [1.0, 0.0, 0.0, 0.0, 3.1, ey]])


def test_verdict_at_its_edges():
    w = 0.4
    assert not lm.lap_left_lane(_x(w), FX, BX)                             # d == 0 is not a violation
    assert not lm.lap_left_lane(_x(-w), FX, BX)
    assert lm.lap_left_lane(_x(np.nextafter(w, 1.0)), FX, BX)               # one ulp outside
    assert lm.lap_left_lane(_x(-np.nextafter(w, 1.0)), FX, BX)
    for bad in (np.nan, np.inf, -np.inf):
        x = _x(0.0)
        x[1, 2] = bad                                                      # a non-finite entry outside the lane rows too
        assert lm.lap_left_lane(x, FX, BX)
    assert not lm.lap_left_lane(np.zeros((0, 6)), FX, BX)                  # no rows: nothing left the lane


def test_update_rule_at_its_edges():
    r = G(2, 0.01, 0.05, 0.02, 0.0025)
    assert lm.adapt(r, 0.01, True) == 0.01 + 0.02
    assert lm.adapt(r, 0.04, True) == 0.05                                 # clamped at margin_max
    assert lm.adapt(r, 0.05, True) == 0.05
    assert lm.adapt(r, 0.03, False) == 0.03 - 0.0025
    assert lm.adapt(r, 0.011, False) == 0.01                               # clamped at margin0
    assert lm.adapt(r, 0.01, False) == 0.01
    ratchet = G(2, 0.0, 0.1, 0.01, 0.0)                                    # step_down 0: the margin only ratchets up
    m = 0.0
    for left in (True, False, False, True, False):
        m = lm.adapt(ratchet, m, left)
    assert m == 0.01 + 0.01
    assert lm.start(G(0, 0.3)) == 0.0 and lm.start(G(1, 0.03)) == 0.03 and lm.start(r) == 0.01
    assert lm.hand_over(G(1, 0.03), 0.03, _x(1.0), FX, BX) == 0.03        # only mode 2 adapts
    assert lm.hand_over(r, 0.01, _x(1.0), FX, BX) == 0.03
    assert np.array_equal(lm.planning_bx(BX, 0.05), np.array([0.4 - 0.05, 0.4 - 0.05]))
    assert np.array_equal(lm.planning_bx(BX, 0.0), BX)


def test_snapshot_decoder_names_section_39():
    assert len(nat.SNAPSHOT_SLOT_NAMES) == nat.SNAPSHOT_SECTIONS == 40
    assert nat.SNAPSHOT_SLOT_NAMES[39] == "lane_margin"
    assert nat.SNAPSHOT_SLOT_NAMES[:39] == nat.SNAPSHOT_SECTIONS_NAMES
    h = nat.SnapshotHeader()
    h.magic, h.version, h.nsect = nat.SNAPSHOT_MAGIC, nat.SNAPSHOT_VERSION, nat.SNAPSHOT_SECTIONS
    h.sect_off[39], h.sect_bytes[39] = 4096, 8
    d = nat.decode_snapshot_header(bytes(h))
    assert d["sections"] == {"lane_margin": (4096, 8)}
    layout = {f: 0 for f in nat.SNAPSHOT_LAYOUT}
    layout["bytes"] = 0
    assert "lane margin layout" in nat.snapshot_layout_mismatch(d, layout)
    assert nat.snapshot_layout_mismatch(d, dict(layout, lane_margin=1)) is None
