"""CPU tier: observer priors (lmpc_rollout_set_observer_priors) -- the ABI size and packing of ObserverPriorParams, every refusal
of make_observer_prior_sets before any native call, ObserverPrior's constructors, and the restatement the GPU tests compare
against (tests/support/observer_prior.py): with zero draws its prior is plant_exact's plant state (with or without a
surface) on the curvilinear channels, whatever the global frame, and the rule that picks the car and surface of the step before
a hand-over."""
import ctypes as C
import math

import mpmath as mp
import numpy as np
import pytest

from racinglmpc_b200 import _native as nat
from racinglmpc_b200 import reference_params as rp
from racinglmpc_b200.reference_params import ObserverPrior, VehicleParams
import observer_prior as op
import plant_exact as pe

B = 8
T0 = rp.TrackParams.l_shaped()
L = float(T0.TrackLength)
TRACK = pe.ExactTrack(T0.seg_table, L)
CAR = VehicleParams.reference()


def test_struct_size_and_packing_match_the_library():
    assert C.sizeof(nat.ObserverPriorParams) == 8 + 80 == C.sizeof(nat.PredictionModelParams)
    assert nat.ObserverPriorParams.source.offset == 0 and nat.ObserverPriorParams.pad.offset == 4
    assert nat.ObserverPriorParams.vehicle.offset == 8
    assert nat.lib().lmpc_sizeof_observer_prior_params() == C.sizeof(nat.ObserverPriorParams)


def test_packing():
    wet = VehicleParams.from_friction(0.6)
    rows = [ObserverPrior.plan(), ObserverPrior.car(wet), ObserverPrior.plant()]
    idx = np.arange(B) % 3
    tab, ix = nat.make_observer_prior_sets(rows, idx, B)
    assert len(tab) == 3 and ix.dtype == np.int32 and np.array_equal(ix, idx)
    assert [t.source for t in tab] == [0, 1, 2] and all(t.pad == 0 for t in tab)
    assert [getattr(tab[1].vehicle, f) for f in pe.VEHICLE_FIELDS] == [getattr(wet, f) for f in pe.VEHICLE_FIELDS]
    for k in (0, 2):                                                     # a vehicle that is not read is not packed
        assert all(getattr(tab[k].vehicle, f) == 0.0 for f in pe.VEHICLE_FIELDS)


def _car(**kw):
    d = {f: getattr(CAR, f) for f in pe.VEHICLE_FIELDS}
    d.update(kw)
    return VehicleParams(**d)


@pytest.mark.parametrize("row", [
    ObserverPrior(3), ObserverPrior(-1), ObserverPrior(True), ObserverPrior(1.0), ObserverPrior(np.float64(2)),
    ObserverPrior(None),
    ObserverPrior(1, _car(m=float("nan"))), ObserverPrior(1, _car(Br=float("inf"))), ObserverPrior(1, _car(Df=-float("inf"))),
    ObserverPrior(1, _car(m=0.0)), ObserverPrior(1, _car(lf=-0.1)), ObserverPrior(1, _car(lr=0.0)), ObserverPrior(1, _car(Iz=-1e-300)),
    ObserverPrior(1, _car(Cf=True)), ObserverPrior(1, _car(Bf="1.0"))])
def test_bad_rows_are_refused(row):
    with pytest.raises(ValueError):
        nat.make_observer_prior_sets([ObserverPrior.plan(), row], np.arange(B) % 2, B)


def test_vehicles_of_sources_zero_and_two_are_not_checked():
    bad = _car(m=float("nan"), Iz=0.0)
    tab, _ = nat.make_observer_prior_sets([ObserverPrior(0, bad), ObserverPrior(2, bad)], np.arange(B) % 2, B)
    assert tab[0].source == 0 and tab[1].source == 2


@pytest.mark.parametrize("rows, idx", [
    ([ObserverPrior.plan()], np.ones(B)), ([ObserverPrior.plan()], -np.ones(B)), ([ObserverPrior.plan()], np.zeros(B - 1)),
    ([ObserverPrior.plan()], np.full(B, 0.5)), ([], np.zeros(B)), ([ObserverPrior.plan()] * (B + 1), np.zeros(B)),
    ([ObserverPrior.plan()], None)])
def test_bad_indices_are_refused(rows, idx):
    with pytest.raises(ValueError):
        nat.make_observer_prior_sets(rows, idx, B)


def test_constructors():
    assert ObserverPrior.plan() == ObserverPrior(0) and ObserverPrior.plant().source == 2
    wet = VehicleParams.from_friction(0.6)
    assert ObserverPrior.car(wet) == ObserverPrior(1, wet)


# ---- the restatement --------------------------------------------------------------------------------------------------------
STATES = [(0.8, 0.01, 0.02, 0.05, 1.0, 0.1), (1.2, -0.03, 0.4, -0.1, 3.9, -0.2), (0.5, 0.0, 0.0, 0.0, L - 0.02, 0.0),
          (2.0, 0.1, -0.5, 0.2, 7.3, 0.3)]
INPUTS = [(0.1, 0.5), (-0.25, -1.0), (0.15, 0.3), (0.3, 2.0)]


@pytest.mark.parametrize("k", range(len(STATES)))
def test_prior_without_surface_is_plant_exact_with_zero_draws(k):
    """The prior is plant_exact's plant with its draws zero -- whatever the noise constants, since a zero draw adds nothing -- and
    its curvilinear state does not depend on the global frame."""
    x, u = STATES[k], INPUTS[k]
    got = op.prior_exact(CAR, TRACK, x, u)
    for g in (np.zeros(6), np.array([0.0, 0.0, 0.0, 1.3, -4.0, 2.5])):
        ref = pe.dyn_model(CAR, TRACK, x, g, u, z=(0.0, 0.0, 0.0), noise=rp.NoiseParams.reference(), on_fail="zero")
        assert all(a == b for a, b in zip(got["x"], ref["x"]))
    assert not got["failed"]


@pytest.mark.parametrize("k", range(len(STATES)))
def test_prior_with_surface_is_plant_exact_with_zero_draws(k):
    x, u = STATES[k], INPUTS[k]
    surf = pe.ExactSurface([(0.0, 2.0, 0.6, 0.5), (3.5, 5.0, 1.1, 0.9), (6.0, L, 0.4, 0.4)])
    got = op.prior_exact(CAR, TRACK, x, u, surface=surf)
    ref = pe.dyn_model(CAR, TRACK, x, np.array([0.0, 0.0, 0.0, -0.7, 2.0, 1.0]), u, z=(0.0, 0.0, 0.0), on_fail="zero",
                       surface=surf)
    assert all(a == b for a, b in zip(got["x"], ref["x"]))
    plain = op.prior_exact(CAR, TRACK, x, u)
    assert any(a != b for a, b in zip(got["x"], plain["x"]))          # the zones change the prior


def test_lookup_failure_is_reported():
    got = op.prior_exact(CAR, TRACK, (1.0, 0.0, 0.0, 0.0, -0.5, 0.0), (0.0, 0.0))
    assert got["failed"]


def test_the_car_of_the_step_before_a_hand_over():
    """A source 2 prior reads the rows of lap lap_n - 1 exactly when the previous estimate lies more than half a lap ahead of y
    (the hand-over moved s back by L and lap_n on), and the rows of lap_n otherwise -- also while a hand-over is still pending
    (both s beyond L) and on the lap of the change itself."""
    assert op.back_laps(L - 0.01, 0.03, L) == 1                       # the first step after a hand-over
    assert op.back_laps(L - 0.05, L - 0.01, L) == 0                   # an ordinary step
    assert op.back_laps(L + 0.02, L + 0.06, L) == 0                   # crossed, hand-over not yet committed
    assert op.back_laps(L + 0.02, 0.06, L) == 1                       # committed one step late
    assert op.back_laps(0.5 * L, 0.0, L) == 0                         # exactly half a lap is not a hand-over
    assert op.back_laps(0.03, L - 0.01, L) == 0                       # y ahead of the estimate: never a lap back
    sched = np.array([0, 0, 1, 1, 2])
    assert [op.scheduled_row(sched, n, 0) for n in range(7)] == [0, 0, 1, 1, 2, 2, 2]
    assert [op.scheduled_row(sched, n, 1) for n in range(7)] == [0, 0, 0, 1, 1, 2, 2]
    # lap_n = 2 is the first lap of row 1: its first step still reads row 0, the next one row 1
    assert op.scheduled_row(sched, 2, op.back_laps(L - 0.01, 0.03, L)) == 0
    assert op.scheduled_row(sched, 2, op.back_laps(0.03, 0.07, L)) == 1


def test_blend_of_a_wrapped_prior_is_the_blend_of_the_unwrapped_one():
    y = np.array([1.0, 0.01, 0.02, 0.03, 0.04, 0.05])
    g = (0.5, 0.25, 0.0, 1.0, 0.5, 0.75)
    p = np.array([1.01, 0.0, 0.01, 0.02, L + 0.03, 0.06])
    pw = p.copy()
    pw[4] = max(p[4] - L, 0.0)
    a, ra = op.blend(y, p, g, L)
    b, rb = op.blend(y, pw, g, L)
    assert a.tobytes() == b.tobytes() and not ra and not rb
    assert a[3] == y[3] and a[2] == p[2]
    assert a[0] == p[0] + 0.5 * (y[0] - p[0])
    bad = p.copy()
    bad[3] = math.nan                                                   # gain 1 on epsi: a NaN there is not read
    assert not op.blend(y, bad, g, L)[1]
    bad[1] = math.nan
    x, r = op.blend(y, bad, g, L)
    assert r and x.tobytes() == y.tobytes()


def test_zero_noise_prior_rounds_to_the_fp64_plant():
    """The exact prior rounded to fp64 is what the device plant would produce within SIM_BOUND: a sanity check of units and
    channel order (vx, vy, wz, epsi, s, ey)."""
    x, u = STATES[0], INPUTS[0]
    got = pe.to_f64(op.prior_exact(CAR, TRACK, x, u)["x"])
    assert got[4] > x[4] and abs(got[4] - x[4] - 0.1 * x[0]) < 0.05
    with mp.workdps(pe.DPS):
        assert pe.sim_error(got, op.prior_exact(CAR, TRACK, x, u)["x"]) <= pe.SIM_BOUND
