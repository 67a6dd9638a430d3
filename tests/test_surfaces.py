"""CPU tier: track surfaces (lmpc_rollout_set_surfaces) -- the ABI record and its packing, every refusal of make_surface_sets,
BatchedController and rollout_mc.run before any native call or device work, the surface rule of the exact plant and nominal model
(tests/support/plant_exact.py, nominal_model.py: identities, sensitivities against numerical differentiation of the exact plant), and the simulator bound rejecting every known-wrong surface variant."""
import ctypes as C
import math
import os
import re
import sys

import mpmath as mp
import numpy as np
import pytest

from racinglmpc_b200 import _native as nat
from racinglmpc_b200 import reference_params as rp, workloads
from racinglmpc_b200.controller import BatchedController
from racinglmpc_b200.reference_params import SurfaceParams, VehicleParams
import nominal_model as nm
import plant_exact as pe

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
try:
    import rollout_mc  # noqa: E402
finally:
    sys.path.pop(0)

SEG = workloads.track_seg_table()
L = rp.TRACK_LENGTH
TRACK = pe.ExactTrack(SEG, L)
CAR = VehicleParams.reference()
WET = SurfaceParams.from_zones([(2.0, 4.0, 0.75, 0.6), (9.0, 11.5, 1.2, 0.9)])


def test_abi_record_and_symbols():
    assert C.sizeof(nat.SurfaceParams) == 8 + 16 * 4 * 8 == nat.lib().lmpc_sizeof_surface_params()
    assert [getattr(nat.SurfaceParams, f).offset for f in ("nzone", "pad", "zone")] == [0, 4, 8]
    txt = re.sub(r"\s+", " ", open(os.path.join(ROOT, "include", "lmpc_b200.h")).read())
    assert re.search(r"#define LMPC_MAX_ZONES 16\b", txt) and re.search(r"#define LMPC_SCHEDULE_SURFACE 3\b", txt)
    assert ("int lmpc_rollout_set_surfaces(lmpc_handle* h, const lmpc_surface_params* sets, int nsets, const int* set_of_instance);"
            in txt)
    for s in ("lmpc_rollout_set_surfaces", "lmpc_sizeof_surface_params"):
        assert s in nat.exported_symbols() and hasattr(nat.lib(), s)
    assert nat.MAX_ZONES == 16 and nat.LAP_SCHEDULE_TABLES["surface"] == 3


def test_surface_params():
    assert SurfaceParams.dry().zones == () and SurfaceParams.from_zones([(0, 1, 1, 1)]).zones == ((0.0, 1.0, 1.0, 1.0),)
    tr = rp.TrackParams.l_shaped()
    s = SurfaceParams.on_segment(tr, 3, 0.75)
    s0, ln = tr.seg_table[3, 0], tr.seg_table[3, 1]
    assert s.zones == ((s0, float(np.float64(s0) + np.float64(ln)), 0.75, 0.75),)
    assert SurfaceParams.on_segment(tr, 1, 0.5, 0.9).zones[0][2:] == (0.5, 0.9)
    with pytest.raises(Exception):
        s.zones = ()                                                  # frozen


def test_packing_field_by_field():
    zones16 = [(k, k + 0.5, 1.0 + k / 32, 0.5 + k / 64) for k in range(16)]
    rows, idx = nat.make_surface_sets([SurfaceParams.dry(), WET, SurfaceParams.from_zones(zones16)], [2, 0, 1, 1], 4)
    assert [r.nzone for r in rows] == [0, 2, 16] and all(r.pad == 0 for r in rows)
    assert list(rows[1].zone[:8]) == [2.0, 4.0, 0.75, 0.6, 9.0, 11.5, 1.2, 0.9] and all(v == 0 for v in rows[1].zone[8:])
    assert list(rows[2].zone) == [v for z in zones16 for v in z]
    assert idx.dtype == np.int32 and list(idx) == [2, 0, 1, 1]
    # touching zones, mu = 0, a zone past the lap and one beyond 64 laps are all accepted
    nat.make_surface_sets([SurfaceParams.from_zones([(0, 1, 0, 0), (1, 2, 3, 3), (3 * L, 1e9, 1, 1)])], [0, 0], 2)


@pytest.mark.parametrize("zones, what", [
    ([(0, 1, 1, 1)] * 17, "at most"), ([(math.nan, 1, 1, 1)], "finite"), ([(0, math.inf, 1, 1)], "finite"),
    ([(0, 1, math.nan, 1)], "finite"), ([(0, 1, 1, -math.inf)], "finite"), ([(-0.5, 1, 1, 1)], "s_start"),
    ([(1, 1, 1, 1)], "s_start"), ([(2, 1, 1, 1)], "s_start"), ([(0, 1, -0.1, 1)], "mu"), ([(0, 1, 1, -1e-300)], "mu"),
    ([(0, 2, 1, 1), (1, 3, 1, 1)], "overlap"), ([(2, 3, 1, 1), (0, 1, 1, 1)], "overlap"), ([(0, 1, 1)], "zone is")])
def test_refused_rows(zones, what):
    with pytest.raises(ValueError, match=what):
        nat.make_surface_sets([SurfaceParams(tuple(map(tuple, zones)))], np.zeros(2, int), 2)


def test_refused_indices():
    for idx in ([0, 1], [0], [0, 0, 0], [-1, 0], [0.5, 0], None):
        with pytest.raises(ValueError):
            nat.make_surface_sets([WET], idx, 2)
    with pytest.raises(ValueError):
        nat.make_surface_sets([WET] * 3, [0, 1], 2)                   # more rows than controllers
    with pytest.raises(ValueError):
        nat.make_surface_sets([], [0, 0], 2)


class _Recorder:
    """A stand-in library: records every lmpc_* call and returns LMPC_OK."""
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("lmpc_"):
            raise AttributeError(name)
        return lambda *a: self.calls.append(name) or 0


@pytest.fixture
def host(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(nat, "lib", lambda: rec)
    _, _, _, _, Qts, par = rp.lmpc_params(12)
    c = BatchedController(par, 4, np.array([[0.0, 19.3, 0.0]]), 19.3, trToUse=4, numSS_Points=48, numSS_it=4, QterminalSlack=Qts,
                          Tmax=64, ss_cap=6, model_cap=5)
    c.enable_rollout(Tcl=64)
    rec.calls.clear()
    return c, rec


def test_controller_installs_reports_and_refuses(host):
    c, rec = host
    assert c.surface_of(0) is None
    with pytest.raises(ValueError, match="surface table"):
        c.set_lap_schedule("surface", [0])
    with pytest.raises(ValueError, match="overlap"):
        c.set_surfaces([SurfaceParams.from_zones([(0, 2, 1, 1), (1, 3, 1, 1)])], [0, 0, 0, 0])
    with pytest.raises(ValueError, match="index"):
        c.set_surfaces([WET])
    with pytest.raises(ValueError, match="takes no index"):
        c.set_surfaces(None, [0, 0, 0, 0])
    assert rec.calls == []
    c.set_surfaces([SurfaceParams.dry(), WET], [0, 1, 1, 0])
    assert rec.calls == ["lmpc_rollout_set_surfaces"]
    assert c.surface_of(1) == WET and c.surface_of(0) == SurfaceParams.dry()
    # both install orders: a schedule naming row 1 keeps a one-row table and the removal out
    c.set_lap_schedule("surface", [[0, 1]] * 4)
    rec.calls.clear()
    with pytest.raises(ValueError, match="names row 1"):
        c.set_surfaces([WET], [0, 0, 0, 0])
    with pytest.raises(ValueError, match="names row 1"):
        c.set_surfaces(None)
    assert rec.calls == []
    c.set_lap_schedule("surface", None)
    c.set_surfaces(None)
    assert c.surface_of(0) is None and rec.calls[-1] == "lmpc_rollout_set_surfaces"


def _no_device(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(rollout_mc.torch.cuda, "set_device", no_device)
    monkeypatch.setattr(rollout_mc, "BatchedController", no_device)


SS = ([SurfaceParams.dry(), WET], np.zeros(8, np.int32))


@pytest.mark.parametrize("kw, what", [
    (dict(lap_schedules={"surface": [0, 1]}, lap_reports=3), "needs surface_sets"),
    (dict(lap_schedules={"surface": [0, 2]}, surface_sets=SS, lap_reports=3), "out of range"),
    (dict(lap_schedules={"surface": [0, 1]}, surface_sets=SS), "lap_reports"),
    (dict(surface_sets=([SurfaceParams.from_zones([(1, 0, 1, 1)])], np.zeros(8, np.int32))), "s_start"),
    (dict(surface_sets=([WET], np.ones(8, np.int32))), "out of range"),
    (dict(surface_sets=([WET], np.zeros(7, np.int32))), "index")])
def test_run_refusals_before_device_work(kw, what, monkeypatch):
    _no_device(monkeypatch)
    with pytest.raises(ValueError, match=what):
        rollout_mc.run(batch=8, laps=3, **kw)


# ---- the surface rule of the exact plant

X0 = [1.4, 0.05, 0.3, 0.02, 3.9, 0.05]            # crosses s_end = 4.0 of WET's first zone within the period
U0 = [0.1, 0.5]


def _step(x, u=U0, surface=None, vehicle=CAR, variant=None):
    return pe.dyn_model(vehicle, TRACK, x, [0.0] * 6, u, dt=0.1, on_fail="zero", variant=variant, surface=surface)


def _eq(a, b):
    return all(p == q or (mp.isnan(p) and mp.isnan(q)) for p, q in zip(a["x"] + a["x_glob"], b["x"] + b["x_glob"]))


def test_neutral_surfaces_are_the_plant_exactly():
    ones = pe.ExactSurface([(k, k + 0.9, 1.0, 1.0) for k in range(16)])
    for x in (X0, [1.0, 0.0, 0.0, 0.0, L - 0.05, 0.0], [0.8, 0.1, 0.2, 0.0, -0.01, 0.0]):
        ref = _step(x)
        assert _eq(_step(x, surface=pe.ExactSurface([])), ref)
        assert _eq(_step(x, surface=ones), ref)


def test_one_zone_over_the_lap_is_the_scaled_vehicle_exactly():
    for muf, mur in ((0.75, 0.6), (0.0, 1.3), (1.0, 0.0)):
        whole = pe.ExactSurface([(0.0, 2 * L, muf, mur)])
        car = VehicleParams(CAR.m, CAR.lf, CAR.lr, CAR.Iz, muf * CAR.Df, CAR.Cf, CAR.Bf, mur * CAR.Dr, CAR.Cr, CAR.Br)
        for x in (X0, [1.0, 0.0, 0.0, 0.0, L - 0.05, 0.0]):                    # the second crosses the finish line
            assert _eq(_step(x, surface=whole), _step(x, vehicle=car))


def test_zone_margin_and_dry_fallbacks():
    r = _step(X0, surface=pe.ExactSurface(WET.zones))
    assert 0 < r["zone_margin"] < 0.2                                      # 4.0 is crossed inside the period
    wet = pe.ExactSurface([(0.0, 2 * L, 0.5, 0.5)])
    for s in (math.nan, math.inf, 65 * L):                                 # not finite or beyond 64 laps: dry, as the device
        assert _eq(_step([1.0, 0.0, 0.1, 0.0, s, 0.0], surface=wet), _step([1.0, 0.0, 0.1, 0.0, s, 0.0]))
    assert not _eq(_step([1.0, 0.0, 0.1, 0.0, 40 * L + 1.0, 0.0], surface=wet), _step([1.0, 0.0, 0.1, 0.0, 40 * L + 1.0, 0.0]))


# (variant, surface, x): each case puts the variant on the wrong side of the rule within the period
VARIANT_CASES = [
    ("mu_at_start", [(2.0, 4.0, 0.3, 0.3)], X0),                           # the zone ends mid-period
    ("mu_front_only", [(0.0, 2 * L, 1.0, 0.4)], X0),                        # a rear-only zone
    ("zone_closed_end", [(2.0, 3.9, 0.3, 0.3)], X0),                        # s starts exactly at s_end
    ("zone_unwrapped", [(0.5, 3.0, 0.3, 0.3)], [1.4, 0.05, 0.3, 0.02, L + 1.0, 0.05])]   # s beyond the finish line


@pytest.mark.parametrize("variant, zones, x", VARIANT_CASES)
def test_every_known_wrong_variant_is_outside_the_bound(variant, zones, x):
    srf = pe.ExactSurface(zones)
    exact = _step(x, surface=srf)
    wrong = _step(x, surface=srf, variant=variant)
    assert pe.sim_error(pe.to_f64(wrong["x"]), exact["x"]) > 1e3 * pe.SIM_BOUND
    assert pe.sim_error(pe.to_f64(exact["x"]), exact["x"]) <= pe.SIM_BOUND


# ---- the nominal model under a surface

def _f64(rows):
    return [np.array([[float(q) for q in r] for r in rows[0]]), np.array([[float(q) for q in r] for r in rows[1]]),
            np.array([float(q) for q in rows[2]])]


@pytest.mark.parametrize("x", [[1.3, 0.12, 0.6, 0.05, 3.0, 0.1], [2.0, -0.05, -0.4, 0.0, 10.0, -0.2]])
def test_nominal_sensitivities_under_a_surface_equal_numerical_differentiation(x):
    srf = pe.ExactSurface(WET.zones)
    phi, S = nm.phi_sens(CAR, x, U0, surface=srf, track=TRACK)
    assert nm.phi_sens.zone_margin > 0.5                                   # no bound within the period
    phn, Sn = nm.numdiff(CAR, x, U0, surface=srf, track=TRACK)
    assert max(abs(float(a - b)) for a, b in zip(phi, phn)) < 1e-50
    err = max(abs(float(S[r][c] - Sn[r][c])) / (1 + abs(float(S[r][c]))) for r in range(3) for c in range(5))
    assert err < 1e-15, err
    # and the surface is felt: the same state dry gives other rows
    assert nm.deviation(_f64(nm.rows(CAR, x, U0)), nm.rows(CAR, x, U0, surface=srf, track=TRACK)) > 1e3 * nm.NOMINAL_BOUND


def test_nominal_phi_across_a_zone_bound_is_the_plant_step():
    srf = pe.ExactSurface(WET.zones)
    phi, _ = nm.phi_sens(CAR, X0, U0, surface=srf, track=TRACK)
    assert 0 < nm.phi_sens.zone_margin < 0.2
    plant = _step(X0, surface=srf)
    with mp.workdps(pe.DPS):
        assert max(abs(a - b) for a, b in zip(phi, plant["x"][:3])) < mp.mpf(10) ** -50


def test_nominal_one_zone_over_the_lap_is_the_scaled_vehicle():
    muf, mur = 0.75, 0.6
    car = VehicleParams(CAR.m, CAR.lf, CAR.lr, CAR.Iz, muf * CAR.Df, CAR.Cf, CAR.Bf, mur * CAR.Dr, CAR.Cr, CAR.Br)
    got = nm.rows(CAR, X0, U0, surface=pe.ExactSurface([(0.0, 2 * L, muf, mur)]), track=TRACK)
    want = nm.rows(car, X0, U0)
    assert nm.deviation(_f64(got), want) <= 2.0 ** -52
