"""GPU tier: track surfaces (lmpc_rollout_set_surfaces, sim_step_kernel, nominal_model_kernel).

No table, an all-dry table, a 16-zone table with every mu = 1 and a removed table drive the same closed loop bit for bit (PID
lap, seeding, three LMPC laps, lap reports, records), also with an all-learned prediction table; under mode 2 a dry row and
the 16 zones of mu = 1 drive one closed loop.  One zone over the whole lap is the
vehicle row fl(mu_f Df), fl(mu_r Dr), in the closed loop and for mode 2 against mode 1.  The simulator meets the exact
restatement (tests/support/plant_exact.py, nominal_model.py) within SIM_BOUND at zone bounds, per-axle, zero and large mu, across the finish line,
at s = TrackLength, s < 0 and a non-finite s; mode 2 rows 0..2 meet its nominal rows within NOMINAL_BOUND, a period
crossing a zone bound included.  Interleaved rows equal one handle per row (with vehicles and tracks); a surface schedule equals
host re-installs at every change of entry and drives mode 2 the same way; an identity schedule equals none; the PID lap ignores
schedules; retired controllers drive nothing; a snapshot resumes bit for bit; refusals change nothing."""
import math

import mpmath as mp
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import closed_loop as cl                                           # noqa: E402
import nominal_model as nm                                         # noqa: E402
import plant_exact as pe                                           # noqa: E402
from racinglmpc_b200 import reference_params as rp                # noqa: E402
from racinglmpc_b200 import _native as nat                        # noqa: E402
from racinglmpc_b200.reference_params import (PredictionModelParams as P, SurfaceParams as S, TrackParams,   # noqa: E402
                                              VehicleParams as V)

LMPC_E_INVALID = -1
LOOKUP_FAILED = 128
T0 = TrackParams.l_shaped()
L = T0.TrackLength
ET = pe.ExactTrack(T0.seg_table, L)
CAR = V.reference()
ONES16 = S.from_zones([(k * L / 16, (k + 0.5) * L / 16, 1.0, 1.0) for k in range(16)])
WET = S.from_zones([(2.0, 4.0, 0.75, 0.6), (9.0, 11.5, 1.2, 0.9), (L - 0.3, 2 * L, 0.5, 0.5)])
ROWS3 = [S.dry(), S.on_segment(T0, 1, 0.75), WET]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _rmc():
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "benchmarks"))
    try:
        import rollout_mc
    finally:
        sys.path.pop(0)
    return rollout_mc


def _run3(B, **kw):
    """rollout_mc: PID lap, seeding, 3 LMPC laps with lap reports and a capture: (result, final + books, capture)."""
    fin, cap = {}, {}
    out = _rmc().run(batch=B, laps=3, mode="independent", local=0, final=fin, books=fin, capture=cap, lap_reports=3, **kw)
    return out, fin, cap


def _same3(a, b, what):
    (oa, fa, ca), (ob, fb, cb) = a, b
    assert oa["closed_loop_steps"] == ob["closed_loop_steps"] and oa["lap_stats_rank0"] == ob["lap_stats_rank0"], what
    assert sorted(fa) == sorted(fb)
    for k in fa:
        if k == "lap_reports":
            for f in fa[k]:
                assert np.array_equal(fa[k][f], fb[k][f]), (what, k, f)
        else:
            assert np.array_equal(np.asarray(fa[k]), np.asarray(fb[k])), (what, k)
    assert torch.equal(ca["records"], cb["records"]), what


# -------------------------------------------------------------------------------------------------------- 1. neutral tables
@pytest.mark.parametrize("models", [None, "learned"])
def test_neutral_tables_equal_no_table(models):
    _need_gpu()
    B = 64
    pm = None if models is None else ([P.learned()], np.zeros(B, int))
    base = _run3(B, prediction_model_sets=pm)
    for rows in ([S.dry()], [ONES16], [S.dry(), ONES16]):
        got = _run3(B, prediction_model_sets=pm, surface_sets=(rows, np.arange(B) % len(rows)))
        _same3(base, got, rows)
        assert got[0]["per_surface_rank0"][0]["controllers"] > 0
    # a table installed and removed again
    a = cl.run(16)
    b = cl.run(16, hook=lambda c: (c.set_surfaces([WET], np.zeros(16, int)), c.set_surfaces(None)))
    assert a[0] == b[0]
    cl.same(a[1:], b[1:], np.ones(16, bool), "removed table")


def test_mode_2_under_a_dry_and_a_16_zone_mu_1_row_is_one_closed_loop():
    """Both rows run the surface path of the simulator and the nominal model, and neither changes a peak force."""
    _need_gpu()
    B = 64
    pm = ([P.plant(), P.learned()], np.arange(B) % 2)
    a = _run3(B, prediction_model_sets=pm, surface_sets=([S.dry()], np.zeros(B, int)))
    b = _run3(B, prediction_model_sets=pm, surface_sets=([ONES16], np.zeros(B, int)))
    _same3(a, b, "mode 2, dry row vs 16 zones of mu = 1")


def test_neutral_tables_in_mpc_and_lti_steps():
    """Rollout modes 0 (LTV-MPC) and 2 (LTI after sysid) under a 16-zone mu = 1 table equal no table."""
    _need_gpu()
    B = 16

    def drive(hook):
        c = cl.controller(B)
        hook(c)
        c.enable_rollout(Tcl=1024)
        c.rollout_set_state(np.tile(cl.X0, (B, 1)), np.tile(cl.X0, (B, 1)))
        for _ in range(1000):
            c.rollout_pid_step(0.8, seed=4321)
        c.rollout_sysid()
        c.rollout_seed_from_record_dev(copies=4)
        c.rollout_set_state(np.tile(cl.X0, (B, 1)), np.tile(cl.X0, (B, 1)))
        for n in range(60):
            c.rollout_step(seed=99, mode=2 if n % 2 else 0)
        out = dict(c.rollout_state(), **{"r_" + k: v for k, v in c.step_results().items()})
        out["flags"], out["unsolved"] = c.rollout_health()
        c.close()
        return out
    a = drive(lambda c: None)
    b = drive(lambda c: c.set_surfaces([ONES16], np.zeros(B, int)))
    for k in a:
        assert np.array_equal(a[k], b[k]), k


# ------------------------------------------------------------------------------------ 2. a zone over the lap is a vehicle row
def _scaled(car, muf, mur):
    return V(car.m, car.lf, car.lr, car.Iz, muf * car.Df, car.Cf, car.Bf, mur * car.Dr, car.Cr, car.Br)


def test_one_zone_over_the_lap_equals_the_scaled_vehicle_row():
    _need_gpu()
    B = 32
    muf, mur = 0.75, 0.6
    cars = [CAR, V.from_friction(1.0)]
    vidx = np.arange(B) % 2
    a = _run3(B, vehicle_sets=(cars, vidx), surface_sets=([S.from_zones([(0.0, 2 * L, muf, mur)])], np.zeros(B, int)))
    b = _run3(B, vehicle_sets=([_scaled(c, muf, mur) for c in cars], vidx))
    _same3(a, b, "zone over the lap")
    # mode 2 with the zone against mode 1 with the scaled row, in the closed loop
    whole = lambda c: c.set_surfaces([S.from_zones([(0.0, 2 * L, muf, mur)])], np.zeros(B, int))   # noqa: E731
    p = cl.run(B, vehicles=cars, vidx=vidx, hook=lambda c: (whole(c), c.set_prediction_models([P.plant()], np.zeros(B, int))))
    q = cl.run(B, vehicles=cars, vidx=vidx, hook=lambda c: (whole(c), c.set_prediction_models(
        [P(1, _scaled(c_, muf, mur)) for c_ in cars], vidx)))
    assert p[0] == q[0]
    cl.same(p[1:], q[1:], np.ones(B, bool), "mode 2 with the zone vs mode 1 with the row")


# ------------------------------------------------------------------------------------------- 3. the simulator against exact
# (name, state, zones, boundary): the sub-step s of a boundary case may sit within rounding of a segment bound
SIM_CASES = [
    ("crosses s_end", [1.4, 0.05, 0.3, 0.02, 3.9, 0.05], [(2.0, 4.0, 0.4, 0.4)], False),
    ("crosses s_start", [1.4, 0.05, 0.3, 0.02, 1.9, 0.05], [(2.0, 4.0, 0.4, 0.4)], False),
    ("per axle", [1.6, 0.1, 0.6, 0.02, 3.0, 0.05], [(2.0, 4.0, 1.0, 0.3)], False),
    ("front only", [1.6, 0.1, 0.6, 0.02, 3.0, 0.05], [(2.0, 4.0, 0.3, 1.0)], False),
    ("mu zero", [1.6, 0.1, 0.6, 0.02, 3.0, 0.05], [(2.0, 4.0, 0.0, 0.0)], False),
    ("mu large", [1.6, 0.1, 0.6, 0.02, 3.0, 0.05], [(2.0, 4.0, 1.8, 2.5)], False),
    ("two zones in a period", [2.0, 0.0, 0.2, 0.0, 5.95, 0.0], [(5.0, 6.0, 0.5, 0.5), (6.0, 6.2, 1.5, 1.5)], False),
    ("finish line", [1.5, 0.02, 0.1, 0.0, L - 0.06, 0.02], [(0.0, 0.2, 0.4, 0.4), (L - 0.5, L - 0.03, 1.3, 1.3)], True),
    ("s at TrackLength", [1.0, 0.0, 0.1, 0.0, L, 0.0], [(0.0, 2 * L, 0.5, 0.5)], True),
    ("s below 0", [0.7, 0.0, 0.1, 0.0, -1e-3, 0.0], [(0.0, 2 * L, 0.5, 0.5)], True),   # crosses 0 between sub-steps 1 and 2
    ("s not finite", [1.0, 0.0, 0.1, 0.0, math.nan, 0.0], [(0.0, 2 * L, 0.5, 0.5)], True),
    ("s beyond 64 laps", [1.0, 0.0, 0.1, 0.0, 65 * L, 0.0], [(0.0, 2 * L, 0.5, 0.5)], True),
    ("a zone past the lap", [1.4, 0.05, 0.3, 0.02, 3.0, 0.05], [(2 * L, 3 * L, 0.2, 0.2)], False),
    ("16 zones", [1.4, 0.05, 0.3, 0.02, 3.0, 0.05], [(k * 0.3 + 1.0, k * 0.3 + 1.2, 0.5 + k / 16, 1.5 - k / 16) for k in range(16)],
     False)]


def test_simulator_with_zones_meets_the_exact_restatement():
    _need_gpu()
    B = len(SIM_CASES)
    c = cl.controller(B)
    c.enable_rollout(Tcl=16)
    c.set_noise([rp.NoiseParams.scaled(0, 0)], np.zeros(B, int))
    c.set_surfaces([S.from_zones(z) for _, _, z, _ in SIM_CASES], np.arange(B))
    x = np.array([k[1] for k in SIM_CASES])
    c.rollout_set_state(x, x)
    c.rollout_pid_step(0.8, z_pid=np.zeros((B, 2)), z_sim=np.zeros((B, 3)))
    st = c.rollout_state()
    u = np.array([c.rollout_get_lap(b)[1][-1] for b in range(B)])
    flags, _ = c.rollout_health()
    c.close()
    worst = 0.0
    for b, (name, xb, zones, boundary) in enumerate(SIM_CASES):
        r = pe.dyn_model(CAR, ET, xb, xb, u[b], noise=rp.NoiseParams.scaled(0, 0), on_fail="zero", surface=pe.ExactSurface(zones))
        e = max(pe.sim_error(st["x"][b], r["x"]), pe.sim_error(st["xglob"][b], r["x_glob"]))
        assert e <= pe.SIM_BOUND, (name, e)
        assert r["zone_margin"] >= 1e-9, (name, float(r["zone_margin"]))      # every case's own margin to the zone bounds
        assert boundary or r["margin"] >= 1e-9, (name, float(r["margin"]))
        assert bool(flags[b] & LOOKUP_FAILED) == r["failed"], name
        worst = max(worst, e)
    assert flags[[k[0] for k in SIM_CASES].index("s not finite")] & LOOKUP_FAILED
    print("\nsim_step_kernel with zones, %d cases: max |device - exact| / (1 + |exact|) = %.3g (bound %.3g)" % (B, worst, pe.SIM_BOUND))


# --------------------------------------------------------------------------------------- 4. mode 2 rows against exact
def test_mode_2_rows_under_a_surface_meet_the_exact_reference():
    _need_gpu()
    zones = WET.zones
    # stages: zone interiors, a period crossing s_end = 4.0 and s_start = 9.0, the finish line, dry stretches
    xs = np.array([[1.3, 0.12, 0.6, 0.05, 3.0, 0.1], [1.4, 0.05, 0.3, 0.02, 3.9, 0.05], [1.8, -0.05, -0.4, 0.0, 8.9, -0.2],
                   [1.5, 0.02, 0.1, 0.0, L - 0.1, 0.02], [2.0, 0.1, 0.5, 0.03, 6.0, 0.0], [0.8, 0.2, 1.0, -0.05, 10.0, 0.1],
                   [1.0, 0.0, 0.0, 0.0, 1.95, 0.0], [2.5, -0.3, 0.8, 0.1, 11.4, -0.1], [1.2, 0.0, 0.2, 0.0, 15.0, 0.0],
                   [1.6, 0.1, -0.2, 0.0, 3.5, 0.1], [1.1, 0.05, 0.1, 0.0, 0.1, 0.0], [1.4, 0.0, 0.4, 0.0, 12.0, 0.0],
                   [1.4, 0.0, 0.4, 0.0, 12.0, 0.0]])
    us = np.array([[0.2, 0.8], [0.1, 0.5], [-0.1, 0.3], [0.05, 1.0], [0.3, -1.0], [-0.4, 2.0], [0.0, 0.5], [0.5, 10.0],
                   [-0.5, -10.0], [0.2, 0.0], [0.1, 0.2], [0.0, 0.0]])
    B = 2
    c = cl.controller(B)
    c.set_surfaces([S.from_zones(zones), S.dry()], np.array([0, 1]))
    c.set_prediction_models([P.plant()], np.zeros(B, int))
    c.set_state(xLin=np.stack([xs, xs]), uLin=np.stack([us, us]), OldInput=np.zeros((B, 2)), timeStep=np.zeros(B))
    abc, flags = c.identify()
    c.set_surfaces(None)
    dry, _ = c.identify()
    c.close()
    # the dry row and no table both plan on the dry car; nominal_model_kernel<true> is another compilation of the same
    # arithmetic, so the two agree to rounding, not bit for bit
    with np.errstate(invalid="ignore"):
        rel = float(np.max(np.abs(abc[1] - dry[1]) / (1.0 + np.abs(dry[1]))))
    print("\nmode 2, dry row against no table: max |diff| / (1 + |no table|) = %.3e" % rel)
    assert rel <= nm.NOMINAL_BOUND and np.array_equal(dry[0], dry[1])
    srf = pe.ExactSurface(zones)
    worst, crossed = 0.0, 0
    for i in range(12):
        exact = nm.rows(CAR, xs[i], us[i], surface=srf, track=ET)
        crossed += nm.phi_sens.zone_margin < 0.2
        assert nm.phi_sens.zone_margin >= 1e-9, i                          # the stage's own margin to the zone bounds
        dev = nm.from_abc(abc[0, i])
        worst = max(worst, nm.deviation(dev, exact))
        assert np.all(dev[0][:, 3:] == 0)
        pred = dev[0] @ xs[i] + dev[1] @ us[i] + dev[2]
        plant = pe.dyn_model(CAR, ET, xs[i], [0.0] * 6, us[i], z=(0.0, 0.0, 0.0), on_fail="zero", surface=srf)
        with mp.workdps(pe.DPS):
            err = max(float(abs(pe._f(p) - e) / (1 + abs(e))) for p, e in zip(pred, plant["x"][:3]))
        assert err <= nm.NOMINAL_BOUND, (i, err)
        assert np.array_equal(abc[0, i, 18:36], abc[1, i, 18:36]) and np.array_equal(abc[0, i, 51:], abc[1, i, 51:])   # rows 3..5
    assert crossed >= 2
    assert worst <= nm.NOMINAL_BOUND, worst
    print("\nmode 2 rows under a surface: worst %.3e (bound %.3e)" % (worst, nm.NOMINAL_BOUND))


# ---------------------------------------------------------------------------------- 5. interleaved rows, vehicles and tracks
def test_interleaved_rows_equal_one_handle_per_row():
    _need_gpu()
    B = 12
    three = [TrackParams.l_shaped(), TrackParams.goggle(), TrackParams.oval()]
    tidx, vidx, sidx = np.zeros(B, int), np.arange(B) % 2, (np.arange(B) // 2) % 3
    cars = [CAR, V.from_friction(1.0)]
    rows = [S.dry(), S.on_segment(T0, 1, 0.7), WET]
    mix = cl.run(B, vehicles=cars, vidx=vidx, tracks=three[:1], tidx=tidx, hook=lambda c: c.set_surfaces(rows, sidx))
    for k, r in enumerate(rows):
        one = cl.run(B, vehicles=cars, vidx=vidx, tracks=three[:1], tidx=tidx, hook=lambda c: c.set_surfaces([r], np.zeros(B, int)))
        cl.same(mix[1:], one[1:], sidx == k, ("row", k))
    # crossed with three circuits: a surface row is in each controller's own track coordinate
    tidx = np.arange(B) % 3
    mix = cl.run(B, tracks=three, tidx=tidx, hook=lambda c: c.set_surfaces(rows, sidx))
    for k, r in enumerate(rows):
        one = cl.run(B, tracks=three, tidx=tidx, hook=lambda c: c.set_surfaces([r], np.zeros(B, int)))
        cl.same(mix[1:], one[1:], sidx == k, ("tracks, row", k))


# ------------------------------------------------------------------------------------------------------ 6. lap schedules
def _seeded(B, rows, idx, sched=None, models=None, budget=None):
    c = cl.controller(B)
    c.set_surfaces(rows, idx)
    if models is not None:
        c.set_prediction_models(*models)
    c.enable_rollout(Tcl=1024)
    if sched is not None:
        c.set_lap_schedule("surface", sched)
    if budget is not None:
        c.set_lap_budget(budget)
    c.rollout_set_state(np.tile(cl.X0, (B, 1)), np.tile(cl.X0, (B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(cl.X0, (B, 1)), np.tile(cl.X0, (B, 1)))
    return c


def _all(c):
    flags, unsolved = c.rollout_health()
    return dict(c.books(), flags=flags, unsolved=unsolved, **c.rollout_state())


def _equal(a, b, what):
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), (what, k)


@pytest.mark.parametrize("models", [False, True])
def test_schedule_equals_host_reinstalls_at_every_change(models):
    _need_gpu()
    B = 8
    own = np.zeros(B, int)
    # switches at entries 0, 1 and 2, L = 3 shorter than the 4 laps driven, per controller
    sched = np.array([[1, 0, 2], [0, 1, 1], [2, 2, 0], [0, 2, 1], [1, 1, 1], [0, 0, 2], [2, 0, 0], [1, 2, 0]])
    pm = ([P.plant(), P.learned()], np.arange(B) % 2) if models else None
    a = _seeded(B, ROWS3, own, sched=sched, models=pm)
    b = _seeded(B, ROWS3, own, models=pm)
    try:
        entry = None
        for n in range(1, 6000):
            lap_n = b.books()["lap_n"]
            e = sched[np.arange(B), np.minimum(lap_n, sched.shape[1] - 1)]
            if entry is None or not np.array_equal(e, entry):
                entry = e
                b.set_surfaces(ROWS3, e)
            a.rollout_step(seed=1234)
            b.rollout_step(seed=1234)
            a.rollout_commit_laps_dev()
            b.rollout_commit_laps_dev()
            if n % 8 == 0 and a.books()["lap_n"].min() >= 4:
                break
        assert a.books()["lap_n"].min() >= 4
        _equal(_all(a), _all(b), "schedule vs host re-installs")
    finally:
        a.close()
        b.close()


def test_identity_schedule_equals_none_and_the_pid_lap_ignores_schedules():
    _need_gpu()
    B = 8
    idx = np.arange(B) % 3

    def drive(c, laps=2):
        try:
            for n in range(1, 4000):
                c.rollout_step(seed=1234)
                c.rollout_commit_laps_dev()
                if n % 8 == 0 and c.books()["lap_n"].min() >= laps:
                    break
            return _all(c)
        finally:
            c.close()
    a = drive(_seeded(B, ROWS3, idx))
    b = drive(_seeded(B, ROWS3, idx, sched=np.stack([idx, idx], 1)))
    _equal(a, b, "identity schedule")
    # a schedule that names another row from entry 0 on leaves the PID lap (and so the seeded stores) as the index drives it
    c = _seeded(B, ROWS3, idx, sched=(idx + 1) % 3)
    d = _seeded(B, ROWS3, idx)
    try:
        for k in ("ss_time", "md_time", "it"):
            assert np.array_equal(c.books()[k], d.books()[k]), k
        assert np.array_equal(c.rollout_get_lap(0)[0], d.rollout_get_lap(0)[0])
    finally:
        c.close()
        d.close()


def test_retired_controllers_drive_nothing():
    _need_gpu()
    B = 8
    c = _seeded(B, ROWS3, np.arange(B) % 3, sched=np.array([0, 2]), budget=1)
    try:
        for n in range(3000):
            c.rollout_step(seed=1234)
            c.rollout_commit_laps_dev()
            if n % 8 == 0 and c.books()["lap_n"].min() >= 1:
                break
        before = _all(c)
        c.set_surfaces([WET, WET, WET], np.zeros(B, int))
        for _ in range(20):
            c.rollout_step(seed=1234)
            c.rollout_commit_laps_dev()
        _equal(before, _all(c), "retired")
    finally:
        c.close()


def test_snapshot_at_lap_2_resumed_to_5_equals_a_straight_run():
    _need_gpu()
    B = 32
    kw = dict(mode="independent", local=0, lap_reports=5, surface_sets=(ROWS3, np.arange(B) % 3),
              lap_schedules={"surface": [0, 2, 1]})
    rmc = _rmc()
    fa, fb, cap = {}, {}, {}
    rmc.run(batch=B, laps=5, final=fa, books=fa, **kw)
    rmc.run(batch=B, laps=2, capture=cap, **kw)
    out = rmc.run(batch=B, laps=5, final=fb, books=fb, start=cap, **kw)
    assert out["resume_exact"]
    for k in fa:
        if k == "lap_reports":
            for f in fa[k]:
                assert np.array_equal(fa[k][f], fb[k][f]), (k, f)
        else:
            assert np.array_equal(np.asarray(fa[k]), np.asarray(fb[k])), k


# ---------------------------------------------------------------------------------------------------------- 7. refusals
def test_refusals_change_nothing():
    _need_gpu()
    Lb = nat.lib()
    B = 8
    idx = np.arange(B) % 3

    def raw(c, rows, index, n=None):
        arr = (nat.SurfaceParams * max(len(rows), 1))()
        for k, (nz, zs) in enumerate(rows):
            arr[k].nzone = nz
            for j, v in enumerate(zs):
                arr[k].zone[j] = v
        ix = None if index is None else nat.ptr(np.ascontiguousarray(index, np.int32))
        return Lb.lmpc_rollout_set_surfaces(c._h, arr, len(rows) if n is None else n, ix)

    def refuse(c):
        z = np.zeros(B, int)
        for bad in ([(17, [])], [(-1, [])], [(1, [math.nan, 1, 1, 1])], [(1, [0, math.inf, 1, 1])], [(1, [-1, 1, 1, 1])],
                    [(1, [1, 1, 1, 1])], [(1, [0, 1, -0.5, 1])], [(1, [0, 1, 1, -0.5])], [(2, [0, 2, 1, 1, 1, 3, 1, 1])]):
            assert raw(c, bad, z) == LMPC_E_INVALID, bad
        assert raw(c, [(0, [])], np.full(B, 1)) == LMPC_E_INVALID                 # index out of range
        assert raw(c, [(0, [])] * (B + 1), z) == LMPC_E_INVALID                   # more rows than controllers
        assert raw(c, [(0, [])], None) == LMPC_E_INVALID
        # install orders under a schedule naming row 2: a two-row table and the removal
        assert raw(c, [(0, [])] * 2, z) == LMPC_E_INVALID
        assert raw(c, [], None, n=0) == LMPC_E_INVALID
        assert Lb.lmpc_rollout_set_lap_schedule(c._h, 3, 1, nat.ptr(np.full(B, 3, np.int32))) == LMPC_E_INVALID
        assert Lb.lmpc_rollout_set_lap_schedule(c._h, 4, 1, nat.ptr(np.zeros(B, np.int32))) == LMPC_E_INVALID

    def drive(c, hook=None):
        try:
            for n in range(1, 4000):
                if hook is not None and n == 5:
                    hook(c)
                c.rollout_step(seed=1234)
                c.rollout_commit_laps_dev()
                if n % 8 == 0 and c.books()["lap_n"].min() >= 2:
                    break
            return _all(c)
        finally:
            c.close()
    sched = np.array([1, 2])
    a = drive(_seeded(B, ROWS3, idx, sched=sched))
    b = drive(_seeded(B, ROWS3, idx, sched=sched), hook=refuse)
    _equal(a, b, "refusals")
    # a surface schedule without a table: its entries name rows of no table
    c = cl.controller(B)
    try:
        c.enable_rollout(Tcl=64)
        assert Lb.lmpc_rollout_set_lap_schedule(c._h, 3, 1, nat.ptr(np.zeros(B, np.int32))) == LMPC_E_INVALID
    finally:
        c.close()
