"""GPU tier: per-controller prediction models (lmpc_set_prediction_models, nominal_model_kernel).

An all-learned table and a table installed then removed equal no table bit for bit (K1 output and a device closed loop).  The
nominal rows 0..2 meet the exact reference (tests/support/nominal_model.py) within NOMINAL_BOUND at closed-loop and edge states
for three cars, rows 3..5 equal a learned controller's bit for bit, and A x + B u + C matches the noise-free plant step.  Mode 2
equals mode 1 with the plant's row, also under a vehicle lap schedule; interleaved rows equal one handle per row; retired and
shaped controllers identify what they should; a snapshot resumes bit for bit; a non-finite xLin sets flag 1024; refusals change
nothing."""
import ctypes as C

import mpmath as mp
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import closed_loop as cl                                           # noqa: E402
import knn_fixtures as kf                                          # noqa: E402
import nominal_model as nm                                         # noqa: E402
import plant_exact as pe                                           # noqa: E402
from closed_loop import KEYS                                       # noqa: E402
from racinglmpc_b200 import reference_params as rp                # noqa: E402
from racinglmpc_b200 import _native as nat                        # noqa: E402
from racinglmpc_b200.controller import BatchedController          # noqa: E402
from racinglmpc_b200.reference_params import PredictionModelParams as P, VehicleParams as V   # noqa: E402

LMPC_E_INVALID, LMPC_E_STATE = -1, -4
FLAG = nat.FLAG_NOMINAL_NONFINITE


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _fixtures():
    """The closed-loop fixtures of knn_fixtures that share N = 12 and dt = 0.1: (fixture, group) with stored laps and xLin."""
    out = []
    for g in kf.groups():
        if g.N == 12 and g.consts["dt"] == 0.1:
            out += [(fx, g) for fx in g.fixtures if fx.flags == 0]
    return out


def _handle(items, models=None, vehicles=None, shapes=None):
    """A host-driven handle with one controller per (fixture, group) of `items`, its laps and linearisation loaded."""
    Bh = len(items)
    c = BatchedController(rp.mpc_params(12), Bh, kf.TRACK.seg_table(), kf.TRACK.TrackLength,
                          trToUse=max(g.trToUse for _, g in items), Tmax=max(g.Tmax for _, g in items),
                          model_cap=max(g.model_cap for _, g in items), model_kwargs=dict(dt=0.1))
    if shapes is not None:                          # before the first lap is stored
        c.set_shapes(*shapes)
    for b, (fx, _) in enumerate(items):
        for x, u in fx.laps:
            c.model_add_trajectory(b, x, u)
    c.set_state(xLin=np.stack([fx.xLin for fx, _ in items]), uLin=np.stack([fx.uLin for fx, _ in items]),
                OldInput=np.zeros((Bh, 2)), timeStep=np.zeros(Bh))
    if vehicles is not None:
        c.set_vehicles(*vehicles)
    if models is not None:
        c.set_prediction_models(*models)
    return c


def _identify(items, **kw):
    c = _handle(items, **kw)
    try:
        return c.identify()
    finally:
        c.close()


def _edge_states(n):
    """n (xLin, uLin) stages at the edges: small vx, large slip angles, delta at its bounds, a at its bounds."""
    rng = np.random.default_rng(7)
    x = np.zeros((n + 1, 6))
    u = np.zeros((n, 2))
    for i in range(n):
        vx = [0.05, 0.2, 1.0, 2.5, 1.0, 1.5][i % 6]
        vy = [0.0, 0.1, 0.8, -0.6, -0.3, 0.05][i % 6]
        wz = [0.0, 1.5, -2.0, 2.0, 0.5, -0.3][i % 6]
        x[i] = [vx, vy, wz, rng.uniform(-0.2, 0.2), rng.uniform(0.5, 15.0), rng.uniform(-0.3, 0.3)]
        u[i] = [[0.5, -0.5, 0.0, 0.3, -0.5, 0.5][i % 6], [10.0, -10.0, 0.5, -1.0, 0.0, 2.0][i % 6]]
    x[n] = x[n - 1]
    return x, u


CARS = (V.reference(), V(2.5, 0.14, 0.11, 0.03, 9.0, 1.4, 1.2, 8.0, 1.3, 0.9), V(1.6, 0.11, 0.14, 0.02, 5.0, 1.2, 0.9, 5.5, 1.1, 1.1))


# ---------------------------------------------------------------------------------------------------- no change under mode 0
def test_learned_table_and_a_removed_table_equal_no_table():
    _need_gpu()
    items = _fixtures()
    Bh = len(items)
    base = _identify(items)
    for models in (([P.learned()], np.zeros(Bh, int)), ([P.learned(), P(0, CARS[1])], np.arange(Bh) % 2)):
        abc, flags = _identify(items, models=models)
        assert np.array_equal(abc, base[0]) and np.array_equal(flags, base[1])
    c = _handle(items, models=([P.plant()], np.zeros(Bh, int)))
    try:
        c.set_prediction_models(None)
        abc, flags = c.identify()
    finally:
        c.close()
    assert np.array_equal(abc, base[0]) and np.array_equal(flags, base[1])
    # the closed loop (PID lap, seeding, LMPC laps): books, states, health and stored laps
    a = cl.run(16)
    b = cl.run(16, hook=lambda c: c.set_prediction_models([P.learned()], np.zeros(16, int)))
    d = cl.run(16, hook=lambda c: (c.set_prediction_models([P.plant()], np.zeros(16, int)), c.set_prediction_models(None)))
    assert a[0] == b[0] == d[0]
    cl.same(a[1:], b[1:], np.ones(16, bool), "learned table")
    cl.same(a[1:], d[1:], np.ones(16, bool), "removed table")


def _rmc():
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "benchmarks"))
    import rollout_mc
    return rollout_mc


@pytest.mark.parametrize("extra", ["plain", "shapes", "param_sets", "warm"])
def test_learned_table_equals_no_table_over_three_laps_with_reports_and_records(extra):
    """rollout_mc (PID lap, seeding, 3 LMPC laps, lap reports, capture): books, end states, health, solver and lap reports and the
    snapshot records of every controller equal a run without a table, with shapes, parameter sets or warm start as well."""
    _need_gpu()
    rmc = _rmc()
    B = 64
    _, _, _, _, _, par = rp.lmpc_params(12)
    kw = {"plain": {}, "shapes": dict(shape_sets=([(12, 48), (10, 48)], np.arange(B) % 2)),
          "param_sets": dict(param_sets=([par], np.zeros(B, int), None)), "warm": dict(warm=True)}[extra]
    res = []
    for models in (None, ([P.learned()], np.zeros(B, int))):
        fin, cap = {}, {}
        out = rmc.run(batch=B, laps=3, mode="independent", local=0, final=fin, books=fin, capture=cap, lap_reports=3,
                      prediction_model_sets=models, **kw)
        res.append((out, fin, cap))
    (oa, fa, ca), (ob, fb, cb) = res
    assert oa["closed_loop_steps"] == ob["closed_loop_steps"] and oa["lap_stats_rank0"] == ob["lap_stats_rank0"]
    for k in fa:
        if k == "lap_reports":
            for f in fa[k]:
                assert np.array_equal(fa[k][f], fb[k][f]), (k, f)
        else:
            assert np.array_equal(np.asarray(fa[k]), np.asarray(fb[k])), k
    assert torch.equal(ca["records"], cb["records"])
    assert ob["per_prediction_model_rank0"][0]["controllers"] == B


# ------------------------------------------------------------------------------------------------------- nominal vs exact
def _check_rows(abc, flags, xs, us, car, learned_abc=None, stages=None):
    """Every stage: rows 0..2 within the bound of the exact reference, the one-step prediction within the bound of the noise-free
    plant, rows 3..5 equal to the learned controller's, and no K1-only flag."""
    assert int(flags) & (1 | 4 | 32) == 0
    worst = 0.0
    for i in (range(len(us)) if stages is None else stages):
        x, u = xs[i], us[i]
        exact = nm.rows(car, x, u)
        dev = nm.from_abc(abc[i])
        worst = max(worst, nm.deviation(dev, exact))
        # A x + B u + C against the noise-free plant step, rows 0..2
        pred = dev[0] @ x + dev[1] @ u + dev[2]
        phi = nm.phi_sens(car, x, u)[0]
        with mp.workdps(pe.DPS):
            err = max(float(abs(pe._f(p) - e) / (1 + abs(e))) for p, e in zip(pred, phi))
        assert err <= nm.NOMINAL_BOUND, (i, err)
        if learned_abc is not None:
            A, Bm, Cc = kf.abc_split(abc[i])
            lA, lB, lC = kf.abc_split(learned_abc[i])
            assert np.array_equal(kf.rows345(A, Bm, Cc), kf.rows345(lA, lB, lC)), i
    assert worst <= nm.NOMINAL_BOUND, worst
    return worst


def test_nominal_rows_meet_the_exact_reference_at_closed_loop_and_edge_states():
    _need_gpu()
    items = _fixtures()[:6]
    Bh = len(items)
    learned = _identify(items)
    worst = 0.0
    for car in CARS:
        abc, flags = _identify(items, models=([P(1, car)], np.zeros(Bh, int)))
        for b, (fx, _) in enumerate(items):
            worst = max(worst, _check_rows(abc[b], flags[b], fx.xLin, fx.uLin, car, learned[0][b], stages=range(0, 12, 3)))
    # edge states: one controller per car, learned rows 3..5 from a mode 0 controller with the same xLin
    x, u = _edge_states(12)
    fx0, g0 = items[0]
    for car in CARS:
        c = _handle([(fx0, g0), (fx0, g0)], models=([P(1, car), P.learned()], np.array([0, 1])))
        try:
            c.set_state(xLin=np.stack([x, x]), uLin=np.stack([u, u]))
            abc, flags = c.identify()
        finally:
            c.close()
        worst = max(worst, _check_rows(abc[0], flags[0], x, u, car, abc[1]))
    print("nominal rows 0..2: worst |dev - exact| / (1 + |exact|) = %.3e (bound %.3e)" % (worst, nm.NOMINAL_BOUND))


# --------------------------------------------------------------------------------------------------- mode 2 and interleaving
def test_mode_2_equals_mode_1_with_the_plant_row_and_interleaved_rows_equal_one_handle_per_row():
    _need_gpu()
    items = _fixtures()[:8]
    Bh = len(items)
    vidx = np.arange(Bh) % 3
    m2, f2 = _identify(items, vehicles=(list(CARS), vidx), models=([P.plant()], np.zeros(Bh, int)))
    for k, car in enumerate(CARS):
        m1, f1 = _identify(items, models=([P(1, car)], np.zeros(Bh, int)))
        sel = vidx == k
        assert np.array_equal(m2[sel], m1[sel]) and np.array_equal(f2[sel], f1[sel]), k
    rows = [P.learned(), P(1, CARS[1]), P.plant(), P(1, CARS[2])]
    ridx = np.arange(Bh) % 4
    mix, fmix = _identify(items, vehicles=(list(CARS), vidx), models=(rows, ridx))
    for k, r in enumerate(rows):
        one, fone = _identify(items, vehicles=(list(CARS), vidx), models=([r], np.zeros(Bh, int)))
        sel = ridx == k
        assert np.array_equal(mix[sel], one[sel]) and np.array_equal(fmix[sel], fone[sel]), k


def test_shaped_handle_identifies_stages_below_its_horizon_only():
    """Stages i < N_b equal an unshaped handle's; the nominal kernel leaves the stages past N_b as K1 left them."""
    _need_gpu()
    items = _fixtures()[:4]
    Bh = len(items)
    c = _handle(items, shapes=([(8, 0), (12, 0)], np.arange(Bh) % 2))
    try:
        before, _ = c.identify()
        c.set_prediction_models([P.plant()], np.zeros(Bh, int))
        abc, flags = c.identify()
    finally:
        c.close()
    full, fflags = _identify(items, models=([P.plant()], np.zeros(Bh, int)))
    assert np.array_equal(flags, fflags)
    for b in range(Bh):
        Nb = 8 if b % 2 == 0 else 12
        assert np.array_equal(abc[b, :Nb], full[b, :Nb]), b
        assert np.array_equal(abc[b, Nb:], before[b, Nb:]), b


# -------------------------------------------------------------------------------------------------------- closed loop
def _seeded(B, hook=None, vehicles=None, schedule=None):
    c = cl.controller(B)
    if vehicles is not None:
        c.set_vehicles(*vehicles)
    if hook is not None:
        hook(c)
    c.enable_rollout(Tcl=1024)
    if schedule is not None:
        c.set_lap_schedule("vehicle", schedule)
    c.rollout_set_state(np.tile(cl.X0, (B, 1)), np.tile(cl.X0, (B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(cl.X0, (B, 1)), np.tile(cl.X0, (B, 1)))
    return c


def test_mode_2_follows_the_vehicle_lap_schedule_at_each_controllers_hand_over():
    """Mode 2 under a vehicle lap schedule equals a handle whose host re-installs mode 1 rows (each controller's scheduled car)
    whenever a controller's schedule entry changes."""
    _need_gpu()
    B = 8
    cars = [CARS[0], V.from_friction(0.6)]
    sched = np.array([0, 1, 0])
    a = _seeded(B, hook=lambda c: c.set_prediction_models([P.plant()], np.zeros(B, int)), vehicles=(cars, np.zeros(B, int)),
                schedule=sched)
    b = _seeded(B, hook=lambda c: c.set_prediction_models([P(1, cars[0])], np.zeros(B, int)), vehicles=(cars, np.zeros(B, int)),
                schedule=sched)
    try:
        entry = np.zeros(B, int)
        for n in range(1, 4000):
            a.rollout_step(seed=1234)
            b.rollout_step(seed=1234)
            a.rollout_commit_laps_dev()
            b.rollout_commit_laps_dev()
            lap_n = b.books()["lap_n"]
            e = sched[np.minimum(lap_n, len(sched) - 1)]
            if not np.array_equal(e, entry):
                entry = e
                b.set_prediction_models([P(1, cars[0]), P(1, cars[1])], e.astype(int))
            if lap_n.min() >= 3:
                break
        assert b.books()["lap_n"].min() >= 3
        fa, ua = a.rollout_health()
        fb, ub = b.rollout_health()
        assert np.array_equal(fa, fb) and np.array_equal(ua, ub)
        ba, bb = a.books(), b.books()
        for k in ba:
            assert np.array_equal(np.asarray(ba[k]), np.asarray(bb[k])), k
        sa, sb = a.rollout_state(), b.rollout_state()
        for k in sa:
            assert np.array_equal(sa[k], sb[k]), k
    finally:
        a.close()
        b.close()


def test_snapshot_under_a_table_resumes_bit_for_bit():
    _need_gpu()
    B = 8
    rows, idx = [P.learned(), P.plant(), P(1, CARS[1])], np.arange(B) % 3
    hook = lambda c: c.set_prediction_models(rows, idx)              # noqa: E731

    def run(split):
        c = _seeded(B, hook=hook)
        try:
            for n in range(1, 3000):
                c.rollout_step(seed=1234)
                c.rollout_commit_laps_dev()
                if split and n == 200:
                    rec, clock = c.snapshot(), c.rollout_clock
                    d = cl.controller(B)
                    hook(d)
                    d.enable_rollout(Tcl=1024)
                    d.restore(rec)
                    d.rollout_clock = clock
                    c.close()
                    c = d
                if n % 8 == 0 and c.books()["lap_n"].min() >= 2:
                    break
            flags, unsolved = c.rollout_health()
            return dict(c.books(), flags=flags, unsolved=unsolved, **c.rollout_state())
        finally:
            c.close()
    a, b = run(False), run(True)
    for key in KEYS:
        assert np.array_equal(a[key], b[key]), key


def test_non_finite_xlin_sets_flag_1024_and_retired_controllers_identify_nothing():
    _need_gpu()
    items = _fixtures()[:4]
    Bh = len(items)
    c = _handle(items, models=([P.plant(), P.learned()], np.array([0, 0, 0, 1])))
    try:
        st = c.get_state()
        x = st["xLin"].copy()
        x[1, 3, 0] = np.nan
        c.set_state(xLin=x)
        abc, flags = c.identify()
    finally:
        c.close()
    assert int(flags[1]) & FLAG and not int(flags[1]) & (1 | 4 | 32)
    assert int(flags[0]) & FLAG == 0 and int(flags[2]) & FLAG == 0 and int(flags[3]) & FLAG == 0
    # retired controllers identify nothing: once every controller has retired at its lap budget, a table that would change every
    # stage model (another car) leaves the models and the step flags as they were
    B = 8
    c = _seeded(B, hook=lambda c: c.set_prediction_models([P.plant()], np.zeros(B, int)))
    try:
        c.set_lap_budget(1)
        for n in range(3000):
            c.rollout_step(seed=1234)
            c.rollout_commit_laps_dev()
            if n % 8 == 0 and c.books()["lap_n"].min() >= 1:
                break
        assert c.books()["lap_n"].min() >= 1
        L = nat.lib()

        def abc():
            a = np.zeros((B, 12, 54))
            nat.check(L.lmpc_read_buffer(c._h, b"abc", 0, nat.ptr(a), a.nbytes))
            return a
        a0 = abc()
        c.set_prediction_models([P(1, CARS[1])], np.zeros(B, int))
        for _ in range(20):
            c.rollout_step(seed=1234)
            assert not c.step_results()["flags"].any()
        assert np.array_equal(abc(), a0)
    finally:
        c.close()


def test_refusals_change_nothing():
    _need_gpu()
    L = nat.lib()
    items = _fixtures()[:4]
    Bh = len(items)
    c = _handle(items, models=([P.plant(), P(1, CARS[1])], np.array([0, 1, 0, 1])))
    try:
        before = c.identify()

        def raw(rows, idx):
            arr = (nat.PredictionModelParams * len(rows))()
            for k, (mode, vals) in enumerate(rows):
                arr[k] = nat.PredictionModelParams(mode, 0, nat.VehicleParams(*vals))
            return L.lmpc_set_prediction_models(c._h, arr, len(rows), nat.ptr(np.ascontiguousarray(idx, np.int32)))
        ref = [getattr(CARS[0], f) for f in nat.VEHICLE_FIELDS]
        zero = np.zeros(Bh)
        for bad in ([(3, ref)], [(-1, ref)], [(1, [0.0] + ref[1:])], [(1, ref[:1] + [-0.1] + ref[2:])],
                    [(1, ref[:3] + [0.0] + ref[4:])], [(2, ref[:5] + [float("nan")] + ref[6:])],
                    [(0, ref[:9] + [float("inf")])]):
            assert raw(bad, zero) == LMPC_E_INVALID, bad
        assert raw([(1, ref)], np.full(Bh, 1)) == LMPC_E_INVALID              # index out of range
        assert L.lmpc_set_prediction_models(c._h, None, 1, None) == LMPC_E_INVALID
        after = c.identify()                                                  # right after the refused calls
        assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
        with pytest.raises(ValueError):
            c.set_prediction_models([P(3)], np.zeros(Bh, int))
        assert c.prediction_models_of(0)[0] == 2 and c.prediction_models_of(1) == (1, CARS[1])
        after = c.identify()
        assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
        assert raw([(2, [0.0] * 10)], zero) == 0                              # modes 0 and 2 do not read the vehicle
    finally:
        c.close()
    # no store: LMPC_E_STATE
    h = C.c_void_p()
    p = nat.make_params(rp.mpc_params(12), 0, 0)
    nat.check(L.lmpc_create(C.byref(p), 2, 0, C.byref(h)))
    try:
        arr = (nat.PredictionModelParams * 1)()
        assert L.lmpc_set_prediction_models(h, arr, 1, nat.ptr(np.zeros(2, np.int32))) == LMPC_E_STATE
    finally:
        L.lmpc_destroy(h)
