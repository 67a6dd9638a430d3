"""GPU tier: observer priors of the device closed loop (lmpc_rollout_set_observer_priors).

No prior table, a table of source 0 rows and a prior table without an observer table equal one another bit for bit, nsets == 0
reverts, refused calls change nothing and no launch is added.  With process noise off and no sensor, the plant prior (source 2)
is the plant state bit for bit at every step with a prior, across finish lines, with and without surfaces, and under vehicle and
surface lap schedules that change at a lap, so x_hat == x; source 1 with the plant's own car is source 2.  Under noise x_prior
is the exact one-period map (tests/support/observer_prior.py) within SIM_BOUND and x_est the blend of it.  The edges (non-finite
inputs, PID and LTI steps, retired and shaped controllers), batches against one handle per row, and snapshots."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                # noqa: E402
from racinglmpc_b200 import _native as nat                        # noqa: E402
from racinglmpc_b200.reference_params import (MeasurementParams, NoiseParams, ObserverParams, ObserverPrior,   # noqa: E402
                                              SurfaceParams, VehicleParams)
import closed_loop as cl                                          # noqa: E402
import observer_prior as op                                       # noqa: E402
import plant_exact as pe                                          # noqa: E402
from closed_loop import N, X0                                     # noqa: E402

LMPC_E_INVALID, LMPC_E_STATE = -1, -4
BASE = MeasurementParams((0.01, 0.01, 0.01, 0.005, 0.01, 0.01), (0.05, 0.05, 0.05, 0.025, 0.05, 0.05))
T0 = rp.TrackParams.l_shaped()
L = float(T0.TrackLength)
TRACK = pe.ExactTrack(T0.seg_table, L)
CAR = VehicleParams.reference()
HALF = ObserverParams.uniform(0.5)
WET = SurfaceParams.from_zones([(2.0, 4.0, 0.7, 0.6), (6.0, 8.0, 0.9, 0.8)])
QUIET = NoiseParams.scaled(0.0, 0.0)


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _read(c, name, shape, dtype=np.float64):
    out = np.zeros(shape, dtype)
    nat.check(c._lib.lmpc_read_buffer(c._h, name.encode(), 0, nat.ptr(out), out.nbytes))
    return out


def _controller(Bs, obs=(HALF,), oidx=None, pri=None, pidx=None, meas=(BASE,), midx=None, noise=None, streams=None,
                surf=None, sidx=None, veh=None, vidx=None, reports=True):
    c = cl.controller(Bs)
    c.enable_rollout(Tcl=1024)
    if reports:
        c.enable_lap_reports(64)
    z = np.zeros(Bs, np.int32)
    if streams is not None:
        c.set_noise_streams(streams)
    if noise is not None:
        c.set_noise([noise], z)
    if veh is not None:
        c.set_vehicles(veh, z if vidx is None else vidx)
    if surf is not None:
        c.set_surfaces(surf, z if sidx is None else sidx)
    if meas is not None:
        c.set_measurement_noise(list(meas), z if midx is None else midx)
    if obs is not None:
        c.set_observers(list(obs), z if oidx is None else oidx)
    if pri is not None:
        c.set_observer_priors(list(pri), z if pidx is None else pidx)
    c.rollout_set_state(np.tile(X0, (Bs, 1)), np.tile(X0, (Bs, 1)))
    return c


def _pid_lap_and_seed(c):
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))


def _drive(c, steps, seed=1234):
    for _ in range(steps):
        c.rollout_step(seed=seed)
        c.rollout_commit_laps_dev()


def _result(c, records=True):
    out = dict(books=c.books(), state=c.rollout_state(), health=c.rollout_health(), solver=c.step_results(),
               reports=c.lap_reports())
    if records:
        out["records"] = c.snapshot().cpu().numpy()
    return out


def _same(a, b, sel, what, path=()):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), (what, path)
        for k in a:
            _same(a[k], b[k], sel, what, path + (k,))
    elif isinstance(a, (tuple, list)):
        for k, (p, q) in enumerate(zip(a, b)):
            _same(p, q, sel, what, path + (k,))
    else:
        p, q = np.asarray(a), np.asarray(b)
        if p.ndim and p.shape[0] == sel.shape[0]:
            p, q = p[sel], q[sel]
        assert p.shape == q.shape and p.tobytes() == q.tobytes(), (what, path)


def _launches(c, f):
    l0 = c.kernel_launches
    f()
    return c.kernel_launches - l0


# ---- 1. identity ------------------------------------------------------------------------------------------------------------
def _reject(c):
    Lb = nat.lib()
    idx = np.arange(c.B, dtype=np.int32) % 3
    good, _ = nat.make_observer_prior_sets([ObserverPrior.plan(), ObserverPrior.car(CAR), ObserverPrior.plant()], idx, c.B)

    def copy_of(mod):
        t = (nat.ObserverPriorParams * 3)()
        C.memmove(t, good, C.sizeof(t))
        mod(t)
        return t
    bad = [copy_of(lambda t: setattr(t[0], "source", 3)), copy_of(lambda t: setattr(t[2], "source", -1)),
           copy_of(lambda t: setattr(t[1].vehicle, "m", float("nan"))), copy_of(lambda t: setattr(t[1].vehicle, "Iz", 0.0)),
           copy_of(lambda t: setattr(t[1].vehicle, "Br", float("inf"))), copy_of(lambda t: setattr(t[1].vehicle, "lf", -1.0))]
    cases = [(t, 3, idx) for t in bad] + [(good, 3, np.full(c.B, 3, np.int32)), (good, 3, np.full(c.B, -1, np.int32)),
                                          (good, 0, idx), (None, 3, idx), (good, 3, None), (good, -1, idx)]
    for tab, n, ix in cases:
        assert Lb.lmpc_rollout_set_observer_priors(c._h, tab, n, nat.ptr(ix) if ix is not None else None) == LMPC_E_INVALID


def test_needs_the_closed_loop_and_adds_no_launch():
    _need_gpu()
    Bs = 8
    c = cl.controller(Bs)
    ok, ix = nat.make_observer_prior_sets([ObserverPrior.plant()], np.zeros(Bs), Bs)
    assert nat.lib().lmpc_rollout_set_observer_priors(c._h, ok, 1, nat.ptr(ix)) == LMPC_E_STATE
    c.enable_rollout(Tcl=1024)
    c.rollout_set_state(np.tile(X0, (Bs, 1)), np.tile(X0, (Bs, 1)))
    _pid_lap_and_seed(c)
    z = np.zeros(Bs)
    counts = {}
    for obs in (False, True):
        c.set_observers([HALF] if obs else None, z if obs else None)
        for pri in (False, True):
            c.set_observer_priors([ObserverPrior.plant()] if pri else None, z if pri else None)
            for mode in (1, 0, 2):
                counts[(obs, pri, mode)] = _launches(c, lambda: c.rollout_step(seed=5, mode=mode))
            counts[(obs, pri, "pid")] = _launches(c, lambda: c.rollout_pid_step(0.8, seed=1))
    for k in (1, 0, 2, "pid"):
        assert counts[(False, True, k)] == counts[(False, False, k)], k
        assert counts[(True, True, k)] == counts[(True, False, k)] == counts[(False, False, k)] + 1, k
    with pytest.raises(ValueError):
        c.set_observer_priors(None, z)
    with pytest.raises(ValueError):
        c.set_observer_priors([ObserverPrior.plant()])
    with pytest.raises(ValueError):
        c.set_observer_priors([ObserverPrior(1, VehicleParams.from_friction(0.8, m=0.0))], z)
    c.close()


@pytest.fixture(scope="module")
def identity_runs():
    """Shared streams, base measurement noise, observer rows of uniform 0.5 and from_noise gains: no prior table, source 0 rows
    (installed, then refused calls), a plant prior table removed by nsets == 0, and a prior table without an observer table
    (against no tables at all)."""
    _need_gpu()
    Bs = 32
    streams = np.arange(Bs) // 2
    obs = [HALF, ObserverParams.from_noise(0.01, 0.03)]
    oidx = np.arange(Bs) % 2
    out = {}
    for name in ("none", "plan", "reverted", "bare", "prior_only"):
        kw = dict(obs=obs, oidx=oidx, streams=streams)
        if name == "plan":
            kw.update(pri=[ObserverPrior.plan()])
        elif name == "reverted":
            kw.update(pri=[ObserverPrior.plant(), ObserverPrior.car(VehicleParams.from_friction(0.5))], pidx=oidx)
        elif name == "bare":
            kw.update(obs=None)
        elif name == "prior_only":
            kw.update(obs=None, pri=[ObserverPrior.plant()])
        c = _controller(Bs, **kw)
        if name == "plan":
            _reject(c)
        if name == "reverted":
            c.set_observer_priors(None)
        _pid_lap_and_seed(c)
        out[name + "_launch"] = _launches(c, lambda: c.rollout_step(seed=1234))
        c.rollout_commit_laps_dev()
        _drive(c, 349)
        out[name] = _result(c)
        c.close()
    return out


def test_source_zero_and_removed_tables_equal_no_table(identity_runs):
    r = identity_runs
    sel = np.ones(32, bool)
    assert r["none"]["books"]["lap_n"].max() >= 1
    for name in ("plan", "reverted"):
        assert r[name + "_launch"] == r["none_launch"]
        _same(r[name], r["none"], sel, name)
    assert r["prior_only_launch"] == r["bare_launch"]
    _same(r["prior_only"], r["bare"], sel, "prior table without observers")


# ---- 2. exactness against the plant -----------------------------------------------------------------------------------------
def _exact_run(Bs, steps, **kw):
    """Process noise off, no sensor, observer 0.5 everywhere: per LMPC step, (has_pred before, plant state before, x_prior,
    x_est, lap_n before), for `steps` steps or until 20 steps after every controller has handed over a lap."""
    c = _controller(Bs, meas=None, noise=QUIET, **kw)
    _pid_lap_and_seed(c)
    rows = []
    after = 0
    for _ in range(steps):
        if c.books()["lap_n"].min() >= 1:
            after += 1
            if after > 20:
                break
        hp = _read(c, "has_pred", Bs, np.int32)
        x = c.rollout_state()["x"].copy()
        lap_n = c.books()["lap_n"].copy()
        c.rollout_step(seed=1234)
        rows.append((hp, x, _read(c, "x_prior", (Bs, 6)), _read(c, "x_est", (Bs, 6)), lap_n))
        c.rollout_commit_laps_dev()
    return c, rows


def _check_exact(rows, Bs, cross=True):
    used = crossed = 0
    for k, (hp, x, xq, xe, lap_n) in enumerate(rows):
        on = hp == 1
        assert xq[on].tobytes() == x[on].tobytes(), k
        assert np.all(np.isnan(xq[~on])), k
        assert xe.tobytes() == x.tobytes(), k
        used += int(on.sum())
        if k:
            crossed += int(np.sum(on & (lap_n > rows[k - 1][4])))
    assert used > 0 and (crossed > 0 or not cross), (used, crossed)


@pytest.mark.parametrize("surface", [False, True])
def test_plant_prior_is_the_plant_state(surface):
    """Without a surface the run crosses the finish line; with WET from the start the first LMPC lap is slow, so the crossing
    under a surface is the schedule test's (below)."""
    _need_gpu()
    Bs = 8
    c, rows = _exact_run(Bs, 400, pri=[ObserverPrior.plant()], surf=[WET] if surface else None)
    _check_exact(rows, Bs, cross=not surface)
    c.close()


def test_plant_prior_follows_lap_schedules_across_the_change():
    """Vehicle and surface tables with two rows, schedules [0, 1]: lap 0 on a dry car without zones, lap 1 on with a wet car and
    zones.  The prior stays the plant state at the first step after the hand-over too (it reads the rows of lap 0 there)."""
    _need_gpu()
    Bs = 8
    c = _controller(Bs, meas=None, noise=QUIET, pri=[ObserverPrior.plant()], surf=[SurfaceParams.dry(), WET],
                    veh=[CAR, VehicleParams.from_friction(0.55)])
    c.set_lap_schedule("vehicle", [0, 1])
    c.set_lap_schedule("surface", [0, 1])
    _pid_lap_and_seed(c)
    rows = []
    for _ in range(400):
        hp = _read(c, "has_pred", Bs, np.int32)
        x = c.rollout_state()["x"].copy()
        lap_n = c.books()["lap_n"].copy()
        c.rollout_step(seed=1234)
        rows.append((hp, x, _read(c, "x_prior", (Bs, 6)), _read(c, "x_est", (Bs, 6)), lap_n))
        c.rollout_commit_laps_dev()
    _check_exact(rows, Bs)
    firsts = sum(int(np.sum((r[0] == 1) & (r[4] == 1) & (rows[k - 1][4] == 0))) for k, r in enumerate(rows) if k)
    assert firsts > 0                                                 # the step right after the change had a prior
    c.close()


def test_believed_plant_car_equals_plant_prior():
    _need_gpu()
    Bs = 8
    a = _controller(Bs, pri=[ObserverPrior.car(CAR)])
    b = _controller(Bs, pri=[ObserverPrior.plant()])
    for c in (a, b):
        _pid_lap_and_seed(c)
    for k in range(300):
        for c in (a, b):
            c.rollout_step(seed=1234)
        assert _read(a, "x_prior", (Bs, 6)).tobytes() == _read(b, "x_prior", (Bs, 6)).tobytes(), k
        assert _read(a, "x_est", (Bs, 6)).tobytes() == _read(b, "x_est", (Bs, 6)).tobytes(), k
        for c in (a, b):
            c.rollout_commit_laps_dev()
    _same(_result(a), _result(b), np.ones(Bs, bool), "source 1 with the plant's car")
    a.close()
    b.close()


# ---- 3. under process and measurement noise ---------------------------------------------------------------------------------
def test_prior_is_the_exact_map_and_x_est_its_blend_under_noise():
    _need_gpu()
    Bs = 8
    gains = [HALF, ObserverParams.gains(0.2, 0.7, 1.0, 0.0, 0.3, 0.9)]
    idx = np.arange(Bs) % 2
    c = _controller(Bs, obs=gains, oidx=idx, pri=[ObserverPrior.plant()], surf=[WET], meas=(MeasurementParams.scaled(3, BASE),))
    _pid_lap_and_seed(c)
    sfc = pe.ExactSurface(WET.zones)
    worst, n, resets = 0.0, 0, 0
    for k in range(260):
        hp = _read(c, "has_pred", Bs, np.int32)
        prev = _read(c, "xPredPrev", (Bs, N + 1, 6))[:, 0]
        u = _read(c, "OldInput", (Bs, 2))
        c.rollout_step(seed=1234)
        y, xq, xe = _read(c, "x_meas", (Bs, 6)), _read(c, "x_prior", (Bs, 6)), _read(c, "x_est", (Bs, 6))
        flagged = (c.step_results()["flags"] & nat.FLAG_OBSERVER_RESET) != 0
        for b in range(Bs):
            if not hp[b]:
                assert np.all(np.isnan(xq[b])) and xe[b].tobytes() == y[b].tobytes()
                continue
            if flagged[b]:                # a noisy estimate with s < 0: the prior's first curvature lookup fails
                assert prev[b][4] < 0 and xe[b].tobytes() == y[b].tobytes(), (k, b)
                assert op.prior_exact(CAR, TRACK, prev[b], u[b], surface=sfc)["failed"]
                resets += 1
                continue
            want, reset = op.blend(y[b], xq[b], gains[idx[b]].gain, L)
            assert not reset and xe[b].tobytes() == want.tobytes(), (k, b)
            if k % 13 == 0:
                ex = op.prior_exact(CAR, TRACK, prev[b], u[b], surface=sfc)
                exs = list(ex["x"])
                if op.back_laps(prev[b][4], y[b][4], L):                    # the prior was wrapped back by L
                    exs[4] = exs[4] - L
                e = pe.sim_error(xq[b], exs)
                assert e <= pe.SIM_BOUND, (k, b, e)
                worst, n = max(worst, e), n + 1
        c.rollout_commit_laps_dev()
    assert n > 20
    print("\nx_prior against the exact map, %d cases: max error %.3g (bound %.3g); %d resets at s < 0" % (n, worst, pe.SIM_BOUND,
                                                                                                      resets))
    c.close()


# ---- 4. edges ---------------------------------------------------------------------------------------------------------------
EDGE_OBS = [ObserverParams.off(), HALF, ObserverParams.uniform(1.0), HALF]
EDGE_PRI = [ObserverPrior.plant(), ObserverPrior.plant(), ObserverPrior.plant(), ObserverPrior.plan()]


def test_a_non_finite_input_resets_and_flags():
    """vx of every xPredPrev[0] (the prior's state input) set to NaN: the plant-prior rows with gains 0.5 read y and flag the step,
    the health word and that lap's report; mode 0, all-ones and own-plan rows do not.  Then a NaN OldInput (the prior's input
    argument) resets the same rows in the step flags."""
    _need_gpu()
    Bs = 16
    idx = np.arange(Bs) % 4
    c = _controller(Bs, obs=EDGE_OBS, oidx=idx, pri=EDGE_PRI, pidx=idx)
    _pid_lap_and_seed(c)
    _drive(c, 20)
    xpp = _read(c, "xPredPrev", (Bs, N + 1, 6))
    hp = _read(c, "has_pred", Bs, np.int32)
    assert np.all(hp == 1)
    xpp[:, 0, 0] = np.nan
    c.set_state(xPred=xpp, has_pred=hp)
    lap_n0 = c.books()["lap_n"].copy()
    c.rollout_step(seed=1234)
    y, xe = _read(c, "x_meas", (Bs, 6)), _read(c, "x_est", (Bs, 6))
    reset = idx == 1                                                  # plant prior, gains 0.5
    assert np.array_equal(xe[reset], y[reset]) and np.all(np.isfinite(xe))
    flags = c.step_results()["flags"]
    assert np.array_equal((flags & nat.FLAG_OBSERVER_RESET) != 0, reset)
    c.rollout_commit_laps_dev()
    assert np.array_equal((c.rollout_health()[0] & nat.FLAG_OBSERVER_RESET) != 0, reset)
    for _ in range(600):
        c.rollout_step(seed=1234)
        c.rollout_commit_laps_dev()
        if (c.books()["lap_n"] > lap_n0).all():
            break
    rep = c.lap_reports()
    assert np.all(rep["n"] > lap_n0)
    got = np.array([(rep["flags"][b, lap_n0[b]] & nat.FLAG_OBSERVER_RESET) != 0 for b in range(Bs)])
    assert np.array_equal(got, reset)
    u = _read(c, "OldInput", (Bs, 2))
    u[:, 1] = np.nan
    c.set_state(OldInput=u)
    c.rollout_step(seed=1234)
    y, xe = _read(c, "x_meas", (Bs, 6)), _read(c, "x_est", (Bs, 6))
    assert np.array_equal((c.step_results()["flags"] & nat.FLAG_OBSERVER_RESET) != 0, reset)
    assert np.array_equal(xe[reset], y[reset])
    c.close()


def test_pid_and_lti_steps_clear_the_prior_of_mode_one_rows_only():
    _need_gpu()
    Bs = 16
    idx = np.arange(Bs) % 4
    c = _controller(Bs, obs=EDGE_OBS, oidx=idx, pri=EDGE_PRI, pidx=idx)
    _pid_lap_and_seed(c)
    _drive(c, 20)
    mode1 = np.array([r.mode for r in EDGE_OBS])[idx] == 1
    for step in (lambda: c.rollout_pid_step(0.8, seed=9), lambda: c.rollout_step(seed=9, mode=2)):
        step()
        assert np.array_equal(_read(c, "has_pred", Bs, np.int32), (~mode1).astype(np.int32))
        assert np.array_equal(_read(c, "x_est", (Bs, 6)), _read(c, "x_meas", (Bs, 6)))
        assert np.all(np.isnan(_read(c, "x_prior", (Bs, 6))))
        c.rollout_step(seed=9)
        assert np.all(_read(c, "has_pred", Bs, np.int32) == 1)
    c.close()


def test_retired_controllers_write_nothing():
    _need_gpu()
    Bs = 16
    c = _controller(Bs, pri=[ObserverPrior.plant()])
    _pid_lap_and_seed(c)
    budget = np.where(np.arange(Bs) % 2 == 0, 1, 3).astype(np.int32)
    c.set_lap_budget(budget)
    for k in range(600):
        c.rollout_step(seed=77)
        c.rollout_commit_laps_dev()
        if k % 8 == 7 and (c.books()["lap_n"][0::2] >= 1).all():
            break
    ret = np.nonzero(c.books()["lap_n"] >= budget)[0]
    assert ret.size == Bs // 2

    def snap():
        rec = [np.frombuffer(b"".join(a.tobytes() for a in c.rollout_get_lap(int(b))), np.uint8) for b in ret]
        return (c.rollout_state(), _read(c, "x_est", (Bs, 6)), _read(c, "x_prior", (Bs, 6)), rec)
    s0 = snap()
    _drive(c, 40, seed=77)
    s1 = snap()
    for key in ("x", "xglob", "done", "cl_len"):
        assert np.array_equal(s0[0][key][ret], s1[0][key][ret]), key
    assert s0[1][ret].tobytes() == s1[1][ret].tobytes() and s0[2][ret].tobytes() == s1[2][ret].tobytes()
    assert all(np.array_equal(a, b) for a, b in zip(s0[3], s1[3]))
    c.close()


def test_shaped_controllers_take_the_plant_prior():
    """Controllers of shapes (8, 48) and (12, 24) (shape sets): with process noise off and no sensor, their plant prior is the
    plant."""
    _need_gpu()
    Bs = 8
    c = _controller(Bs, meas=None, noise=QUIET, pri=[ObserverPrior.plant()])
    c.set_shapes([(8, 48), (12, 24)], np.arange(Bs) % 2)
    _pid_lap_and_seed(c)
    rows = []
    for _ in range(200):
        hp = _read(c, "has_pred", Bs, np.int32)
        x = c.rollout_state()["x"].copy()
        lap_n = c.books()["lap_n"].copy()
        c.rollout_step(seed=1234)
        rows.append((hp, x, _read(c, "x_prior", (Bs, 6)), _read(c, "x_est", (Bs, 6)), lap_n))
        c.rollout_commit_laps_dev()
    used = sum(int(r[0].sum()) for r in rows)
    assert used > 0
    for k, (hp, x, xq, xe, _) in enumerate(rows):
        on = hp == 1
        assert xq[on].tobytes() == x[on].tobytes() and xe.tobytes() == x.tobytes(), k
    c.close()


# ---- 5. batches -------------------------------------------------------------------------------------------------------------
def test_batch_of_sources_gains_and_sensors_equals_one_handle_per_row():
    _need_gpu()
    Bs = 32
    b = np.arange(Bs)
    pri = [ObserverPrior.plan(), ObserverPrior.car(VehicleParams.from_friction(0.6)), ObserverPrior.plant()]
    obs = [HALF, ObserverParams.from_noise(0.01, 0.03)]
    meas = [BASE, MeasurementParams.scaled(3, BASE)]
    pidx, oidx, midx = b % 3, (b // 3) % 2, (b // 6) % 2

    def hook(p_rows, p_idx, o_rows, o_idx, m_rows, m_idx):
        def h(c):
            enable = c.enable_rollout

            def enable_then(Tcl=512):
                enable(Tcl)
                c.set_measurement_noise(m_rows, m_idx)
                c.set_observers(o_rows, o_idx)
                c.set_observer_priors(p_rows, p_idx)
            c.enable_rollout = enable_then
        return h
    n, het, het_laps = cl.run(Bs, hook=hook(pri, pidx, obs, oidx, meas, midx))
    assert (het["lap_n"] >= 1).mean() > 0.9
    z = np.zeros(Bs, np.int32)
    for p in range(3):
        for o in range(2):
            for m in range(2):
                sel = (pidx == p) & (oidx == o) & (midx == m)
                if not sel.any():
                    continue
                ref = cl.run(Bs, hook=hook([pri[p]], z, [obs[o]], z, [meas[m]], z), steps=n)[1:]
                cl.same((het, het_laps), ref, sel, "prior %d observer %d meas %d" % (p, o, m))


# ---- 6. snapshots -----------------------------------------------------------------------------------------------------------
def test_snapshot_restore_and_clone_continue_exactly():
    _need_gpu()
    Bs = 16
    streams = np.arange(Bs) % 8
    pri = [ObserverPrior.plant(), ObserverPrior.car(VehicleParams.from_friction(0.6))]
    pidx = (np.arange(Bs) % 8) % 2
    kw = dict(pri=pri, pidx=pidx, streams=streams, surf=[WET])
    c = _controller(Bs, **kw)
    _pid_lap_and_seed(c)
    _drive(c, 150)
    rec = c.snapshot().clone()
    clock = c.rollout_clock
    _drive(c, 200)
    straight = _result(c)
    c.close()

    d = _controller(Bs, **kw)
    d.restore(rec)
    d.rollout_clock = clock
    _drive(d, 200)
    _same(_result(d), straight, np.ones(Bs, bool), "restored")
    d.close()

    e = _controller(Bs, **kw)
    _pid_lap_and_seed(e)
    _drive(e, 150)
    e.clone(np.arange(8), np.arange(8, 16))
    _drive(e, 200)
    r = _result(e, records=False)
    for key in ("x", "xglob", "done", "cl_len"):
        assert np.array_equal(r["state"][key][:8], r["state"][key][8:]), key
    assert _read(e, "x_prior", (Bs, 6))[:8].tobytes() == _read(e, "x_prior", (Bs, 6))[8:].tobytes()
    e.close()
