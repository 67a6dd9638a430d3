"""GPU tier: model-based observer gains of the device closed loop (lmpc_rollout_set_observer_gains).

No gain table, a table of mode 0 rows and a table removed by nsets == 0 equal one another bit for bit; refused calls, the
cross-table ones in both directions included, change nothing; the gain kernel adds one launch to rollout steps of mode 0 and 1
and none to PID and mode 2 steps.  Under mode 1 the prior is what it is without the table, obs_jac is the numpy tangent
restatement (tests/support/observer_gain.py) across finish lines, surfaces and lap schedules, obs_cov solves the DARE, obs_gain is
scipy's gain and x_est the restated blend of the device's K, p and y bit for bit.  With process noise off and no sensor the
estimate is the plant state.  The limits, the failure flags, PID, LTI, retired and shaped controllers, batches against one handle
per row, and snapshots."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy import linalg

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                # noqa: E402
from racinglmpc_b200 import _native as nat                        # noqa: E402
from racinglmpc_b200.reference_params import (MeasurementParams, NoiseParams, ObserverGains, ObserverParams,   # noqa: E402
                                              ObserverPrior, SurfaceParams, VehicleParams)
import closed_loop as cl                                          # noqa: E402
import observer_gain as og                                        # noqa: E402
import observer_prior as op                                       # noqa: E402
from closed_loop import N, X0                                     # noqa: E402

LMPC_E_INVALID, LMPC_E_STATE = -1, -4
BASE = MeasurementParams((0.01, 0.01, 0.01, 0.005, 0.01, 0.01), (0.05, 0.05, 0.05, 0.025, 0.05, 0.05))
T0 = rp.TrackParams.l_shaped()
L = float(T0.TrackLength)
SEG = np.asarray(T0.seg_table, float)
CAR = VehicleParams.reference()
WETCAR = VehicleParams.from_friction(0.55)
HALF = ObserverParams.uniform(0.5)
WET = SurfaceParams.from_zones([(2.0, 4.0, 0.7, 0.6), (6.0, 8.0, 0.9, 0.8)])
QUIET = NoiseParams.scaled(0.0, 0.0)
KAL = ObserverGains.kalman((1e-5, 1e-5, 1e-5, 1e-7, 1e-7, 1e-7), tuple(rp.clipped_normal_variance(s, c)
                                                                       for s, c in zip(BASE.sigma, BASE.clip)))
KAL2 = ObserverGains.kalman((1e-3, 1e-4, 1e-3, 1e-5, 1e-6, 1e-5), (1e-4,) * 6)
NAN36 = np.full(36, np.nan)


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _read(c, name, shape, dtype=np.float64):
    out = np.zeros(shape, dtype)
    nat.check(c._lib.lmpc_read_buffer(c._h, name.encode(), 0, nat.ptr(out), out.nbytes))
    return out


def _controller(Bs, obs=(HALF,), oidx=None, pri=(ObserverPrior.plant(),), pidx=None, gains=(KAL,), gidx=None, meas=(BASE,),
                midx=None, noise=None, streams=None, surf=None, sidx=None, veh=None, vidx=None, reports=True):
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
    if gains is not None:
        c.set_observer_gains(list(gains), z if gidx is None else gidx)
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


def _bufs(c):
    Bs = c.B
    return {k: _read(c, k, (Bs, 36)) for k in ("obs_jac", "obs_cov", "obs_gain")}


# ---- 1. refusals, launches, identity ----------------------------------------------------------------------------------------
def _reject(c):
    """Every refusal of the gain call and the cross-table refusals of the prior call; returns nothing, changes nothing."""
    Lb = nat.lib()
    B = c.B
    idx = np.arange(B, dtype=np.int32) % 2
    good, _ = nat.make_observer_gain_sets([ObserverGains.fixed(), KAL], idx, B)

    def copy_of(mod):
        t = (nat.ObserverGainParams * 2)()
        C.memmove(t, good, C.sizeof(t))
        mod(t)
        return t
    bad = [copy_of(lambda t: setattr(t[0], "mode", 2)), copy_of(lambda t: setattr(t[1], "mode", -1)),
           copy_of(lambda t: t[1].q.__setitem__(0, 0.0)), copy_of(lambda t: t[1].q.__setitem__(5, -1.0)),
           copy_of(lambda t: t[1].r.__setitem__(2, float("nan"))), copy_of(lambda t: t[1].r.__setitem__(3, float("inf"))),
           copy_of(lambda t: t[1].r.__setitem__(4, 0.0))]
    cases = [(t, 2, idx) for t in bad] + [(good, 2, np.full(B, 2, np.int32)), (good, 2, np.full(B, -1, np.int32)),
                                          (good, 0, idx), (None, 2, idx), (good, 2, None), (good, -1, idx)]
    for tab, n, ix in cases:
        assert Lb.lmpc_rollout_set_observer_gains(c._h, tab, n, nat.ptr(ix) if ix is not None else None) == LMPC_E_INVALID


def test_needs_the_closed_loop_refuses_and_counts_launches():
    _need_gpu()
    Bs = 8
    c = cl.controller(Bs)
    ok, ix = nat.make_observer_gain_sets([KAL], np.zeros(Bs), Bs)
    assert nat.lib().lmpc_rollout_set_observer_gains(c._h, ok, 1, nat.ptr(ix)) == LMPC_E_STATE
    c.enable_rollout(Tcl=1024)
    c.rollout_set_state(np.tile(X0, (Bs, 1)), np.tile(X0, (Bs, 1)))
    _pid_lap_and_seed(c)
    z = np.zeros(Bs)
    half = np.arange(Bs) % 2
    c.set_observers([HALF], z)
    with pytest.raises(nat.NativeError):                                # no prior table
        c.set_observer_gains([KAL], z)
    c.set_observer_priors([ObserverPrior.plan(), ObserverPrior.plant()], half)
    with pytest.raises(nat.NativeError):                                # controller 0 has source 0
        c.set_observer_gains([KAL], z)
    c.set_observer_gains([ObserverGains.fixed(), KAL], half)            # mode 1 only where the source is a car
    with pytest.raises(nat.NativeError):                                # would give a mode 1 row source 0
        c.set_observer_priors([ObserverPrior.plan()], z)
    with pytest.raises(nat.NativeError):                                # a removal would too
        c.set_observer_priors(None)
    c.set_observer_priors([ObserverPrior.car(CAR), ObserverPrior.plant()], 1 - half)   # source 1 for the mode 1 rows: allowed
    with pytest.raises(ValueError):
        c.set_observer_gains([ObserverGains.kalman(0.0, 1.0)], z)
    counts = {}
    for g in (False, True):
        c.set_observer_gains([ObserverGains.fixed(), KAL] if g else None, half if g else None)
        for mode in (1, 0, 2):
            counts[(g, mode)] = _launches(c, lambda: c.rollout_step(seed=5, mode=mode))
        counts[(g, "pid")] = _launches(c, lambda: c.rollout_pid_step(0.8, seed=1))
    assert counts[(True, 1)] == counts[(False, 1)] + 1 and counts[(True, 0)] == counts[(False, 0)] + 1
    assert counts[(True, 2)] == counts[(False, 2)] and counts[(True, "pid")] == counts[(False, "pid")]
    c.set_observer_gains(None)
    c.set_observer_priors([ObserverPrior.plan()], z)                    # without a gain table: as before
    c.close()


@pytest.fixture(scope="module")
def identity_runs():
    """Shared streams, base measurement noise, plant and believed-car priors, observer rows of 0.5 and from_noise gains: no gain
    table, mode 0 rows (installed, then every refused call), and a mode 1 table removed by nsets == 0."""
    _need_gpu()
    Bs = 32
    streams = np.arange(Bs) // 2
    obs = [HALF, ObserverParams.from_noise(0.01, 0.03)]
    oidx = np.arange(Bs) % 2
    pri = [ObserverPrior.plant(), ObserverPrior.car(VehicleParams.from_friction(0.7))]
    pidx = (np.arange(Bs) // 2) % 2
    out = {}
    for name in ("none", "fixed", "reverted"):
        kw = dict(obs=obs, oidx=oidx, pri=pri, pidx=pidx, streams=streams, gains=None)
        if name == "fixed":
            kw.update(gains=[ObserverGains.fixed()])
        elif name == "reverted":
            kw.update(gains=[KAL, KAL2], gidx=oidx)
        c = _controller(Bs, **kw)
        if name == "fixed":
            _reject(c)
        if name == "reverted":
            c.set_observer_gains(None)
        _pid_lap_and_seed(c)
        out[name + "_launch"] = _launches(c, lambda: c.rollout_step(seed=1234))
        c.rollout_commit_laps_dev()
        _drive(c, 349)
        out[name] = _result(c)
        c.close()
    return out


def test_mode_zero_and_removed_tables_equal_no_table(identity_runs):
    r = identity_runs
    sel = np.ones(32, bool)
    assert r["none"]["books"]["lap_n"].max() >= 1
    assert r["fixed_launch"] == r["none_launch"] + 1 and r["reverted_launch"] == r["none_launch"]
    for name in ("fixed", "reverted"):
        _same(r[name], r["none"], sel, name)


# ---- 2. the prior, the Jacobian, the DARE, the gain and the blend -----------------------------------------------------------
def test_prior_is_unchanged_by_the_gain_table():
    """From the same record and clock, one step with a mode 1 gain table and one without form the same x_prior bit for bit."""
    _need_gpu()
    Bs = 16
    c = _controller(Bs, surf=[WET], meas=(MeasurementParams.scaled(3, BASE),),
                    pri=[ObserverPrior.plant(), ObserverPrior.car(WETCAR)], pidx=np.arange(Bs) % 2)
    _pid_lap_and_seed(c)
    checked = 0
    for k in range(240):
        if k % 20 == 5:
            rec, clock = c.snapshot().clone(), c.rollout_clock
            c.rollout_step(seed=1234)
            with_gain = _read(c, "x_prior", (Bs, 6))
            c.restore(rec)
            c.rollout_clock = clock
            c.set_observer_gains(None)
            c.rollout_step(seed=1234)
            without = _read(c, "x_prior", (Bs, 6))
            assert with_gain.tobytes() == without.tobytes(), k
            checked += int(np.isfinite(with_gain[:, 0]).sum())
            c.restore(rec)
            c.rollout_clock = clock
            c.set_observer_gains([KAL], np.zeros(Bs))
        c.rollout_step(seed=1234)
        c.rollout_commit_laps_dev()
    assert checked > 0
    c.close()


def _check_step(b, xpp0, u, y, lap_n, xq, xe, bufs, rows, gain, tol_jac=1e-12):
    """One controller's step against the restatement.  rows: (vehicle, zones) the prior used.  Returns True when a gain was
    formed."""
    K = bufs["obs_gain"][b].reshape(6, 6)
    if not np.all(np.isfinite(K)):
        return False
    veh, zones = rows
    p, A, ok = og.tangent_period(veh, SEG, L, xpp0, u, zones=zones)
    assert ok
    Ad = bufs["obs_jac"][b].reshape(6, 6)
    assert np.max(np.abs(Ad - A)) <= tol_jac * np.max(np.abs(A)), (b, Ad - A)
    P = bufs["obs_cov"][b].reshape(6, 6)
    q, r = np.array(gain.q), np.array(gain.r)
    assert og.dare_residual(Ad, P, q, r) <= 1e-10
    ref = linalg.solve_discrete_are(Ad.T, np.eye(6), np.diag(q), np.diag(r))
    Ksc = ref @ np.linalg.inv(ref + np.diag(r))
    assert np.max(np.abs(K - Ksc)) <= 1e-9, (b, K - Ksc)
    assert xe.tobytes() == og.blend(y, xq, K, L).tobytes(), b
    return True


def test_jacobian_dare_gain_and_blend_across_laps_surfaces_and_schedules():
    """Plant priors under vehicle and surface schedules that change at lap 1 and believed-car priors, two (q, r) rows, sensor
    noise: every formed gain is checked, including the steps right after a hand-over."""
    _need_gpu()
    Bs = 8
    b = np.arange(Bs)
    pri = [ObserverPrior.plant(), ObserverPrior.car(WETCAR)]
    pidx, gidx = b % 2, (b // 2) % 2
    gains = [KAL, KAL2]
    c = _controller(Bs, pri=pri, pidx=pidx, gains=gains, gidx=gidx, surf=[SurfaceParams.dry(), WET], veh=[CAR, WETCAR])
    c.set_lap_schedule("vehicle", [0, 1])
    c.set_lap_schedule("surface", [0, 1])
    _pid_lap_and_seed(c)
    vehs, surfs = [CAR, WETCAR], [None, list(WET.zones)]
    formed = after = 0
    for k in range(420):
        hp = _read(c, "has_pred", Bs, np.int32)
        xpp0 = _read(c, "xPredPrev", (Bs, N + 1, 6))[:, 0]
        u = _read(c, "OldInput", (Bs, 2))
        lap_n = c.books()["lap_n"].copy()
        c.rollout_step(seed=1234)
        y, xq, xe = _read(c, "x_meas", (Bs, 6)), _read(c, "x_prior", (Bs, 6)), _read(c, "x_est", (Bs, 6))
        bufs = _bufs(c)
        flags = c.step_results()["flags"]
        assert not np.any(flags & nat.FLAG_OBSERVER_GAIN), k
        for i in range(Bs):
            if not hp[i]:
                assert np.all(np.isnan(bufs["obs_gain"][i])) and xe[i].tobytes() == y[i].tobytes()
                continue
            if flags[i] & nat.FLAG_OBSERVER_RESET:
                continue
            if pidx[i] == 0:
                back = op.back_laps(xpp0[i][4], y[i][4], L)
                row = op.scheduled_row([0, 1], lap_n[i], back)
                rows = (vehs[row], surfs[row])
                after += int(back == 1)
            else:
                rows = (WETCAR, None)
            if k % 3 == 0 or (pidx[i] == 0 and op.back_laps(xpp0[i][4], y[i][4], L)):
                formed += _check_step(i, xpp0[i], u[i], y[i], lap_n[i], xq[i], xe[i], bufs, rows, gains[gidx[i]])
            else:
                assert np.all(np.isfinite(bufs["obs_gain"][i]))
        c.rollout_commit_laps_dev()
    assert formed > 100 and after > 0 and c.books()["lap_n"].min() >= 1, (formed, after)
    c.close()


def test_noise_free_estimate_is_the_plant_state():
    _need_gpu()
    Bs = 8
    c = _controller(Bs, meas=None, noise=QUIET, gains=[KAL, KAL2], gidx=np.arange(Bs) % 2)
    _pid_lap_and_seed(c)
    used = 0
    for k in range(400):
        hp = _read(c, "has_pred", Bs, np.int32)
        x = c.rollout_state()["x"].copy()
        c.rollout_step(seed=1234)
        xe = _read(c, "x_est", (Bs, 6))
        assert xe.tobytes() == x.tobytes(), k
        on = hp == 1
        assert np.all(np.isfinite(_read(c, "obs_gain", (Bs, 36))[on])), k
        used += int(on.sum())
        c.rollout_commit_laps_dev()
    assert used > 0 and c.books()["lap_n"].min() >= 1
    c.close()


def test_measurement_dominated_limit_reads_y():
    """r << q: K -> I and x_hat -> y."""
    _need_gpu()
    Bs = 8
    c = _controller(Bs, gains=[ObserverGains.kalman(1.0, 1e-12)])
    _pid_lap_and_seed(c)
    _drive(c, 30)
    c.rollout_step(seed=1234)
    K = _read(c, "obs_gain", (Bs, 36)).reshape(Bs, 6, 6)
    assert np.max(np.abs(K - np.eye(6))) < 1e-9
    y, xe = _read(c, "x_meas", (Bs, 6)), _read(c, "x_est", (Bs, 6))
    assert np.max(np.abs(xe - y)) < 1e-9
    c.close()


# ---- 3. failures ------------------------------------------------------------------------------------------------------------
def _to_next_lap(c, lap_n0):
    for _ in range(600):
        c.rollout_step(seed=1234)
        c.rollout_commit_laps_dev()
        if (c.books()["lap_n"] > lap_n0).all():
            break
    rep = c.lap_reports()
    assert np.all(rep["n"] > lap_n0)
    return rep


def test_an_overflowing_dare_flags_and_reads_y():
    """q = 1e308 overflows P (its symmetric part (H + H') / 2 exceeds the largest double): those rows flag
    LMPC_FLAG_OBSERVER_GAIN and read y, the others do not; the flag reaches the health word and the lap report.  (The doubling
    itself stays finite for q = 1e200, r = 1e-200: W^-1 A and W^-1 G round to 0 and the gain is I.)"""
    _need_gpu()
    Bs = 8
    idx = np.arange(Bs) % 2
    c = _controller(Bs, gains=[KAL, ObserverGains.kalman(1e308, 1.0)], gidx=idx)
    _pid_lap_and_seed(c)
    _drive(c, 20)
    lap_n0 = c.books()["lap_n"].copy()
    c.rollout_step(seed=1234)
    bad = idx == 1
    flags = c.step_results()["flags"]
    assert np.array_equal((flags & nat.FLAG_OBSERVER_GAIN) != 0, bad)
    assert not np.any(flags & nat.FLAG_OBSERVER_RESET)
    y, xe = _read(c, "x_meas", (Bs, 6)), _read(c, "x_est", (Bs, 6))
    assert xe[bad].tobytes() == y[bad].tobytes()
    K = _read(c, "obs_gain", (Bs, 36))
    assert np.all(np.isnan(K[bad])) and np.all(np.isfinite(K[~bad]))
    c.rollout_commit_laps_dev()
    assert np.array_equal((c.rollout_health()[0] & nat.FLAG_OBSERVER_GAIN) != 0, bad)
    rep = _to_next_lap(c, lap_n0)
    got = np.array([(rep["flags"][b, lap_n0[b]] & nat.FLAG_OBSERVER_GAIN) != 0 for b in range(Bs)])
    assert np.array_equal(got, bad)
    c.close()


@pytest.mark.parametrize("where", ["xPredPrev", "OldInput"])
def test_a_non_finite_input_resets_those_rows_only(where):
    _need_gpu()
    Bs = 8
    c = _controller(Bs)
    _pid_lap_and_seed(c)
    _drive(c, 20)
    sel = np.arange(Bs) % 3 == 1
    if where == "xPredPrev":
        xpp = _read(c, "xPredPrev", (Bs, N + 1, 6))
        hp = _read(c, "has_pred", Bs, np.int32)
        xpp[sel, 0, 2] = np.nan
        c.set_state(xPred=xpp, has_pred=hp)
    else:
        u = _read(c, "OldInput", (Bs, 2))
        u[sel, 0] = np.nan
        c.set_state(OldInput=u)
    lap_n0 = c.books()["lap_n"].copy()
    c.rollout_step(seed=1234)
    flags = c.step_results()["flags"]
    assert np.array_equal((flags & nat.FLAG_OBSERVER_RESET) != 0, sel)
    assert not np.any(flags & nat.FLAG_OBSERVER_GAIN)
    y, xe = _read(c, "x_meas", (Bs, 6)), _read(c, "x_est", (Bs, 6))
    assert xe[sel].tobytes() == y[sel].tobytes()
    bufs = _bufs(c)
    for k in bufs:
        assert np.all(np.isnan(bufs[k][sel])) and np.all(np.isfinite(bufs[k][~sel])), k
    c.rollout_commit_laps_dev()
    # the health word and the reports are cumulative: a noisy estimate with s < 0 at a lap start resets on its own (DESIGN.md,
    # "Observer priors"), so only the rows made non-finite are known to carry the flag
    assert np.all((c.rollout_health()[0][sel] & nat.FLAG_OBSERVER_RESET) != 0)
    if where == "OldInput":       # OldInput is also the QP's input-rate reference: a NaN there stalls those controllers' laps
        c.close()
        return
    rep = _to_next_lap(c, lap_n0)
    got = np.array([(rep["flags"][b, lap_n0[b]] & nat.FLAG_OBSERVER_RESET) != 0 for b in range(Bs)])
    assert np.all(got[sel])
    c.close()


# ---- 4. step kinds ----------------------------------------------------------------------------------------------------------
def test_pid_and_lti_steps_clear_the_prior_and_form_no_gain():
    _need_gpu()
    Bs = 8
    c = _controller(Bs)
    _pid_lap_and_seed(c)
    _drive(c, 20)
    for step in (lambda: c.rollout_pid_step(0.8, seed=9), lambda: c.rollout_step(seed=9, mode=2)):
        step()
        assert np.all(_read(c, "has_pred", Bs, np.int32) == 0)
        assert np.array_equal(_read(c, "x_est", (Bs, 6)), _read(c, "x_meas", (Bs, 6)))
        assert all(np.all(np.isnan(v)) for v in _bufs(c).values())
        c.rollout_step(seed=9)
        assert np.all(_read(c, "has_pred", Bs, np.int32) == 1)
        c.rollout_step(seed=9)
        assert np.all(np.isfinite(_read(c, "obs_gain", (Bs, 36))))
    c.close()


def test_retired_controllers_write_nothing():
    _need_gpu()
    Bs = 16
    c = _controller(Bs)
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
        bufs = [_read(c, k, (Bs, 6))[ret].tobytes() for k in ("x_est", "x_prior")]
        bufs += [v[ret].tobytes() for v in _bufs(c).values()]
        return c.rollout_state(), bufs, rec
    s0 = snap()
    _drive(c, 40, seed=77)
    s1 = snap()
    for key in ("x", "xglob", "done", "cl_len"):
        assert np.array_equal(s0[0][key][ret], s1[0][key][ret]), key
    assert s0[1] == s1[1]
    assert all(np.array_equal(a, b) for a, b in zip(s0[2], s1[2]))
    c.close()


def test_shaped_controllers_get_model_gains():
    _need_gpu()
    Bs = 8
    c = _controller(Bs, meas=None, noise=QUIET)
    c.set_shapes([(8, 48), (12, 24)], np.arange(Bs) % 2)
    _pid_lap_and_seed(c)
    used = 0
    for k in range(200):
        hp = _read(c, "has_pred", Bs, np.int32)
        x = c.rollout_state()["x"].copy()
        c.rollout_step(seed=1234)
        assert _read(c, "x_est", (Bs, 6)).tobytes() == x.tobytes(), k
        K = _read(c, "obs_gain", (Bs, 36))
        assert np.all(np.isfinite(K[hp == 1])) and np.all(np.isnan(K[hp == 0])), k
        used += int(hp.sum())
        c.rollout_commit_laps_dev()
    assert used > 0
    c.close()


# ---- 5. batches -------------------------------------------------------------------------------------------------------------
def test_batch_of_gains_sources_and_sensors_equals_one_handle_per_row():
    _need_gpu()
    Bs = 24
    b = np.arange(Bs)
    gains = [ObserverGains.fixed(), KAL, KAL2]
    pri = [ObserverPrior.car(VehicleParams.from_friction(0.7)), ObserverPrior.plant()]
    meas = [BASE, MeasurementParams.scaled(3, BASE)]
    gidx, pidx, midx = b % 3, (b // 3) % 2, (b // 6) % 2

    def hook(g_rows, g_idx, p_rows, p_idx, m_rows, m_idx):
        def h(c):
            enable = c.enable_rollout

            def enable_then(Tcl=512):
                enable(Tcl)
                c.set_measurement_noise(m_rows, m_idx)
                c.set_observers([HALF], np.zeros(c.B, np.int32))
                c.set_observer_priors(p_rows, p_idx)
                c.set_observer_gains(g_rows, g_idx)
            c.enable_rollout = enable_then
        return h
    n, het, het_laps = cl.run(Bs, hook=hook(gains, gidx, pri, pidx, meas, midx))
    assert (het["lap_n"] >= 1).mean() > 0.9
    z = np.zeros(Bs, np.int32)
    for g in range(3):
        for p in range(2):
            for m in range(2):
                sel = (gidx == g) & (pidx == p) & (midx == m)
                if not sel.any():
                    continue
                ref = cl.run(Bs, hook=hook([gains[g]], z, [pri[p]], z, [meas[m]], z), steps=n)[1:]
                cl.same((het, het_laps), ref, sel, "gains %d prior %d meas %d" % (g, p, m))


# ---- 6. snapshots -----------------------------------------------------------------------------------------------------------
def test_snapshot_restore_and_clone_continue_exactly():
    _need_gpu()
    Bs = 16
    streams = np.arange(Bs) % 8
    pri = [ObserverPrior.plant(), ObserverPrior.car(VehicleParams.from_friction(0.6))]
    pidx = (np.arange(Bs) % 8) % 2
    kw = dict(pri=pri, pidx=pidx, streams=streams, surf=[WET], gains=[KAL, KAL2], gidx=(np.arange(Bs) % 8) // 4)
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
    g = _read(e, "obs_gain", (Bs, 36))
    assert g[:8].tobytes() == g[8:].tobytes()
    e.close()
