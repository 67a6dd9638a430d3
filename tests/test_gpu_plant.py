"""GPU tier: the plant kernels against the exact reference of tests/support/plant_exact.py (checked itself by
tests/test_plant_reference.py), at their edges.

  sim_step_kernel     every case of plant_cases.sim_cases() in one launch (cars, circuits and noise sets interleaved, one case
                      per controller), and 50 consecutive steps at 3 m/s each checked from the device's own previous state:
                      |device - exact| <= SIM_BOUND (1 + |exact|) per component; `done` as the exact s says
  failed lookups      s = -1e-3, TrackLength, NaN and 65 TrackLength set health bit 128 in lmpc_rollout_pid_step and
                      lmpc_rollout_step; the arithmetic is the exact one with curvature 0 where the lookup fails
  record overflow     a lap longer than Tcl sets health bit 256
  pid_input_kernel    within one ulp of the exact PID.solve, clip edges, noise sets interleaved
  ridge_sysid_kernel  within SYSID_C max(cond, T) eps max|W| of the exact ridge solve on device-driven records; flag bit 1
                      exactly when T < 12, and with every non-finite result of a singular system
  lap_cost_block      bit-equal to computeCost through lmpc_ss_put_lap (rollout_cost_kernel) and through the lap hand-over
The largest device-vs-exact errors are printed (pytest -s)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                  # noqa: E402
from racinglmpc_b200.controller import BatchedController            # noqa: E402
from racinglmpc_b200.reference_params import NoiseParams, TrackParams   # noqa: E402
import plant_cases as pc                                            # noqa: E402
import plant_exact as pe                                            # noqa: E402

N = 12
LOOKUP_FAILED, RECORD_FULL = 128, 256


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _mpc(B, Tcl, Tmax=1024):
    t = pc.TRACKS[0]
    c = BatchedController(rp.mpc_params(N), B, t.seg_table, t.TrackLength, trToUse=1, Tmax=Tmax, model_cap=2)
    c.enable_rollout(Tcl=Tcl)
    return c


def _lmpc(B, Tcl, Tmax=1024):
    t = pc.TRACKS[0]
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, B, t.seg_table, t.TrackLength, trToUse=4, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=Tmax, ss_cap=6, model_cap=5)
    c.enable_rollout(Tcl=Tcl)
    return c


def _applied_u(c):
    """The input each controller's last step applied: the last row of its record."""
    return np.array([c.rollout_get_lap(b)[1][-1] for b in range(c.B)])


def _check_step(case_x, case_xg, u, st, b, vehicle, etrack, z, noise, what):
    r = pe.dyn_model(vehicle, etrack, case_x, case_xg, u, z=z, noise=noise)
    ex, eg = pe.sim_error(st["x"][b], r["x"]), pe.sim_error(st["xglob"][b], r["x_glob"])
    assert ex <= pe.SIM_BOUND and eg <= pe.SIM_BOUND, (what, ex, eg)
    assert bool(st["done"][b]) == r["done"], what
    return r, max(ex, eg)


def test_simulator_case_list_in_one_launch():
    _need_gpu()
    cases = pc.sim_cases()
    B = len(cases)
    c = _mpc(B, Tcl=16)
    c.set_vehicles(pc.VEHICLES, np.array([k.veh for k in cases]))
    c.set_tracks(pc.TRACKS, np.array([k.trk for k in cases]))
    c.set_noise(pc.NOISES, np.array([k.noise_idx for k in cases]))
    x = np.array([k.x for k in cases])
    xg = np.array([k.xg for k in cases])
    c.rollout_set_state(x, xg)
    c.rollout_pid_step(pc.VT, z_pid=np.array([k.z_pid() for k in cases]), z_sim=np.array([k.z for k in cases]))
    st = c.rollout_state()
    u = _applied_u(c)
    flags, _ = c.rollout_health()
    assert np.all(flags == 0), flags
    worst = 0.0
    for b, k in enumerate(cases):
        xr, _ = c.rollout_get_lap(b)
        assert np.array_equal(xr[-1], k.x) or (np.isnan(xr[-1]) == np.isnan(k.x)).all(), k.name
        assert np.max(np.abs(u[b] - k.u)) < 1e-12, k.name       # the PID's draw set the input the case asked for
        r, e = _check_step(k.x, k.xg, u[b], st, b, k.vehicle, k.exact_track, k.z, k.noise, k.name)
        assert k.boundary_case or r["margin"] >= 1e-9, (k.name, float(r["margin"]))
        worst = max(worst, e)
        if k.noise_idx != 0:                                      # the draw shows in x - xglob, within one rounding of the sum
            for j in range(3):
                d = st["x"][b, j] - st["xglob"][b, j]
                assert abs(d - float(r["draw"][j])) <= pe.ulp(st["x"][b, j]), (k.name, j)
    assert any(k.name.startswith("finish") for k in cases) and st["done"].any() and not st["done"].all()
    print("\nsim_step_kernel, %d cases: max |device - exact| / (1 + |exact|) = %.3g (bound %.3g)" % (B, worst, pe.SIM_BOUND))
    c.close()


def test_simulator_fifty_steps_at_speed():
    """50 steps at 3 m/s on four cars and three circuits, each step checked from the device's own previous state."""
    _need_gpu()
    B, K = 4, 50
    c = _mpc(B, Tcl=64)
    vidx, tidx = np.arange(B), np.arange(B) % 3
    c.set_vehicles(pc.VEHICLES[:B], vidx)
    c.set_tracks(pc.TRACKS, tidx)
    c.set_noise(pc.NOISES, np.zeros(B, np.int32))
    x0 = np.tile([3.0, 0.0, 0.0, 0.0, 0.1, 0.0], (B, 1))
    c.rollout_set_state(x0, x0)
    zs = np.random.default_rng(5).standard_normal((K, B, 3))
    et = [pe.ExactTrack(t.seg_table, t.TrackLength) for t in pc.TRACKS]
    worst = 0.0
    prev = c.rollout_state()
    for k in range(K):
        c.rollout_pid_step(3.0, z_pid=np.zeros((B, 2)), z_sim=zs[k])
        st = c.rollout_state()
        u = _applied_u(c)
        for b in range(B):
            r, e = _check_step(prev["x"][b], prev["xglob"][b], u[b], st, b, pc.VEHICLES[vidx[b]], et[tidx[b]], zs[k, b],
                               pc.NOISES[0], (k, b))
            assert r["margin"] >= 1e-9, (k, b)
            worst = max(worst, e)
        prev = st
    assert np.all(prev["x"][:, 0] > 1.5)
    print("\nsim_step_kernel, %d chained steps: max |device - exact| / (1 + |exact|) = %.3g" % (K * B, worst))
    c.close()


def _bad_states(L):
    s = [-1e-3, L, float("nan"), 65 * L, 5.0]                  # the last one is a control: its lookups succeed
    return np.array([[0.7, 0.01, 0.05, 0.0, sv, 0.02] for sv in s])


def test_failed_lookup_is_flagged_in_the_pid_step():
    _need_gpu()
    L = pc.TRACKS[0].TrackLength
    x = _bad_states(L)
    c = _mpc(x.shape[0], Tcl=16)
    c.rollout_set_state(x, x)
    c.rollout_pid_step(pc.VT, z_pid=np.zeros((x.shape[0], 2)), z_sim=np.zeros((x.shape[0], 3)))
    flags, _ = c.rollout_health()
    assert [bool(f & LOOKUP_FAILED) for f in flags] == [True] * 4 + [False], flags
    st, u = c.rollout_state(), _applied_u(c)
    et = pe.ExactTrack(pc.TRACKS[0].seg_table, L)
    for b in (0, 1, 3, 4):                                       # the state arithmetic goes on with curvature 0
        r = pe.dyn_model(rp.VehicleParams.reference(), et, x[b], x[b], u[b], on_fail="zero")
        assert r["failed"] == (b != 4)
        assert pe.sim_error(st["x"][b], r["x"]) <= pe.SIM_BOUND, b
    c.close()


def test_failed_lookup_is_flagged_in_the_closed_loop_step():
    _need_gpu()
    L = pc.TRACKS[0].TrackLength
    x = _bad_states(L)
    B = x.shape[0]
    c = _mpc(B, Tcl=64)
    x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (B, 1))
    c.rollout_set_state(x0, x0)
    for _ in range(30):
        c.rollout_pid_step(0.8, z_pid=np.zeros((B, 2)), z_sim=np.zeros((B, 3)))
    assert np.all(c.rollout_health()[0] == 0)
    c.rollout_sysid(1e-7)
    c.rollout_set_state(x, x)
    c.rollout_step(z=np.zeros((B, 3)), mode=2)
    flags, _ = c.rollout_health()
    assert [bool(f & LOOKUP_FAILED) for f in flags] == [True] * 4 + [False], flags
    c.close()


def test_record_overflow_is_flagged():
    _need_gpu()
    B, Tcl = 2, 16
    c = _mpc(B, Tcl=Tcl)
    x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (B, 1))
    c.rollout_set_state(x0, x0)
    for k in range(Tcl + 4):
        c.rollout_pid_step(0.8, z_pid=np.zeros((B, 2)), z_sim=np.zeros((B, 3)))
        flags, _ = c.rollout_health()
        full = k >= Tcl                                           # step k finds k rows recorded
        assert np.all(((flags & RECORD_FULL) != 0) == full), (k, flags)
        assert np.all(flags & ~RECORD_FULL == 0), (k, flags)
    _, n = c.rollout_done()
    assert np.all(n == Tcl)
    c.close()


def test_pid_input_within_one_ulp():
    _need_gpu()
    cases = pc.pid_cases()
    B = len(cases)
    c = _mpc(B, Tcl=16)
    c.set_noise(pc.PID_NOISES, np.array([k.noise_idx for k in cases]))
    c.rollout_set_state(np.array([k.x for k in cases]), np.array([k.x for k in cases]))
    c.rollout_pid_step(pc.VT, z_pid=np.array([k.z for k in cases]), z_sim=np.zeros((B, 3)))
    u = _applied_u(c)
    worst = 0.0
    for b, k in enumerate(cases):
        e = pe.pid_input(k.x, k.vt, k.z, k.noise.pid_sigma, k.noise.pid_clip)
        for j in range(2):
            d = abs(u[b, j] - float(e[j])) / pe.ulp(e[j])
            assert d <= 1.0, (k.name, j, d)
            worst = max(worst, d)
    # the clip edges clip
    for b, k in enumerate(cases):
        if k.noise_idx == 1 and abs(k.z[0]) > 0.9:
            e = pe.pid_input(k.x, k.vt, (0.0, 0.0), (1.0, 1.0), (0.9, 0.2))
            assert abs(u[b, 0] - (float(e[0]) - 0.9)) <= 2 * pe.ulp(u[b, 0]), k.name
    print("\npid_input_kernel, %d controllers: max |device - exact| = %.3g ulp" % (B, worst))
    c.close()


def _check_sysid(c, lamb, T, what, expect_flag=0):
    A, Bm, flags = c.rollout_sysid(lamb)
    assert np.all(flags == expect_flag), (what, lamb, flags)
    worst = 0.0
    if expect_flag:
        return worst
    for b in range(c.B):
        x, u = c.rollout_get_lap(b)
        assert x.shape[0] == T
        ref = pe.regression(x, u, lamb)
        e = pe.sysid_error(A[b], Bm[b], ref)
        assert e <= pe.SYSID_C, (what, lamb, b, e, ref["cond"])
        worst = max(worst, e)
    return worst


def test_sysid_on_pid_laps_of_eight_cars():
    _need_gpu()
    B, T = 8, 1000
    c = _mpc(B, Tcl=T)
    c.set_vehicles(pc.VEHICLES, np.arange(B))
    x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (B, 1))
    c.rollout_set_state(x0, x0)
    for _ in range(T):
        c.rollout_pid_step(0.8, seed=11)
    worst = max(_check_sysid(c, lamb, T, "pid lap") for lamb in (1e-7, 0.0, 1e3))
    print("\nridge_sysid_kernel, 1000-step PID laps: max error / (max(cond, T) eps max|W|) = %.3g (bound %.3g)" % (worst, pe.SYSID_C))
    c.close()


def test_sysid_flag_rule_at_eleven_twelve_and_tcl_rows():
    _need_gpu()
    B, Tcl = 3, 16
    c = _mpc(B, Tcl=Tcl)
    c.set_vehicles([pc.VEHICLES[k] for k in (0, 3, 6)], np.arange(B))
    x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (B, 1))
    c.rollout_set_state(x0, x0)
    rng = np.random.default_rng(3)
    for T in range(1, Tcl + 1):
        c.rollout_pid_step(0.8, z_pid=rng.standard_normal((B, 2)), z_sim=rng.standard_normal((B, 3)))
        if T == 11:
            _check_sysid(c, 1e-7, T, "T = 11", expect_flag=1)
        elif T in (12, 13, Tcl):
            _check_sysid(c, 1e-7, T, "T = %d" % T)
    c.close()


def test_sysid_rank_deficient_record():
    """Constant vx on a straight with no input: well-posed with a ridge, and with lambda = 0 every non-finite entry comes with
    flag bit 1."""
    _need_gpu()
    B, T = 2, 40
    c = _mpc(B, Tcl=T)
    c.set_tracks([TrackParams([[100.0, 0.0, 0.0, 0.0, 100.0, 0.0]])], np.zeros(B, np.int32))
    c.set_noise([NoiseParams.scaled(0.0, 0.0)], np.zeros(B, np.int32))
    x0 = np.tile(np.array([1.0, 0, 0, 0, 0, 0.0]), (B, 1))
    c.rollout_set_state(x0, x0)
    for _ in range(T):
        c.rollout_pid_step(1.0)
    x, u = c.rollout_get_lap(0)
    assert np.all(x[:, 0] == 1.0) and not np.any(x[:, [1, 2, 3, 5]]) and not np.any(u)
    for lamb in (1e-7, 1e3):
        _check_sysid(c, lamb, T, "rank deficient")
    A, Bm, flags = c.rollout_sysid(0.0)
    bad = ~(np.isfinite(A).all(axis=(1, 2)) & np.isfinite(Bm).all(axis=(1, 2)))
    assert np.all(flags[bad] & 1), flags
    assert np.all(flags & 1)                                     # the zero columns give exact zero pivots
    c.close()


def test_lap_cost_through_put_lap_at_chunk_edges():
    _need_gpu()
    Tmax = 1024
    c = _lmpc(1, Tcl=16, Tmax=Tmax)
    L = c.TrackLength
    for s, T in pc.cost_cases(L, Tmax):
        if T < 2:
            continue                                             # lmpc_ss_put_lap takes laps of two rows or more
        x = np.zeros((T, 6))
        x[:, 4] = s
        c.add_trajectory(0, x, np.zeros((T, 2)))
        _, _, q = c.get_lap(0, c.it[0] - 1)
        assert np.array_equal(q, pe.compute_cost(s, L)), T
    c.close()


def test_lap_cost_through_the_hand_over_across_the_finish_line():
    _need_gpu()
    B = 2
    c = _lmpc(B, Tcl=64)
    L = c.TrackLength
    x0 = np.array([[1.0, 0, 0, 0, L - 0.35, 0.0], [1.0, 0, 0, 0, L - 0.05, 0.0]])
    c.rollout_set_state(x0, x0)
    for _ in range(12):
        c.rollout_pid_step(1.0, z_pid=np.zeros((B, 2)), z_sim=np.zeros((B, 3)))
    done, n = c.rollout_done()
    recs = [c.rollout_get_lap(b)[0] for b in range(B)]
    for r in recs:
        assert (r[:, 4] < L).any() and (r[:, 4] >= L).any() and r[-1, 4] >= L    # the lap crossed the line mid-record
    c.rollout_finish_laps(np.ones(B, np.int32), n)
    for b in range(B):
        x, _, q = c.get_lap(b, 0)
        assert np.array_equal(x, recs[b]) and np.array_equal(q, pe.compute_cost(recs[b][:, 4], L)), b
    c.close()
