"""GPU tier: per-controller state observers of the device closed loop (lmpc_rollout_set_observers).

A table of all-ones rows or of mode 0 rows equals no table bit for bit, nsets == 0 reverts, refused calls change nothing, and a
table adds exactly one launch per step.  Step by step over a PID lap, the seeding and LMPC laps that cross a finish line, x_est
is the numpy restatement (tests/support/observer.py) fed x_meas, xPredPrev and has_pred, and it is what the QP, the record and
addPoint take, while rollout_state and the trace keep the plant state.  The edges: no prior after the seeding, a PID or mode 2
step clears the prior of mode 1 rows only, a non-finite prior resets and flags, retired controllers write nothing.  A batch of
rows is one handle per row, crossed with measurement sets and QP tunings too, and snapshots, restores and clones continue
exactly."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                # noqa: E402
from racinglmpc_b200 import _native as nat                        # noqa: E402
from racinglmpc_b200.reference_params import MeasurementParams, ObserverParams   # noqa: E402
import closed_loop as cl                                          # noqa: E402
import observer as ob                                             # noqa: E402
from closed_loop import N, X0                                     # noqa: E402

LMPC_E_INVALID, LMPC_E_STATE = -1, -4
BASE = MeasurementParams((0.01, 0.01, 0.01, 0.005, 0.01, 0.01), (0.05, 0.05, 0.05, 0.025, 0.05, 0.05))
L = float(rp.TrackParams.l_shaped().TrackLength)
ROWS = [ObserverParams.off(), ObserverParams.uniform(0.5), ObserverParams.gains(0.2, 0.7, 1.0, 0.0, 0.3, 0.9),
        ObserverParams.from_noise(0.01, 0.03)]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _read(c, name, shape, dtype=np.float64):
    out = np.zeros(shape, dtype)
    nat.check(c._lib.lmpc_read_buffer(c._h, name.encode(), 0, nat.ptr(out), out.nbytes))
    return out


def _tables(rows):
    """modes [K], gains [K, 6] of observer rows"""
    return np.array([r.mode for r in rows]), np.array([r.gain for r in rows], np.float64)


def _controller(Bs, obs=None, oidx=None, meas=(BASE,), midx=None, streams=None, psets=None, par=None, reports=True):
    c = cl.controller(Bs, par=par)
    if psets is not None:
        c.set_param_sets(*psets)
    c.enable_rollout(Tcl=1024)
    if reports:
        c.enable_lap_reports(64)
    if streams is not None:
        c.set_noise_streams(streams)
    if meas is not None:
        c.set_measurement_noise(list(meas), np.zeros(Bs, np.int32) if midx is None else midx)
    if obs is not None:
        c.set_observers(obs, oidx)
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
    """books, end state, health, solver report, lap reports and (records) snapshot records of every controller"""
    out = dict(books=c.books(), state=c.rollout_state(), health=c.rollout_health(), solver=c.step_results(),
               reports=c.lap_reports())
    if records:
        out["records"] = c.snapshot().cpu().numpy()
    return out


def _same(a, b, sel, what, path=()):
    """Results a and b (nested dicts / tuples of arrays) agree bit for bit on the controllers of the boolean mask sel."""
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


def observed(obs, index, then=None):
    """A closed_loop.run hook: measurement noise (BASE) and the observer table go in right after enable_rollout, then
    ``then(c)`` runs, if given."""
    def hook(c):
        enable = c.enable_rollout

        def enable_then_observe(Tcl=512):
            enable(Tcl)
            c.set_measurement_noise([BASE], np.zeros(c.B, np.int32))
            if obs is not None:
                c.set_observers(obs, index)
            if then is not None:
                then(c)
        c.enable_rollout = enable_then_observe
    return hook


# ---- 1. identity: no table, all-ones rows, mode 0 rows, revert, refusals, launches --------------------------------------------
def _reject(c):
    """Refused calls, each returning LMPC_E_INVALID; the handle must stay as it was."""
    Lb = nat.lib()
    idx = np.arange(c.B, dtype=np.int32) % 4
    good, _ = nat.make_observer_sets(ROWS, idx, c.B)

    def copy_of(mod):
        t = (nat.ObserverParams * 4)()
        C.memmove(t, good, C.sizeof(t))
        mod(t)
        return t
    bad = [copy_of(lambda t: setattr(t[1], "mode", 2)), copy_of(lambda t: setattr(t[0], "mode", -1)),
           copy_of(lambda t: t[2].gain.__setitem__(5, float("nan"))), copy_of(lambda t: t[3].gain.__setitem__(0, 1.5)),
           copy_of(lambda t: t[1].gain.__setitem__(4, -1e-300)), copy_of(lambda t: t[0].gain.__setitem__(2, float("inf")))]
    cases = [(t, 4, idx) for t in bad] + [(good, 4, np.full(c.B, 4, np.int32)), (good, 4, np.full(c.B, -1, np.int32)),
                                          (good, 0, idx), (None, 4, idx), (good, 4, None), (good, -1, idx)]
    for tab, n, ix in cases:
        assert Lb.lmpc_rollout_set_observers(c._h, tab, n, nat.ptr(ix) if ix is not None else None) == LMPC_E_INVALID
    big = (nat.ObserverParams * (c.B + 1))(*([good[0]] * (c.B + 1)))
    assert Lb.lmpc_rollout_set_observers(c._h, big, c.B + 1, nat.ptr(np.zeros(c.B, np.int32))) == LMPC_E_INVALID


def _launches(c, f):
    l0 = c.kernel_launches
    f()
    return c.kernel_launches - l0


def test_table_needs_the_closed_loop_and_adds_one_launch_per_step():
    _need_gpu()
    Bs = 8
    c = cl.controller(Bs)
    ok, ix = nat.make_observer_sets([ObserverParams.uniform(0.5)], np.zeros(Bs), Bs)
    assert nat.lib().lmpc_rollout_set_observers(c._h, ok, 1, nat.ptr(ix)) == LMPC_E_STATE
    c.enable_rollout(Tcl=1024)
    c.rollout_set_state(np.tile(X0, (Bs, 1)), np.tile(X0, (Bs, 1)))
    pid = lambda: c.rollout_pid_step(0.8, seed=1)                    # noqa: E731
    assert _launches(c, pid) == 2                                       # pid_input, sim_step
    c.set_observers([ObserverParams.uniform(0.5)], np.zeros(Bs))
    assert _launches(c, pid) == 3                                       # + observe
    c.set_measurement_noise([BASE], np.zeros(Bs, np.int32))
    assert _launches(c, pid) == 4                                       # + measure
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (Bs, 1)), np.tile(X0, (Bs, 1)))
    counts = {}
    for obs in (True, False):
        c.set_observers([ObserverParams.uniform(0.5)] if obs else None, np.zeros(Bs) if obs else None)
        for mode in (1, 0, 2):
            counts[(obs, mode)] = _launches(c, lambda: c.rollout_step(seed=5, mode=mode))
        counts[(obs, "pid")] = _launches(c, pid)
    for k in (1, 0, 2, "pid"):
        assert counts[(True, k)] == counts[(False, k)] + 1, (k, counts)
    with pytest.raises(ValueError):
        c.set_observers(None, np.zeros(Bs))                           # removing takes no index
    with pytest.raises(ValueError):
        c.set_observers(ROWS)                                         # rows need one
    with pytest.raises(ValueError):
        c.set_observers([ObserverParams(1, (0.5,) * 5 + (1.01,))], np.zeros(Bs))
    c.close()


@pytest.fixture(scope="module")
def identity_runs():
    """Shared streams (controllers 2k, 2k + 1 on stream k) and base measurement noise: no table, all-ones rows (installed, then
    refused calls), mode 0 rows with gains that are not read, and a real table removed by nsets == 0 before the first step."""
    _need_gpu()
    Bs = 64
    streams = np.arange(Bs) // 2
    out = {}
    for name in ("none", "ones", "mode0", "reverted"):
        if name == "none":
            c = _controller(Bs, streams=streams)
        elif name == "ones":
            c = _controller(Bs, obs=[ObserverParams.uniform(1.0), ObserverParams.gains(1, 1, 1, 1, 1, 1)],
                            oidx=np.arange(Bs) % 2, streams=streams)
            _reject(c)
        elif name == "mode0":
            c = _controller(Bs, obs=[ObserverParams(0, (0.0, 0.5, 0.25, 0.0, 0.1, 0.9)), ObserverParams.off()],
                            oidx=np.arange(Bs) % 2, streams=streams)
        else:
            c = _controller(Bs, obs=ROWS, oidx=np.arange(Bs) % 4, streams=streams)
            c.set_observers(None)
        _pid_lap_and_seed(c)
        if name == "ones":                                               # the table survived the refusals: one more launch
            out["ones_launch"] = _launches(c, lambda: c.rollout_step(seed=1234))
            c.rollout_commit_laps_dev()
        elif name == "none":
            out["none_launch"] = _launches(c, lambda: c.rollout_step(seed=1234))
            c.rollout_commit_laps_dev()
        else:
            _drive(c, 1)
        _drive(c, 349)
        out[name] = _result(c)
        c.close()
    return out


def test_all_ones_and_mode_zero_tables_equal_no_table(identity_runs):
    r = identity_runs
    sel = np.ones(64, bool)
    assert r["ones_launch"] == r["none_launch"] + 1
    assert r["none"]["books"]["lap_n"].max() >= 1                       # a finish line was crossed
    for name in ("ones", "mode0", "reverted"):
        _same(r[name], r["none"], sel, name)


# ---- 2. the restatement, step by step ---------------------------------------------------------------------------------------
def _trace_x(c, tr, cap):
    steps = C.c_int(0)
    x = np.zeros((cap, 6))
    nat.check(c._lib.lmpc_rollout_trace_get(c._h, tr, C.byref(steps), nat.ptr(x), None, None, None, None, None))
    return x[:steps.value]


def test_x_est_is_the_restatement_step_by_step():
    """PID lap, seeding and 400 LMPC steps: x_est equals the numpy restatement fed x_meas, xPredPrev and has_pred read before the
    step, bit for bit.  In the LMPC steps xPred[0] == x_est, the record's new row == x_est, addPoint's row == x_est + L e_s; the
    trace and rollout_state hold the plant state."""
    _need_gpu()
    Bs = 16
    idx = np.arange(Bs) % 4
    c = _controller(Bs, obs=ROWS, oidx=idx, meas=(MeasurementParams.scaled(3, BASE),))
    modes, gains = _tables(ROWS)
    modes, gains = modes[idx], gains[idx]
    mode1 = modes == 1
    for k in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
        y, xe = _read(c, "x_meas", (Bs, 6)), _read(c, "x_est", (Bs, 6))
        assert np.array_equal(xe, y), k
        assert np.all(_read(c, "has_pred", Bs, np.int32) == 0), k
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (Bs, 1)), np.tile(X0, (Bs, 1)))
    cap = 16
    inst = np.arange(4, dtype=np.int32)
    nat.check(nat.lib().lmpc_rollout_trace_create(c._h, len(inst), nat.ptr(inst), cap))
    wraps = blends = 0
    for k in range(400):
        hp = _read(c, "has_pred", Bs, np.int32)
        prior = _read(c, "xPredPrev", (Bs, N + 1, 6))[:, 1]
        x = c.rollout_state()["x"]
        if k == 0:
            assert np.all(hp == 0)                                    # the seeding leaves no prior
        c.rollout_step(seed=1234)
        y, xe = _read(c, "x_meas", (Bs, 6)), _read(c, "x_est", (Bs, 6))
        want, hp_after, fl = ob.observe(y, prior, hp, modes, gains, L)
        assert xe.tobytes() == want.tobytes(), k
        assert not fl.any()
        if k == 0:
            assert np.array_equal(xe, y)
        wraps += int(np.sum(mode1 & (hp == 1) & (prior[:, 4] - y[:, 4] > L / 2)))
        blends += int(np.sum(mode1 & (hp == 1)))
        xp = _read(c, "xPred", (Bs, N + 1, 6))
        assert np.array_equal(xp[:, 0], xe), k
        for b in range(Bs):
            xr, _ = c.rollout_get_lap(b)
            assert np.array_equal(xr[-1], xe[b]), (k, b)
        if k % 10 == 0:
            bk = c.books()
            full = (c.step_results()["flags"] & 16) != 0               # lap it-1 already holds Tmax rows: nothing appended
            for b in np.nonzero(~full)[0]:
                T = C.c_int(0)
                xs = np.zeros((1280, 6))
                nat.check(nat.lib().lmpc_ss_get_lap(c._h, int(b), int(bk["prev_slot"][b]), C.byref(T), nat.ptr(xs), None, None))
                assert np.array_equal(xs[T.value - 1], xe[b] + np.array([0, 0, 0, 0, L, 0])), (k, b)
        if k < cap:
            for t in range(4):
                assert np.array_equal(_trace_x(c, t, cap)[k], x[t]), (k, t)
        c.rollout_commit_laps_dev()
    assert blends > 0 and wraps > 0, (blends, wraps)                 # the prior was used, across a finish line too
    assert c.books()["lap_n"].max() >= 1
    c.close()


# ---- 3. edges ---------------------------------------------------------------------------------------------------------------
EDGE_ROWS = [ObserverParams.off(), ObserverParams.uniform(0.5), ObserverParams.uniform(1.0),
             ObserverParams.gains(1.0, 0.5, 0.5, 0.5, 0.5, 0.5)]


def test_pid_and_lti_steps_clear_the_prior_of_mode_one_rows_only():
    _need_gpu()
    Bs = 16
    idx = np.arange(Bs) % 4
    c = _controller(Bs, obs=EDGE_ROWS, oidx=idx)
    _pid_lap_and_seed(c)
    _drive(c, 20)
    mode1 = np.array([r.mode for r in EDGE_ROWS])[idx] == 1
    assert np.all(_read(c, "has_pred", Bs, np.int32) == 1)
    c.rollout_pid_step(0.8, seed=9)
    assert np.array_equal(_read(c, "has_pred", Bs, np.int32), (~mode1).astype(np.int32))
    assert np.array_equal(_read(c, "x_est", (Bs, 6)), _read(c, "x_meas", (Bs, 6)))
    c.rollout_step(seed=9)                                            # reads y, then has a prior again
    assert np.array_equal(_read(c, "x_est", (Bs, 6)), _read(c, "x_meas", (Bs, 6)))
    assert np.all(_read(c, "has_pred", Bs, np.int32) == 1)
    c.rollout_step(seed=9, mode=2)
    assert np.array_equal(_read(c, "has_pred", Bs, np.int32), (~mode1).astype(np.int32))
    assert np.array_equal(_read(c, "x_est", (Bs, 6)), _read(c, "x_meas", (Bs, 6)))
    c.close()


def test_a_non_finite_prior_reads_y_and_flags_the_step():
    """vx of every prior set to NaN through set_state: the uniform 0.5 rows read y and flag LMPC_FLAG_OBSERVER_RESET into the
    step flags, the health word and the lap report; mode 0, all-ones rows and the row with gain 1 on vx do not."""
    _need_gpu()
    Bs = 16
    idx = np.arange(Bs) % 4
    c = _controller(Bs, obs=EDGE_ROWS, oidx=idx)
    _pid_lap_and_seed(c)
    _drive(c, 20)
    xpp = _read(c, "xPredPrev", (Bs, N + 1, 6))
    hp = _read(c, "has_pred", Bs, np.int32)
    assert np.all(hp == 1)
    xpp[:, 1, 0] = np.nan
    c.set_state(xPred=xpp, has_pred=hp)
    prior = xpp[:, 1]
    lap_n0 = c.books()["lap_n"].copy()
    c.rollout_step(seed=1234)
    y, xe = _read(c, "x_meas", (Bs, 6)), _read(c, "x_est", (Bs, 6))
    modes, gains = _tables(EDGE_ROWS)
    want, _, fl = ob.observe(y, prior, hp, modes[idx], gains[idx], L)
    assert xe.tobytes() == want.tobytes()
    reset = idx == 1
    assert np.array_equal(fl != 0, reset)
    assert np.array_equal(xe[reset | (idx == 0) | (idx == 2)], y[reset | (idx == 0) | (idx == 2)])
    assert np.all(np.isfinite(xe))
    flags = c.step_results()["flags"]
    assert np.array_equal((flags & nat.FLAG_OBSERVER_RESET) != 0, reset)
    c.rollout_commit_laps_dev()
    health = c.rollout_health()[0]
    assert np.array_equal((health & nat.FLAG_OBSERVER_RESET) != 0, reset)
    for _ in range(600):
        c.rollout_step(seed=1234)
        c.rollout_commit_laps_dev()
        assert not (c.step_results()["flags"] & nat.FLAG_OBSERVER_RESET).any()      # the next prior is finite again
        if (c.books()["lap_n"] > lap_n0).all():
            break
    rep = c.lap_reports()
    assert np.all(rep["n"] > lap_n0)
    got = np.array([(rep["flags"][b, lap_n0[b]] & nat.FLAG_OBSERVER_RESET) != 0 for b in range(Bs)])
    assert np.array_equal(got, reset)
    c.close()


def test_retired_controllers_write_nothing():
    _need_gpu()
    Bs = 32
    c = _controller(Bs, obs=ROWS, oidx=np.arange(Bs) % 4)
    _pid_lap_and_seed(c)
    budget = np.where(np.arange(Bs) % 2 == 0, 1, 3).astype(np.int32)
    c.set_lap_budget(budget)
    for k in range(600):
        c.rollout_step(seed=77)
        c.rollout_commit_laps_dev()
        if k % 8 == 7 and (c.books()["lap_n"][0::2] >= 1).all():
            break
    ret = np.nonzero(c.books()["lap_n"] >= budget)[0]
    assert ret.size == Bs // 2 and np.all(ret % 2 == 0)

    def snap():
        st = c.rollout_state()
        xe = _read(c, "x_est", (Bs, 6))
        hp = _read(c, "has_pred", Bs, np.int32)
        rec = [np.frombuffer(b"".join(a.tobytes() for a in c.rollout_get_lap(int(b))), np.uint8) for b in ret]
        return st, xe, hp, rec, c.rollout_health()[0]
    s0 = snap()
    _drive(c, 40, seed=77)
    s1 = snap()
    for key in ("x", "xglob", "done", "cl_len"):
        assert np.array_equal(s0[0][key][ret], s1[0][key][ret]), key
    assert s0[1][ret].tobytes() == s1[1][ret].tobytes()
    assert np.array_equal(s0[2][ret], s1[2][ret]) and np.array_equal(s0[4][ret], s1[4][ret])
    assert all(np.array_equal(a, b) for a, b in zip(s0[3], s1[3]))
    live = np.setdiff1d(np.arange(Bs), ret)
    assert not np.array_equal(s0[1][live], s1[1][live])
    c.close()


# ---- 4. batches -------------------------------------------------------------------------------------------------------------
def test_batch_of_observer_rows_equals_one_handle_per_row():
    _need_gpu()
    Bs = 64
    idx = np.arange(Bs) % 4
    n, het, het_laps = cl.run(Bs, hook=observed(ROWS, idx))
    assert (het["lap_n"] >= 1).mean() > 0.9
    for k in range(4):
        ref = cl.run(Bs, hook=observed([ROWS[k]], np.zeros(Bs, np.int32)), steps=n)[1:]
        cl.same((het, het_laps), ref, idx == k, "observer row %d" % k)


def _tunings():
    import copy
    _, _, _, _, Qts, base = rp.lmpc_params(N)
    ps = []
    for k in range(2):
        p = copy.deepcopy(base)
        p.dR = (0.5, 2.0)[k] * np.asarray(base.dR, float)
        ps.append(p)
    return ps, Qts


def test_crossed_with_measurement_sets_and_tunings():
    """2 observer rows x 2 measurement sets x 2 QP tunings in one batch equal one handle per combination."""
    _need_gpu()
    Bs = 64
    b = np.arange(Bs)
    oidx, midx, pidx = b % 2, (b // 2) % 2, (b // 4) % 2
    obs = [ObserverParams.uniform(0.5), ObserverParams.from_noise(0.01, 0.03)]
    meas = [BASE, MeasurementParams.scaled(3, BASE)]
    ps, Qts = _tunings()

    def hook(o_rows, o_idx, m_rows, m_idx):
        def h(c):
            enable = c.enable_rollout

            def enable_then(Tcl=512):
                enable(Tcl)
                c.set_measurement_noise(m_rows, m_idx)
                c.set_observers(o_rows, o_idx)
            c.enable_rollout = enable_then
        return h
    n, het, het_laps = cl.run(Bs, psets=(ps, pidx, [Qts, Qts]), hook=hook(obs, oidx, meas, midx))
    assert (het["lap_n"] >= 1).mean() > 0.9
    z = np.zeros(Bs, np.int32)
    for o in range(2):
        for m in range(2):
            for p in range(2):
                ref = cl.run(Bs, par=ps[p], qts=Qts, hook=hook([obs[o]], z, [meas[m]], z), steps=n)[1:]
                cl.same((het, het_laps), ref, (oidx == o) & (midx == m) & (pidx == p), "observer %d meas %d tuning %d" % (o, m, p))


# ---- 5. snapshots -----------------------------------------------------------------------------------------------------------
def test_snapshot_restore_and_clone_continue_exactly():
    """With a table: snapshot after 150 LMPC steps, restore into a fresh handle with the same tables and clock, 200 more steps
    equal the straight run bit for bit.  Cloning controllers 0..15 onto 16..31 (same streams and rows) makes them follow."""
    _need_gpu()
    Bs = 32
    streams = np.arange(Bs) % 16
    idx = (np.arange(Bs) % 16) % 4
    c = _controller(Bs, obs=ROWS, oidx=idx, streams=streams)
    _pid_lap_and_seed(c)
    _drive(c, 150)
    rec = c.snapshot().clone()
    clock = c.rollout_clock
    _drive(c, 200)
    straight = _result(c)
    c.close()

    d = _controller(Bs, obs=ROWS, oidx=idx, streams=streams)
    d.restore(rec)
    d.rollout_clock = clock
    _drive(d, 200)
    _same(_result(d), straight, np.ones(Bs, bool), "restored")
    d.close()

    e = _controller(Bs, obs=ROWS, oidx=idx, streams=streams)
    _pid_lap_and_seed(e)
    _drive(e, 150)
    e.clone(np.arange(16), np.arange(16, 32))
    _drive(e, 200)
    r = _result(e, records=False)
    st, bk = r["state"], r["books"]
    for key in ("x", "xglob", "done", "cl_len"):
        assert np.array_equal(st[key][:16], st[key][16:]), key
    for key in ("lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt"):
        assert np.array_equal(bk[key][:16], bk[key][16:]), key
    assert np.array_equal(_read(e, "x_est", (Bs, 6))[:16], _read(e, "x_est", (Bs, 6))[16:])
    e.close()
