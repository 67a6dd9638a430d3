"""GPU tier: per-controller measurement noise of the device closed loop (lmpc_rollout_set_measurement_noise).

Without a table nothing changes: no kernel is added and the closed loop is the one of a handle that never heard of measurements;
an all-zero set launches the kernel and still equals no table bit for bit, and nsets == 0 reverts.  With a table everything the
controller knows comes through y = x + clip(z * sigma, +-clip): the PID's input, the QP's x0, addPoint's row and the record's state
rows, while the plant, rollout_state and the trace keep x.  The draws have the clipped form per channel in the channel order, are
uncorrelated with the process and PID draws, and pair on the noise streams.  A batch of sets is one handle per set, retired
controllers draw nothing and write nothing, and a run captured and resumed with measurement noise equals a straight run."""
import copy
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                # noqa: E402
from racinglmpc_b200 import _native as nat                        # noqa: E402
from racinglmpc_b200.reference_params import MeasurementParams, NoiseParams   # noqa: E402
import closed_loop as cl                                          # noqa: E402
import noise_model as nm                                          # noqa: E402
from closed_loop import N, X0                                     # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LMPC_E_INVALID, LMPC_E_STATE = -1, -4
B = 256
# the base set of the benchmark: 1 cm (m/s, rad/s) on velocities, positions and s, 5 mrad on epsi; clip at five sigma
BASE = MeasurementParams((0.01, 0.01, 0.01, 0.005, 0.01, 0.01), (0.05, 0.05, 0.05, 0.025, 0.05, 0.05))
FOUR = [MeasurementParams.zero(), BASE, MeasurementParams.scaled(3, BASE),
        MeasurementParams((0.02, 0.0, 0.01, 0.002, 0.03, 0.0), (0.01, 0.0, 0.05, 0.1, 0.02, 0.0))]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def measured(meas, index, then=None):
    """A closed_loop.run hook: the measurement table goes in right after enable_rollout (it belongs to the closed loop), then
    ``then(c)`` runs, if given."""
    def hook(c):
        enable = c.enable_rollout

        def enable_then_measure(Tcl=512):
            enable(Tcl)
            c.set_measurement_noise(meas, index)
            if then is not None:
                then(c)
        c.enable_rollout = enable_then_measure
    return hook


class _Fake:
    def __init__(self, z):
        self._it = iter(np.asarray(z, float).ravel())

    def standard_normal(self):
        return next(self._it)


def _controller(Bs, **kw):
    c = cl.controller(Bs, **kw)
    c.enable_rollout(Tcl=1024)
    c.rollout_set_state(np.tile(X0, (Bs, 1)), np.tile(X0, (Bs, 1)))
    return c


def _reject(c):
    """Refused calls, each returning LMPC_E_INVALID; the handle must stay as it was."""
    L = nat.lib()
    idx = np.arange(c.B, dtype=np.int32) % 4
    good, _ = nat.make_measurement_sets(FOUR, idx, c.B)

    def copy_of(mod):
        t = (nat.MeasurementParams * 4)()
        C.memmove(t, good, C.sizeof(t))
        mod(t)
        return t
    bad = [copy_of(lambda t: t[1].sigma.__setitem__(5, -0.01)), copy_of(lambda t: t[2].clip.__setitem__(0, float("nan"))),
           copy_of(lambda t: t[3].sigma.__setitem__(3, float("inf"))), copy_of(lambda t: t[0].clip.__setitem__(4, -1e-300))]
    cases = [(t, 4, idx) for t in bad] + [(good, 4, np.full(c.B, 4, np.int32)), (good, 4, np.full(c.B, -1, np.int32)),
                                          (good, 0, idx), (None, 4, idx), (good, 4, None)]
    for tab, n, ix in cases:
        assert L.lmpc_rollout_set_measurement_noise(c._h, tab, n, nat.ptr(ix) if ix is not None else None) == LMPC_E_INVALID
    big = (nat.MeasurementParams * (c.B + 1))(*([good[0]] * (c.B + 1)))
    assert L.lmpc_rollout_set_measurement_noise(c._h, big, c.B + 1, nat.ptr(np.zeros(c.B, np.int32))) == LMPC_E_INVALID


# ---- 1. no table, zero set, revert ------------------------------------------------------------------------------------------
def test_table_needs_the_closed_loop_and_launches_one_kernel_per_step():
    _need_gpu()
    c = cl.controller(8)
    L = nat.lib()
    ok, _ = nat.make_measurement_sets([BASE], np.zeros(8, np.int32), 8)
    assert L.lmpc_rollout_set_measurement_noise(c._h, ok, 1, nat.ptr(np.zeros(8, np.int32))) == LMPC_E_STATE
    c.enable_rollout(Tcl=64)
    c.rollout_set_state(np.tile(X0, (8, 1)), np.tile(X0, (8, 1)))

    def launches(f):
        l0 = c.kernel_launches
        f()
        return c.kernel_launches - l0
    pid = lambda: c.rollout_pid_step(0.8, seed=1)                    # noqa: E731
    assert launches(pid) == 2                                           # pid_input, sim_step: as before
    c.set_measurement_noise([MeasurementParams.zero()], np.zeros(8, np.int32))
    assert launches(pid) == 3                                           # + measure
    c.set_measurement_noise(None)
    assert launches(pid) == 2
    c.close()


@pytest.fixture(scope="module")
def base_runs():
    """No table; an all-zero set installed after refused calls; a set installed then reverted by nsets == 0."""
    _need_gpu()
    n, none, none_laps = cl.run(B)
    assert none["lap_n"].min() >= 1
    zero = cl.run(B, hook=measured([MeasurementParams.zero()], np.zeros(B, np.int32), then=_reject), steps=n)[1:]

    def revert(c):
        with pytest.raises(ValueError):
            c.set_measurement_noise(None, np.zeros(B))            # reverting takes no index
        with pytest.raises(ValueError):
            c.set_measurement_noise(FOUR)                         # sets need one
        c.set_measurement_noise(None)
    reverted = cl.run(B, hook=measured(FOUR, np.arange(B) % 4, then=revert), steps=n)[1:]
    noisy = cl.run(B, hook=measured([BASE], np.zeros(B, np.int32)), steps=n)[1:]
    return dict(n=n, none=(none, none_laps), zero=zero, reverted=reverted, noisy=noisy)


def test_zero_set_and_revert_equal_no_table(base_runs):
    every = np.ones(B, bool)
    cl.same(base_runs["zero"], base_runs["none"], every, "all-zero set vs no table")
    cl.same(base_runs["reverted"], base_runs["none"], every, "nsets == 0 reverts")
    # and the noise acts
    assert not np.array_equal(base_runs["noisy"][0]["x"], base_runs["none"][0]["x"])


def _rollout_mc():
    sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
    try:
        import rollout_mc
    finally:
        sys.path.pop(0)
    return rollout_mc


def test_zero_set_equals_no_table_in_the_monte_carlo_driver():
    """Books, end state, health, solver report and snapshot records of rollout_mc.run: an all-zero set equals no table."""
    _need_gpu()
    rm = _rollout_mc()
    Bs = 256
    out = []
    for meas in (None, ([MeasurementParams.zero()], np.zeros(Bs, np.int32))):
        fin, bk, cap = {}, {}, {}
        o = rm.run(batch=Bs, laps=1, mode="independent", local=0, final=fin, books=bk, capture=cap, measurement_sets=meas)
        out.append((o, fin, bk, cap))
    (o0, f0, b0, c0), (o1, f1, b1, c1) = out
    for k in f0:
        assert np.array_equal(np.asarray(f0[k]), np.asarray(f1[k])), ("end state / solver report", k)
    for k in b0:
        assert np.array_equal(np.asarray(b0[k]), np.asarray(b1[k])), ("books", k)
    assert torch.equal(c0["records"], c1["records"])
    for k in ("closed_loop_steps", "lap_stats_rank0", "instances_with_flags_rank0", "unsolved_steps_rank0"):
        assert o0[k] == o1[k], k
    assert len(o1["per_measurement_rank0"]) == 1 and "per_measurement_rank0" not in o0


# ---- 2. routing in the PID lap -------------------------------------------------------------------------------------------------
def test_pid_lap_follows_the_test_side_model_fed_the_measurements(track):
    """Host-given PID and process draws, Philox measurements: the test-side PID fed y and dynModel on x follow the device to
    1e-12 after one step and 1e-9 after 300; the record's state rows are the y's bit for bit; rollout_state holds x."""
    _need_gpu()
    Bs, K = 16, 300
    meas = [MeasurementParams.scaled(k, BASE) for k in (0, 1, 2, 5)]
    idx = np.arange(Bs) % 4
    c = _controller(Bs)
    c.set_measurement_noise(meas, idx)
    zs = np.random.default_rng(17).standard_normal((Bs, K, 5))
    car, noise = rp.VehicleParams.reference(), NoiseParams.reference()
    xs, gs = np.tile(X0, (Bs, 1)), np.tile(X0, (Bs, 1))
    ys = np.zeros((K, Bs, 6))
    prev = np.tile(X0, (Bs, 1))
    for k in range(K):
        c.rollout_pid_step(0.8, z_pid=zs[:, k, 0:2], z_sim=zs[:, k, 2:5], seed=99)
        y = np.stack([c.read_buffer("x_meas", b, (6,)) for b in range(Bs)])
        ys[k] = y
        for b in range(Bs):
            fake = _Fake(zs[b, k])
            pid = nm.PIDFollower(0.8, noise, rng=fake)
            pid.solve(y[b])
            xs[b], gs[b] = nm.dyn_model(track, xs[b], gs[b], pid.uPred[0], car, noise, rng=fake)
        st = c.rollout_state()
        tol = 1e-12 if k == 0 else 1e-9
        assert np.max(np.abs(st["x"] - xs)) < tol and np.max(np.abs(st["xglob"] - gs)) < tol, k
        # set 0 measures the plant exactly, the others do not
        assert np.array_equal(y[idx == 0], prev[idx == 0]) and not np.array_equal(y[idx == 1], prev[idx == 1]), k
        prev = st["x"]
    for b in range(Bs):
        xr, _ = c.rollout_get_lap(b)
        assert xr.shape[0] == K and np.array_equal(xr, ys[:, b]), b
    c.close()


def test_zero_channels_measure_the_plant_and_the_record_keeps_it():
    """With set 0 (all zero) y equals x exactly at every step: the record equals the plant's states."""
    _need_gpu()
    Bs = 8
    c = _controller(Bs)
    c.set_measurement_noise([MeasurementParams.zero(), BASE], np.arange(Bs) % 2)
    prev = np.tile(X0, (Bs, 1))
    for k in range(20):
        c.rollout_pid_step(0.8, seed=3)
        y = np.stack([c.read_buffer("x_meas", b, (6,)) for b in range(Bs)])
        assert np.array_equal(y[0::2], prev[0::2]) and not np.array_equal(y[1::2], prev[1::2]), k
        prev = c.rollout_state()["x"]
    c.close()


# ---- 3. routing in modes 0, 1, 2 -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [1, 0, 2])
def test_controller_steps_take_the_measurement(mode):
    """xPred[0] == y, the record's rows equal y, addPoint's row equals y + [0,0,0,0,L,0] (mode 1), the trace and rollout_state
    hold the plant state x."""
    _need_gpu()
    Bs = 32
    c = _controller(Bs)
    c.set_measurement_noise([MeasurementParams.scaled(10, BASE)], np.zeros(Bs, np.int32))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    if mode == 2:
        c.rollout_sysid()
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (Bs, 1)), np.tile(X0, (Bs, 1)))
    inst = np.arange(4, dtype=np.int32)
    nat.check(nat.lib().lmpc_rollout_trace_create(c._h, len(inst), nat.ptr(inst), 16))
    L = float(rp.TrackParams.l_shaped().TrackLength)
    for k in range(8):
        x = c.rollout_state()["x"]
        c.rollout_step(seed=1234 + k, mode=mode)
        y = np.stack([c.read_buffer("x_meas", b, (6,)) for b in range(Bs)])
        assert not np.array_equal(y, x)
        for b in range(Bs):
            xp = c.read_buffer("xPred", b, (N + 1, 6))
            assert np.array_equal(xp[0], y[b]), (mode, k, b)
            xr, _ = c.rollout_get_lap(b)
            assert xr.shape[0] == k + 1 and np.array_equal(xr[k], y[b]), (mode, k, b)
        if mode == 1:
            bk = c.books()
            for b in range(Bs):
                T = C.c_int(0)
                xs = np.zeros((1280, 6))
                nat.check(nat.lib().lmpc_ss_get_lap(c._h, b, int(bk["prev_slot"][b]), C.byref(T), nat.ptr(xs), None, None))
                assert np.array_equal(xs[T.value - 1], y[b] + np.array([0, 0, 0, 0, L, 0])), (k, b)
        for t in range(4):
            tr = np.asarray(_trace_x(c, t))
            assert tr.shape[0] == k + 1 and np.array_equal(tr[k], x[t]), (mode, k, t)
    c.close()


def _trace_x(c, tr):
    steps = C.c_int(0)
    x = np.zeros((16, 6))
    nat.check(c._lib.lmpc_rollout_trace_get(c._h, tr, C.byref(steps), nat.ptr(x), None, None, None, None, None))
    return x[:steps.value]


# ---- 4. the clipped form, the channel order, the statistics ---------------------------------------------------------------
def test_saturating_and_zero_sigma_channels_are_exact():
    """Huge sigma, a different small clip per channel: y == x +- clip_j exactly, on every channel, in the channel order; a
    zero-sigma channel gives y == x."""
    _need_gpu()
    Bs = 512
    clip = np.array([1, 2, 3, 4, 5, 6]) * 1e-3
    sat = MeasurementParams((1e6,) * 6, tuple(clip))
    half = MeasurementParams((1e6, 0.0, 1e6, 0.0, 1e6, 0.0), tuple(clip))
    c = _controller(Bs)
    c.set_measurement_noise([sat, half], np.arange(Bs) % 2)
    signs = []
    for k in range(10):
        x = c.rollout_state()["x"]
        c.rollout_pid_step(0.8, seed=5)
        y = np.stack([c.read_buffer("x_meas", b, (6,)) for b in range(Bs)])
        up, down = y == x + clip, y == x - clip
        assert np.all(up[0::2] | down[0::2]), k
        assert np.all((up | down)[1::2][:, 0::2]) and np.array_equal(y[1::2][:, 1::2], x[1::2][:, 1::2]), k
        signs.append(up[0::2])
    s = np.asarray(signs, float)
    assert np.all(np.abs(s.mean(axis=(0, 1)) - 0.5) < 0.05)      # both signs, on every channel
    c.close()


def _clipped_normal(sig, clip):
    a = clip / sig
    phi, Phi = math.exp(-a * a / 2) / math.sqrt(2 * math.pi), 0.5 * (1 + math.erf(a / math.sqrt(2)))
    var = sig * sig * ((2 * Phi - 1) - 2 * a * phi) + clip * clip * 2 * (1 - Phi)
    return var, 2 * (1 - Phi)


def test_moments_and_independence_from_the_process_and_pid_draws():
    """8192 controllers x 50 steps at a fixed seed, each step from one state: the moments of y - x match the clipped normal per
    channel, and y - x is uncorrelated with the process noise (the plant's difference to a handle without process noise) and the
    PID noise (the applied input minus the PID law of y)."""
    _need_gpu()
    Bs, K = 8192, 50
    sig = np.array([0.01, 0.02, 0.03, 0.005, 0.04, 0.015])
    clp = sig * np.array([1.0, 1.5, 2.0, 0.5, 3.0, 1.2])
    meas = MeasurementParams(tuple(sig), tuple(clp))
    big = NoiseParams((0.01, 0.01, 0.005), (0.05, 0.05, 0.05), 1.0, (0.25, 0.10), (0.9, 0.2))
    quiet = NoiseParams((0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 1.0, (0.25, 0.10), (0.9, 0.2))
    cs = []
    for noise in (big, quiet):
        c = _controller(Bs, Tmax=64, ss_cap=6, model_cap=5)
        c.set_noise([noise], np.zeros(Bs, np.int32))
        c.set_measurement_noise([meas], np.zeros(Bs, np.int32))
        cs.append(c)
    x0 = np.tile(np.array([0.8, 0.01, 0.02, 0.01, 3.0, 0.05]), (Bs, 1))
    nmeas, nproc, npid = [], [], []
    for k in range(K):
        for c in cs:
            c.rollout_set_state(x0, x0)
            c.rollout_pid_step(0.8, seed=2024)
        y = np.frombuffer(_read_all(cs[0], "x_meas", Bs * 6), np.float64).reshape(Bs, 6)
        y1 = np.frombuffer(_read_all(cs[1], "x_meas", Bs * 6), np.float64).reshape(Bs, 6)
        assert np.array_equal(y, y1)                                 # the process noise does not move the measurement draws
        nmeas.append(y - x0)
        nproc.append(cs[0].rollout_state()["x"][:, :3] - cs[1].rollout_state()["x"][:, :3])
        u = np.stack([_last_u(cs[0], b, k) for b in range(0, Bs, 16)])
        ys = y[0::16]
        law = np.stack([-0.6 * ys[:, 5] - 0.9 * ys[:, 3], 1.5 * (0.8 - ys[:, 0])], axis=1)
        npid.append(np.concatenate([u - law, nmeas[-1][0::16]], axis=1))
    nm_ = np.concatenate(nmeas)
    npr = np.concatenate(nproc)
    npd = np.concatenate(npid)
    n = nm_.shape[0]
    for j in range(6):
        var, p_sat = _clipped_normal(sig[j], clp[j])
        v = nm_[:, j]
        assert abs(v.mean()) < 5 * math.sqrt(var / n), j
        assert abs((v * v).mean() / var - 1) < 0.02, (j, (v * v).mean(), var)
        sat = np.isclose(np.abs(v), clp[j], rtol=0, atol=1e-13)
        assert abs(sat.mean() - p_sat) < 5 * math.sqrt(p_sat * (1 - p_sat) / n) + 1e-3, (j, sat.mean(), p_sat)
    assert np.std(npr, axis=0).min() > 1e-3                             # the process noise is there
    cor = np.corrcoef(np.concatenate([nm_, npr], axis=1).T)[:6, 6:]
    assert np.max(np.abs(cor)) < 0.01, cor
    cor = np.corrcoef(npd.T)[:2, 2:]
    assert np.max(np.abs(cor)) < 0.04, cor
    for c in cs:
        c.close()


def _read_all(c, name, n):
    out = np.zeros(n)
    nat.check(c._lib.lmpc_read_buffer(c._h, name.encode(), 0, nat.ptr(out), out.nbytes))
    return out.tobytes()


def _last_u(c, b, k):
    _, u = c.rollout_get_lap(b)
    return u[k]


# ---- 5. batches and crossed tables ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def four_runs():
    _need_gpu()
    midx = np.arange(B) % 4
    n, het, het_laps = cl.run(B, hook=measured(FOUR, midx))
    # the noisiest sets may keep a few controllers from their first lap within the run; they are compared all the same
    assert (het["lap_n"] >= 1).mean() > 0.9, "most controllers finish an LMPC lap in %d steps" % n
    refs = [cl.run(B, hook=measured([m], np.zeros(B, np.int32)), steps=n)[1:] for m in FOUR]
    return dict(n=n, midx=midx, het=(het, het_laps), refs=refs)


def test_batch_of_measurement_sets_equals_one_handle_per_set(four_runs):
    for k in range(4):
        cl.same(four_runs["het"], four_runs["refs"][k], four_runs["midx"] == k, "measurement set %d" % k)
    h = four_runs["het"][0]
    assert len({float(h["lap_hist"][four_runs["midx"] == k, 0].mean()) for k in range(4)}) >= 3


def test_traced_batch_gives_the_same_results(four_runs):
    _, het, laps = cl.run(B, hook=measured(FOUR, four_runs["midx"]), steps=four_runs["n"], trace=True)
    for k in range(4):
        cl.same((het, laps), four_runs["refs"][k], four_runs["midx"] == k, "traced, measurement set %d" % k)


def _tunings():
    _, _, _, _, Qts, base = rp.lmpc_params(N)
    ps = []
    for k in range(2):
        p = copy.deepcopy(base)
        p.dR = (0.5, 2.0)[k] * np.asarray(base.dR, float)
        ps.append(p)
    return ps, Qts


def test_crossed_with_tunings_and_cars():
    """2 measurement sets x 2 QP tunings x 2 cars in one batch equal one handle per combination."""
    _need_gpu()
    Bs = 64
    b = np.arange(Bs)
    midx, pidx, vidx = b % 2, (b // 2) % 2, (b // 4) % 2
    meas = [MeasurementParams.scaled(0.5, BASE), BASE]
    ps, Qts = _tunings()
    cars = [rp.VehicleParams.reference(), rp.VehicleParams.from_friction(0.6)]
    n, het, het_laps = cl.run(Bs, psets=(ps, pidx, [Qts, Qts]), vehicles=cars, vidx=vidx, hook=measured(meas, midx))
    assert (het["lap_n"] >= 1).mean() > 0.9
    for m in range(2):
        for p in range(2):
            for v in range(2):
                ref = cl.run(Bs, par=ps[p], qts=Qts, vehicles=[cars[v]], vidx=np.zeros(Bs, np.int32),
                             hook=measured([meas[m]], np.zeros(Bs, np.int32)), steps=n)[1:]
                cl.same((het, het_laps), ref, (midx == m) & (pidx == p) & (vidx == v), "set %d tuning %d car %d" % (m, p, v))


# ---- 6. streams -------------------------------------------------------------------------------------------------------------
def _same_mapped(a, b, dst, src, what):
    (ar, _), (br, _) = a, b
    for key in cl.KEYS:
        assert np.array_equal(ar[key][dst], br[key][src]), (what, key)


def test_streams_move_the_measurements(base_runs):
    """Every controller on stream 0 drives controller 0's closed loop; a permutation of streams permutes the closed loops."""
    n, b = base_runs["n"], np.arange(B)
    one = [BASE]
    zero = cl.run(B, hook=measured(one, np.zeros(B, np.int32), then=lambda c: c.set_noise_streams(np.zeros(B, np.int32))),
                  steps=n)[1:]
    _same_mapped(zero, base_runs["noisy"], b, np.zeros(B, int), "stream 0 everywhere")
    perm = np.random.default_rng(5).permutation(B)
    p = cl.run(B, hook=measured(one, np.zeros(B, np.int32), then=lambda c: c.set_noise_streams(perm)), steps=n)[1:]
    _same_mapped(p, base_runs["noisy"], b, perm, "permuted streams")


def test_tuning_pairs_on_one_stream_see_the_same_measurement_noise():
    """Two tunings interleaved on streams b // 2: the pair's measurement noise y - x is the same at every step, while their
    closed loops differ."""
    _need_gpu()
    Bs = 64
    b = np.arange(Bs)
    ps, Qts = _tunings()
    c = _controller(Bs)
    c.set_param_sets(ps, b % 2, [Qts, Qts])
    c.set_noise_streams(b // 2)
    c.set_measurement_noise([MeasurementParams.scaled(10, BASE)], np.zeros(Bs, np.int32))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (Bs, 1)), np.tile(X0, (Bs, 1)))
    for k in range(120):
        x = c.rollout_state()["x"]
        c.rollout_step(seed=1234)
        c.rollout_commit_laps_dev()
        y = np.frombuffer(_read_all(c, "x_meas", Bs * 6), np.float64).reshape(Bs, 6)
        nz = y - x
        assert np.max(np.abs(nz[0::2] - nz[1::2])) < 1e-12, k
    assert not np.array_equal(x[0::2], x[1::2])
    c.close()


# ---- 7. lap budgets ---------------------------------------------------------------------------------------------------------
def test_retired_controllers_draw_nothing_and_write_nothing():
    _need_gpu()
    Bs = 64
    c = _controller(Bs)
    c.set_measurement_noise([BASE], np.zeros(Bs, np.int32))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (Bs, 1)), np.tile(X0, (Bs, 1)))
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
        y = np.frombuffer(_read_all(c, "x_meas", Bs * 6), np.float64).reshape(Bs, 6)
        rec = [np.frombuffer(b"".join(a.tobytes() for a in c.rollout_get_lap(int(b))), np.uint8) for b in ret]
        return st, y.copy(), rec
    st0, y0, rec0 = snap()
    for _ in range(40):
        c.rollout_step(seed=77)
        c.rollout_commit_laps_dev()
    st1, y1, rec1 = snap()
    for key in ("x", "xglob", "done", "cl_len"):
        assert np.array_equal(st0[key][ret], st1[key][ret]), key
    assert np.array_equal(y0[ret], y1[ret])
    assert all(np.array_equal(a, b) for a, b in zip(rec0, rec1))
    live = np.setdiff1d(np.arange(Bs), ret)
    assert not np.array_equal(y0[live], y1[live]) and not np.array_equal(st0["x"][live], st1["x"][live])
    c.close()


# ---- 8. snapshots -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pooled", [False, True])
def test_capture_and_resume_with_measurement_noise(pooled):
    """rollout_mc.run with measurement noise: 1 lap captured and resumed to 2 equals a straight run to 2 laps (books, end states,
    health, exchange steps); pooled under group readiness too."""
    _need_gpu()
    rm = _rollout_mc()
    Bs = 256
    kw = dict(batch=Bs, local=0, measurement_sets=(FOUR, np.arange(Bs) % 4))
    if pooled:
        kw.update(mode="pooled", readiness="group", pool_groups=((np.arange(Bs) // 4) % 4, 4))   # every group holds all four sets
    else:
        kw.update(mode="independent")
    fin2, bk2, cap2 = {}, {}, {}
    o2 = rm.run(laps=2, final=fin2, books=bk2, capture=cap2, **kw)
    cap = {}
    rm.run(laps=1, capture=cap, **kw)
    assert cap["diverged_step"] is None
    fin, bk, capr = {}, {}, {}
    o = rm.run(laps=2, start=cap, final=fin, books=bk, capture=capr, **kw)
    assert o["resume_exact"] and o["closed_loop_steps"] == o2["closed_loop_steps"]
    assert capr["exchange_steps"] == cap2["exchange_steps"]
    assert torch.equal(capr["records"], cap2["records"])
    for k in bk2:
        assert np.array_equal(np.asarray(bk2[k]), np.asarray(bk[k])), ("books", k)
    for k in fin2:
        assert np.array_equal(np.asarray(fin2[k]), np.asarray(fin[k])), ("end state", k)
    for k in ("lap_stats_rank0", "per_measurement_rank0", "instances_with_flags_rank0", "unsolved_steps_rank0"):
        assert o2.get(k) == o.get(k), k
    assert len(o2["per_measurement_rank0"]) == 4
