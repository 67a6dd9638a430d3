"""CPU tier: the per-controller state observers (lmpc_rollout_set_observers) -- packing and refusals of make_observer_sets, the
ABI size, ObserverParams and its steady-state Kalman gain, and the numpy restatement of the observer the GPU tests compare
against (tests/support/observer.py)."""
import ctypes as C
import math

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat
from racinglmpc_b200.reference_params import ObserverParams, TRACK_LENGTH
import observer as ob

B = 8


def test_struct_size_matches_the_library():
    assert C.sizeof(nat.ObserverParams) == 56
    assert nat.lib().lmpc_sizeof_observer_params() == C.sizeof(nat.ObserverParams)
    assert nat.FLAG_OBSERVER_RESET == ob.FLAG_OBSERVER_RESET == 2048
    assert nat.FLAG_OBSERVER_RESET & (nat.FLAG_NOMINAL_NONFINITE | 512 | 256 | 128 | 64 | 32 | 16 | 8 | 4 | 2 | 1) == 0


def test_packing():
    rows = [ObserverParams.off(), ObserverParams.uniform(0.5), ObserverParams.gains(0, 0.1, 0.2, 0.3, 0.4, 1)]
    idx = np.arange(B) % 3
    tab, ix = nat.make_observer_sets(rows, idx, B)
    assert len(tab) == 3 and ix.dtype == np.int32 and np.array_equal(ix, idx)
    assert tab[0].mode == 0 and list(tab[0].gain) == [1.0] * 6
    assert tab[1].mode == 1 and list(tab[1].gain) == [0.5] * 6
    assert tab[2].mode == 1 and list(tab[2].gain) == [0, 0.1, 0.2, 0.3, 0.4, 1] and tab[2].pad == 0


@pytest.mark.parametrize("row", [
    ObserverParams(2, (1.0,) * 6), ObserverParams(-1, (1.0,) * 6), ObserverParams(True, (1.0,) * 6),
    ObserverParams(1.0, (1.0,) * 6), ObserverParams(1, (1.0,) * 5), ObserverParams(1, (1.0,) * 7),
    ObserverParams(1, (0.5, 0.5, float("nan"), 0.5, 0.5, 0.5)), ObserverParams(1, (0.5, float("inf"), 0.5, 0.5, 0.5, 0.5)),
    ObserverParams(1, (0.5, 0.5, 0.5, -1e-300, 0.5, 0.5)), ObserverParams(1, (0.5, 0.5, 0.5, 0.5, 1.0 + 2 ** -52, 0.5)),
    ObserverParams(0, (2.0,) * 6)])
def test_bad_rows_are_refused(row):
    with pytest.raises(ValueError):
        nat.make_observer_sets([ObserverParams.off(), row], np.arange(B) % 2, B)


@pytest.mark.parametrize("rows, idx", [
    ([ObserverParams.off()], np.ones(B)), ([ObserverParams.off()], -np.ones(B)), ([ObserverParams.off()], np.zeros(B - 1)),
    ([ObserverParams.off()], np.full(B, 0.5)), ([], np.zeros(B)), ([ObserverParams.off()] * (B + 1), np.zeros(B)),
    ([ObserverParams.off()], None)])
def test_bad_indices_are_refused(rows, idx):
    with pytest.raises(ValueError):
        nat.make_observer_sets(rows, idx, B)


def test_constructors():
    assert ObserverParams.off() == ObserverParams(0, (1.0,) * 6)
    assert ObserverParams.uniform(0.25) == ObserverParams(1, (0.25,) * 6)
    assert ObserverParams.gains(1, 2 ** -3, 0, 1, 0.5, 0.75).gain == (1.0, 0.125, 0.0, 1.0, 0.5, 0.75)


def _riccati_gain(q, r, iters=100000):
    """The scalar random walk's Kalman filter run to its fixed point: prior P-, gain l = P- / (P- + r), posterior
    (1 - l) P-, next prior posterior + q."""
    P = q + r
    for _ in range(iters):
        l = P / (P + r)
        Pn = (1.0 - l) * P + q
        if abs(Pn - P) <= 1e-16 * P:
            break
        P = Pn
    return P / (P + r)


@pytest.mark.parametrize("model_sigma, meas_sigma", [(0.01, 0.01), (0.003, 0.1), (0.1, 0.003), (1e-4, 0.05), (0.2, 0.2),
                                                     (0.02, 0.0), (0.0, 0.0)])
def test_from_noise_is_the_steady_state_kalman_gain(model_sigma, meas_sigma):
    o = ObserverParams.from_noise(model_sigma, meas_sigma)
    assert o.mode == 1 and len(o.gain) == 6
    q, r = model_sigma ** 2, meas_sigma ** 2
    want = 1.0 if r == 0 else _riccati_gain(q, r)
    for l in o.gain:
        assert 0.0 <= l <= 1.0
        assert math.isclose(l, want, rel_tol=1e-9, abs_tol=1e-15), (l, want)


def test_from_noise_per_channel_and_edges():
    ms = (0.01, 0.02, 0.0, 0.001, 0.05, 0.01)
    rs = (0.01, 0.0, 0.01, 0.005, 0.01, 0.1)
    o = ObserverParams.from_noise(ms, rs)
    for j in range(6):
        assert o.gain[j] == ObserverParams.from_noise(ms[j], rs[j]).gain[0]
    assert o.gain[1] == 1.0 and o.gain[2] == 0.0           # a perfect sensor; a perfect model
    assert nat.make_observer_sets([o], np.zeros(B), B)[0][0].gain[1] == 1.0
    for bad in ((-0.1, 0.1), (0.1, float("nan")), (float("inf"), 0.1)):
        with pytest.raises(ValueError):
            ObserverParams.from_noise(*bad)


# ---- the restatement ---------------------------------------------------------------------------------------------------------
L = TRACK_LENGTH
Y = np.array([1.1, 0.02, -0.3, 0.04, 7.5, -0.12])
P = np.array([1.05, 0.025, -0.28, 0.05, 7.45, -0.1])


def test_blend_is_one_rounding_per_operation():
    g = np.array([0.5, 0.3, 0.7, 0.25, 0.9, 0.1])
    x, hp, r = ob.observe_one(Y, P, 1, 1, g, L)
    assert hp == 1 and not r
    for j in range(6):
        d = np.float64(Y[j]) - np.float64(P[j])
        assert x[j] == np.float64(P[j]) + np.float64(g[j]) * d
    # numpy computes no fused multiply-add: the float64 scalar operations above round one by one
    assert x.dtype == np.float64


def test_gain_one_copies_y_and_gain_zero_takes_p():
    # p + 1 * (y - p) is not y for every pair: the copy rule does not depend on the rounding
    y, p = np.full(6, 0.1), np.full(6, 1e17)
    assert (p + 1.0 * (y - p))[0] != y[0]
    x, _, _ = ob.observe_one(y, p, 1, 1, np.ones(6), L)
    assert np.array_equal(x, y)
    pz = np.array([-0.0, 0.0, 1.0, -2.0, 3.0, -0.0])
    x, _, _ = ob.observe_one(Y, pz, 1, 1, np.zeros(6), L)
    assert np.array_equal(x, pz) and np.array_equal(np.signbit(x), np.signbit(pz))     # -0.0 stays -0.0


def test_no_prior_mode_zero_and_no_blend_read_y():
    x, hp, r = ob.observe_one(Y, P, 0, 1, np.full(6, 0.5), L)
    assert np.array_equal(x, Y) and hp == 0 and not r
    x, hp, r = ob.observe_one(Y, P, 1, 0, np.full(6, 0.5), L)
    assert np.array_equal(x, Y) and hp == 1 and not r
    x, hp, r = ob.observe_one(Y, P, 1, 1, np.full(6, 0.5), L, blend=False)       # PID or LTI step: has_pred cleared
    assert np.array_equal(x, Y) and hp == 0 and not r
    x, hp, r = ob.observe_one(Y, P, 1, 0, np.full(6, 0.5), L, blend=False)       # mode 0 rows keep it
    assert hp == 1


def test_the_lap_wrap_of_the_prior():
    # after a hand-over y's s has moved back by L, the prior's has not
    y = Y.copy(); y[4] = 0.03
    p = P.copy(); p[4] = L + 0.02
    g = np.full(6, 0.5)
    x, _, _ = ob.observe_one(y, p, 1, 1, g, L)
    ps = np.fmax(np.float64(p[4]) - np.float64(L), 0.0)
    assert x[4] == ps + 0.5 * (y[4] - ps)
    assert abs(x[4] - 0.025) < 1e-12
    p[4] = L - 1e-3                                             # a prior just short of the line wraps to 0
    x, _, _ = ob.observe_one(y, p, 1, 1, g, L)
    assert x[4] == 0.0 + 0.5 * (y[4] - 0.0)
    p[4] = y[4] + L / 2                                         # exactly half a lap ahead: no wrap
    assert ob.wrap_guess_s(p[4], y[4], L) == p[4]
    assert ob.wrap_guess_s(float("nan"), y[4], L) != ob.wrap_guess_s(float("nan"), y[4], L)   # NaN stays NaN


@pytest.mark.parametrize("j", range(6))
def test_a_non_finite_prior_resets(j):
    p = P.copy(); p[j] = (float("nan"), float("inf"), -float("inf"))[j % 3]
    g = np.full(6, 0.5)
    x, hp, r = ob.observe_one(Y, p, 1, 1, g, L)
    assert r and hp == 1 and np.array_equal(x, Y)
    g[j] = 1.0                                                  # the channel that is not finite is not read
    x, hp, r = ob.observe_one(Y, p, 1, 1, g, L)
    assert not r and x[j] == Y[j] and np.all(np.isfinite(x))
    x, hp, r = ob.observe_one(Y, p, 1, 1, np.ones(6), L)        # an all-ones row never reads the prior
    assert not r and np.array_equal(x, Y)


def test_batch_form_matches_one_by_one():
    rng = np.random.default_rng(3)
    Bn = 32
    y, p = rng.normal(size=(Bn, 6)), rng.normal(size=(Bn, 6))
    p[3, 2] = np.nan
    hp = rng.integers(0, 2, Bn)
    modes = rng.integers(0, 2, Bn)
    gains = rng.uniform(size=(Bn, 6))
    gains[::5] = 1.0
    xh, hpo, fl = ob.observe(y, p, hp, modes, gains, L)
    for b in range(Bn):
        x1, h1, r1 = ob.observe_one(y[b], p[b], hp[b], modes[b], gains[b], L)
        assert np.array_equal(xh[b], x1) and hpo[b] == h1 and fl[b] == (ob.FLAG_OBSERVER_RESET if r1 else 0)
