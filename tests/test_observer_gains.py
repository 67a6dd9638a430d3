"""CPU tier: observer gains (lmpc_rollout_set_observer_gains) -- the ABI size and packing of ObserverGainParams, every refusal of
make_observer_gain_sets before any native call, ObserverGains' constructors and its clipped-noise variance, and the restatement
the GPU tests compare against (tests/support/observer_gain.py): the tangent propagation of Phi_car against central differences of
the exact prior, the doubling against scipy's DARE solver, and the rounding order of the blend."""
import ctypes as C
import math

import mpmath as mp
import numpy as np
import pytest
from scipy import integrate, linalg, stats

from racinglmpc_b200 import _native as nat
from racinglmpc_b200 import reference_params as rp
from racinglmpc_b200.reference_params import ObserverGains, VehicleParams
import observer_gain as og
import observer_prior as op
import plant_exact as pe

B = 8
T0 = rp.TrackParams.l_shaped()
L = float(T0.TrackLength)
SEG = np.asarray(T0.seg_table, float)
TRACK = pe.ExactTrack(T0.seg_table, L)
CAR = VehicleParams.reference()


def test_struct_size_and_packing_match_the_library():
    assert C.sizeof(nat.ObserverGainParams) == 8 + 96
    assert nat.ObserverGainParams.mode.offset == 0 and nat.ObserverGainParams.pad.offset == 4
    assert nat.ObserverGainParams.q.offset == 8 and nat.ObserverGainParams.r.offset == 56
    assert nat.lib().lmpc_sizeof_observer_gain_params() == C.sizeof(nat.ObserverGainParams)
    assert nat.FLAG_OBSERVER_GAIN == 4096
    used = [1, 2, 4, 32, 64, 128, 256, 1024, nat.FLAG_OBSERVER_RESET, nat.REPORT_LANE_UNSAFE]
    assert all(nat.FLAG_OBSERVER_GAIN & u == 0 for u in used)


def test_packing():
    rows = [ObserverGains.fixed(), ObserverGains.kalman(1e-4, 1e-3), ObserverGains.kalman(range(1, 7), [2.0] * 6)]
    idx = np.arange(B) % 3
    tab, ix = nat.make_observer_gain_sets(rows, idx, B)
    assert len(tab) == 3 and ix.dtype == np.int32 and np.array_equal(ix, idx)
    assert [t.mode for t in tab] == [0, 1, 1] and all(t.pad == 0 for t in tab)
    assert list(tab[0].q) == [0.0] * 6 and list(tab[0].r) == [0.0] * 6        # not read under mode 0: not packed
    assert list(tab[1].q) == [1e-4] * 6 and list(tab[1].r) == [1e-3] * 6
    assert list(tab[2].q) == [1.0, 2.0, 3.0, 4.0, 5.0, 6.0] and list(tab[2].r) == [2.0] * 6


def test_mode_zero_rows_are_not_checked():
    tab, _ = nat.make_observer_gain_sets([ObserverGains(0, (float("nan"),) * 6, (-1.0,) * 6)], np.zeros(B), B)
    assert tab[0].mode == 0


NAN, INF = float("nan"), float("inf")


@pytest.mark.parametrize("row", [
    ObserverGains(2), ObserverGains(-1), ObserverGains(True), ObserverGains(1.0), ObserverGains(None),
    ObserverGains(1, (0.0,) + (1.0,) * 5), ObserverGains(1, (1.0,) * 5 + (-1e-300,)), ObserverGains(1, (NAN,) * 6),
    ObserverGains(1, (1.0,) * 6, (INF,) + (1.0,) * 5), ObserverGains(1, (1.0,) * 6, (1.0,) * 5 + (0.0,)),
    ObserverGains(1, (1.0,) * 6, (-2.0,) * 6), ObserverGains(1, (1.0,) * 5), ObserverGains(1, (1.0,) * 6, (1.0,) * 7)])
def test_bad_rows_are_refused(row):
    with pytest.raises(ValueError):
        nat.make_observer_gain_sets([ObserverGains.fixed(), row], np.arange(B) % 2, B)


@pytest.mark.parametrize("rows, idx", [
    ([ObserverGains.fixed()], np.ones(B)), ([ObserverGains.fixed()], -np.ones(B)), ([ObserverGains.fixed()], np.zeros(B - 1)),
    ([ObserverGains.fixed()], np.full(B, 0.5)), ([], np.zeros(B)), ([ObserverGains.fixed()] * (B + 1), np.zeros(B)),
    ([ObserverGains.fixed()], None)])
def test_bad_indices_are_refused(rows, idx):
    with pytest.raises(ValueError):
        nat.make_observer_gain_sets(rows, idx, B)


def test_constructors():
    assert ObserverGains.fixed() == ObserverGains(0)
    k = ObserverGains.kalman(2.0, (1, 2, 3, 4, 5, 6))
    assert k.mode == 1 and k.q == (2.0,) * 6 and k.r == (1.0, 2.0, 3.0, 4.0, 5.0, 6.0)


def _quad_variance(sigma, clip):
    f = lambda z: np.clip(sigma * z, -clip, clip) ** 2 * stats.norm.pdf(z)
    a = clip / sigma
    inner = integrate.quad(f, -a, a, epsabs=0, epsrel=1e-13, limit=200)[0]
    return inner + 2 * clip * clip * stats.norm.sf(a)


@pytest.mark.parametrize("sigma, clip", [(0.01, 0.05), (0.05, 0.05), (1.0, 0.3), (0.02, 1.0), (3e-4, 2e-4), (1.0, 8.0)])
def test_clipped_variance_against_quadrature(sigma, clip):
    got = rp.clipped_normal_variance(sigma, clip)
    assert abs(got - _quad_variance(sigma, clip)) <= 1e-12 * sigma * sigma
    assert got <= sigma * sigma and got <= clip * clip


def test_clipped_variance_edges():
    assert rp.clipped_normal_variance(0.0, 1.0) == 0.0 and rp.clipped_normal_variance(1.0, 0.0) == 0.0
    assert rp.clipped_normal_variance(0.5, INF) == 0.25


def test_from_noise():
    noise = rp.NoiseParams.reference()
    meas = rp.MeasurementParams((0.01, 0.01, 0.005, 0.002, 0.01, 0.005), (0.05, 0.05, 0.05, 0.01, 0.05, 0.02))
    ms = (1e-3, 2e-3, 3e-3, 4e-4, 5e-4, 6e-4)
    g = ObserverGains.from_noise(noise, meas, ms)
    assert g.mode == 1
    for j in range(3):
        want = noise.sim_gain ** 2 * rp.clipped_normal_variance(noise.sim_sigma[j], noise.sim_clip[j]) + ms[j] ** 2
        assert g.q[j] == want
    assert g.q[3:] == tuple(m * m for m in ms[3:])
    assert g.r == tuple(rp.clipped_normal_variance(s, c) for s, c in zip(meas.sigma, meas.clip))
    with pytest.raises(ValueError):                                     # no model error on epsi: q_3 = 0
        ObserverGains.from_noise(noise, meas, (1e-3, 1e-3, 1e-3, 0.0, 1e-3, 1e-3))
    with pytest.raises(ValueError):                                     # a noise-free sensor channel: r = 0
        ObserverGains.from_noise(noise, rp.MeasurementParams.zero(), 1e-3)
    with pytest.raises(ValueError):
        ObserverGains.from_noise(noise, meas, -1.0)


# ---- the tangent propagation ------------------------------------------------------------------------------------------------
def _exact(x, u, surf):
    return np.array(pe.to_f64(op.prior_exact(CAR, TRACK, x, u, surface=surf)["x"]))


def _central(x, u, surf=None, eps=1e-6):
    J = np.empty((6, 6))
    for j in range(6):
        hj = eps * max(1.0, abs(x[j]))
        xp, xm = np.array(x, float), np.array(x, float)
        xp[j] += hj
        xm[j] -= hj
        J[:, j] = (_exact(xp, u, surf) - _exact(xm, u, surf)) / (xp[j] - xm[j])
    return J


SURF = [(0.0, 2.0, 0.6, 0.5), (3.5, 5.0, 1.1, 0.9), (6.0, L, 0.4, 0.4)]
# (x, u, zones): a straight, a curve, a friction zone (inside, away from its bounds), and a period crossing a segment join
CASES = {
    "straight": ((0.8, 0.01, 0.02, 0.05, 0.3, 0.1), (0.1, 0.5), None),
    "curve": ((1.2, -0.03, 0.4, -0.1, 3.9, -0.2), (-0.25, -1.0), None),
    "zone": ((1.0, 0.02, 0.1, 0.02, 4.0, 0.05), (0.05, 0.3), SURF),
    "join": ((1.5, 0.05, 0.3, 0.02, None, 0.1), (0.15, 0.3), None),
}


def _join_state():
    """A state whose period crosses the first segment join, placed so that the join lies as far as possible from the s of every
    sub-step: moving s then does not move the sub-step at which the curvature changes, and the map is smooth there."""
    s_join = float(SEG[1, 0])
    x, u, _ = CASES["join"]
    best, best_x = -1.0, None
    for off in np.linspace(0.03, 0.12, 91):
        xs = list(x)
        xs[4] = s_join - off
        tr = []
        og.tangent_period(CAR, SEG, L, xs, u, s_trace=tr)
        tr = np.array(tr)
        if not (tr[0] < s_join < tr[-1]):
            continue
        margin = np.min(np.abs(tr - s_join))
        if margin > best:
            best, best_x = margin, tuple(xs)
    assert best > 3e-4
    return best_x


@pytest.mark.parametrize("case", list(CASES))
def test_tangent_against_central_differences(case):
    x, u, zones = CASES[case]
    if case == "join":
        x = _join_state()
    surf = pe.ExactSurface(zones) if zones else None
    p, A, ok = og.tangent_period(CAR, SEG, L, x, u, zones=zones)
    assert ok
    assert np.max(np.abs(p - _exact(x, u, surf))) <= 1e-12 * max(1.0, np.max(np.abs(p)))
    J = _central(x, u, surf)
    assert np.max(np.abs(A - J)) <= 1e-6 * np.max(np.abs(J)), (A, J)
    assert abs(A[4, 4] - 1.0) < 1e-15 and np.all(A[:3, 4] == 0)         # s enters only through the constant curvature


def test_tangent_sees_the_zone_forces():
    x, u, _ = CASES["zone"]
    _, A0, _ = og.tangent_period(CAR, SEG, L, x, u)
    _, A1, _ = og.tangent_period(CAR, SEG, L, x, u, zones=SURF)
    assert np.max(np.abs(A0[:3] - A1[:3])) > 1e-4


# ---- the DARE -----------------------------------------------------------------------------------------------------------
QR = [((1e-4,) * 6, (1e-3,) * 6), ((1e-5, 1e-5, 1e-5, 1e-8, 1e-8, 1e-8), (1e-4, 1e-4, 2.5e-5, 1e-6, 1e-4, 2.5e-5)),
      ((1.0,) * 6, (1e-8,) * 6), ((1e-10,) * 6, (1.0,) * 6), ((3.0, 1e-3, 0.2, 1e-6, 5.0, 1e-2), (0.5, 2.0, 1e-3, 1e-1, 1e-6, 4.0))]


@pytest.mark.parametrize("case", ["straight", "curve", "zone"])
@pytest.mark.parametrize("k", range(len(QR)))
def test_sda_against_scipy(case, k):
    x, u, zones = CASES[case]
    _, A, _ = og.tangent_period(CAR, SEG, L, x, u, zones=zones)
    q, r = QR[k]
    P, conv, it = og.sda(A, q, r)
    assert conv and it < og.DARE_ITERS
    ref = linalg.solve_discrete_are(A.T, np.eye(6), np.diag(q), np.diag(r))
    assert og.dare_residual(A, P, q, r) <= 1e-12
    if k == 3:
        # q / r = 1e-10: the closed loop's eigenvalues lie within ~1e-5 of 1 and scipy's Schur solution is the less accurate
        # one (its residual is the larger); there the doubling is held to scipy's residual instead of to its P
        assert og.dare_residual(A, P, q, r) <= og.dare_residual(A, ref, q, r)
        assert np.max(np.abs(P - ref)) <= 1e-7 * np.max(np.abs(ref))
        return
    assert np.max(np.abs(P - ref)) <= 1e-10 * np.max(np.abs(ref))
    K = og.kalman_gain(P, r)
    assert np.allclose(K, ref @ np.linalg.inv(ref + np.diag(r)), rtol=0, atol=1e-10)


def test_gain_limits():
    _, A, _ = og.tangent_period(CAR, SEG, L, *CASES["curve"][:2])
    P, _, _ = og.sda(A, (1.0,) * 6, (1e-12,) * 6)
    assert np.max(np.abs(og.kalman_gain(P, (1e-12,) * 6) - np.eye(6))) < 1e-9       # r << q: read y
    P, _, _ = og.sda(A, (1e-12,) * 6, (1.0,) * 6)
    assert np.max(np.abs(og.kalman_gain(P, (1.0,) * 6))) < 1e-4                     # q << r: trust the model


# ---- the blend ----------------------------------------------------------------------------------------------------------
def test_blend_rounding_order():
    rng = np.random.default_rng(3)
    K = rng.uniform(-1, 1, (6, 6))
    y = rng.normal(size=6)
    p = y + 1e-3 * rng.normal(size=6)
    got = og.blend(y, p, K, L)
    for i in range(6):
        c = 0.0
        terms = [math.fsum([K[i, j] * (y[j] - p[j])]) for j in range(6)]      # each product rounded once
        c = terms[0]
        for t in terms[1:]:
            c = c + t
        assert got[i] == p[i] + c
    # K = I reads y up to the rounding of p + (y - p); K = 0 takes p
    assert np.array_equal(og.blend(y, p, np.zeros((6, 6)), L), p)
    assert np.max(np.abs(og.blend(y, p, np.eye(6), L) - y)) <= 4e-16 * np.max(np.abs(y))


def test_blend_wraps_the_prior_first():
    y = np.array([1.0, 0.01, 0.02, 0.03, 0.04, 0.05])
    p = np.array([1.01, 0.0, 0.01, 0.02, L + 0.03, 0.06])
    pw = p.copy()
    pw[4] = max(p[4] - L, 0.0)
    K = np.full((6, 6), 0.1)
    assert og.blend(y, p, K, L).tobytes() == og.blend(y, pw, K, L).tobytes()
