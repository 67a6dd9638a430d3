"""CPU tier: per-controller noise models and noise streams (lmpc_rollout_set_noise, lmpc_rollout_set_noise_streams).
reference_params.NoiseParams against the reference's literal constants, the test-side dynModel with a noise set
(tests/support/noise_model.py) against the golden data and against the formula computed by hand, and the Python-side checks
and packing of _native.make_noise_sets / make_noise_streams."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import noise_model as nm
from racinglmpc_b200 import _native as nat
from racinglmpc_b200.reference_params import NoiseParams, VehicleParams

B = 32
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vehicle_golden.npz")
FIELDS = ("sim_sigma", "sim_clip", "sim_gain", "pid_sigma", "pid_clip")


class Draws:
    """An rng whose standard_normal() hands out fixed draws in order (the reference consumes np.random.randn())."""

    def __init__(self, z):
        self._it = iter(np.asarray(z, float).ravel())

    def standard_normal(self):
        return next(self._it)


def _bits(n):
    return [np.asarray(getattr(n, f), float).tobytes() for f in FIELDS]


def test_reference_equals_the_literal_constants():
    r = NoiseParams.reference()
    assert r.sim_sigma == (0.01, 0.01, 0.005) and r.sim_clip == (0.05, 0.05, 0.05)     # SysModel.py:139-141
    assert r.sim_gain == 0.01                                                          # SysModel.py:143-145
    assert r.pid_sigma == (0.25, 0.10) and r.pid_clip == (0.9, 0.2)                    # Utilities.py:42-68


def test_scaled_by_one_is_the_reference_bit_for_bit_and_zero_is_noise_free():
    assert _bits(NoiseParams.scaled(1, 1)) == _bits(NoiseParams.reference())
    assert _bits(NoiseParams.scaled(1.0, 1.0)) == _bits(NoiseParams.reference())
    z = NoiseParams.scaled(0, 0)
    assert z.sim_sigma == z.sim_clip == (0.0, 0.0, 0.0) and z.pid_sigma == z.pid_clip == (0.0, 0.0)
    assert z.sim_gain == 0.01
    s = NoiseParams.scaled(10, 0.5)
    r = NoiseParams.reference()
    assert s.sim_sigma == tuple(v * 10 for v in r.sim_sigma) and s.sim_clip == tuple(v * 10 for v in r.sim_clip)
    assert s.pid_sigma == tuple(v * 0.5 for v in r.pid_sigma) and s.pid_clip == tuple(v * 0.5 for v in r.pid_clip)


def test_dyn_model_with_the_reference_noise_equals_the_golden_data(track):
    vg = np.load(GOLD)
    noise = NoiseParams.reference()
    for k, row in enumerate(vg["vehicles"]):
        veh = VehicleParams(*row)
        for i in range(vg["x"].shape[0]):
            xn, gn = nm.dyn_model(track, vg["x"][i], vg["x_glob"][i], vg["u"][i], veh, noise, rng=Draws(vg["z"][k, i]))
            assert np.array_equal(xn, vg["x_next"][k, i]) and np.array_equal(gn, vg["x_glob_next"][k, i]), (k, i)


def test_dyn_model_with_a_scaled_set_follows_the_formula(track):
    """The noise enters the curvilinear copy only, as gain * clip(z * sigma, +-clip), and no clip is left inactive: the draws
    put one channel past its clip and leave another inside it."""
    vg = np.load(GOLD)
    veh = VehicleParams.reference()
    noise = NoiseParams((0.3, 0.02, 0.7), (0.1, 0.5, 0.2), 0.04, (0.25, 0.10), (0.9, 0.2))
    z = np.array([1.5, -0.8, -2.0])
    for i in range(4):
        quiet = nm.dyn_model(track, vg["x"][i], vg["x_glob"][i], vg["u"][i], veh, NoiseParams.scaled(0, 0), rng=Draws(np.zeros(3)))
        xn, gn = nm.dyn_model(track, vg["x"][i], vg["x_glob"][i], vg["u"][i], veh, noise, rng=Draws(z))
        assert np.array_equal(gn, quiet[1]) and np.array_equal(xn[3:], quiet[0][3:])
        n = [max(-noise.sim_clip[j], min(z[j] * noise.sim_sigma[j], noise.sim_clip[j])) for j in range(3)]
        assert n[0] == noise.sim_clip[0] and n[1] == z[1] * noise.sim_sigma[1] and n[2] == -noise.sim_clip[2]
        assert all(xn[j] == quiet[0][j] + noise.sim_gain * n[j] for j in range(3)), i


def test_test_side_pid_with_the_reference_noise_equals_the_oracle():
    from oracle import vehicle as ov
    rng = np.random.default_rng(3)
    for _ in range(16):
        x, z = rng.standard_normal(6), rng.standard_normal(2) * 3
        a, b = ov.PIDFollower(0.8, rng=Draws(z)), nm.PIDFollower(0.8, NoiseParams.reference(), rng=Draws(z))
        a.solve(x)
        b.solve(x)
        assert np.array_equal(a.uPred, b.uPred)


def test_library_exports_the_noise_calls_and_the_struct_size_matches():
    syms = nat.exported_symbols()
    assert {"lmpc_rollout_set_noise", "lmpc_rollout_set_noise_streams", "lmpc_sizeof_noise_params"} <= set(syms)
    L = nat.lib()                                             # asserts lmpc_sizeof_noise_params() == sizeof(NoiseParams)
    assert L.lmpc_sizeof_noise_params() == C.sizeof(nat.NoiseParams) == 88


def test_valid_sets_pack_field_by_field():
    ns = [NoiseParams.reference(), NoiseParams.scaled(0, 0), NoiseParams.scaled(10, 0.5)]
    idx = (5 * np.arange(B)) % 3
    packed, pidx = nat.make_noise_sets(ns, idx, B)
    assert len(packed) == 3 and pidx.dtype == np.int32 and np.array_equal(pidx, idx)
    for k, n in enumerate(ns):
        for f in FIELDS:
            got = getattr(packed[k], f)
            assert list(got) == list(getattr(n, f)) if f != "sim_gain" else got == n.sim_gain, (k, f)


@pytest.mark.parametrize("index", [np.zeros(B - 1, int), np.zeros(B + 1, int), np.full(B, 2), np.full(B, -1), np.full(B, 0.5), None])
def test_bad_index_is_a_value_error(index):
    with pytest.raises(ValueError):
        nat.make_noise_sets([NoiseParams.reference()] * 2, index, B)


def test_no_sets_or_more_than_batch_is_a_value_error():
    with pytest.raises(ValueError):
        nat.make_noise_sets([], np.zeros(B, int), B)
    with pytest.raises(ValueError):
        nat.make_noise_sets([NoiseParams.reference()] * (B + 1), np.zeros(B, int), B)


def _with(field, j, v):
    r = NoiseParams.reference()
    vals = {f: getattr(r, f) for f in FIELDS}
    if j is None:
        vals[field] = v
    else:
        t = list(vals[field])
        t[j] = v
        vals[field] = tuple(t)
    return NoiseParams(**vals)


BAD = [(f, j, v) for f, n in (("sim_sigma", 3), ("sim_clip", 3), ("pid_sigma", 2), ("pid_clip", 2)) for j in range(n)
       for v in (math.nan, math.inf, -1e-3)] + [("sim_gain", None, v) for v in (math.nan, math.inf, -0.01)]


@pytest.mark.parametrize("field,j,v", BAD)
def test_bad_value_is_a_value_error(field, j, v):
    with pytest.raises(ValueError):
        nat.make_noise_sets([NoiseParams.reference(), _with(field, j, v)], np.arange(B) % 2, B)


@pytest.mark.parametrize("field,value", [("sim_sigma", (0.01, 0.01)), ("sim_clip", (0.05,) * 4), ("pid_sigma", (0.25,)),
                                         ("pid_clip", (0.9, 0.2, 0.1)), ("sim_gain", (0.01, 0.01))])
def test_wrong_length_is_a_value_error(field, value):
    r = NoiseParams.reference()
    bad = NoiseParams(**dict({f: getattr(r, f) for f in FIELDS}, **{field: value}))
    with pytest.raises(ValueError):
        nat.make_noise_sets([bad], np.zeros(B, int), B)


def test_zero_sigma_and_clip_are_allowed():
    packed, _ = nat.make_noise_sets([NoiseParams((0, 0, 0), (0, 0, 0), 0, (0, 0), (0, 0))], np.zeros(B, int), B)
    assert packed[0].sim_gain == 0.0 and list(packed[0].pid_clip) == [0.0, 0.0]


def test_streams_pack_and_none_means_stream_b():
    assert nat.make_noise_streams(None, B) is None
    s = nat.make_noise_streams(np.arange(B) // 2, B)
    assert s.dtype == np.int32 and np.array_equal(s, np.arange(B) // 2)
    assert np.array_equal(nat.make_noise_streams([0] * B, B), np.zeros(B))        # repeats are the point
    assert nat.make_noise_streams(np.full(B, 2 ** 31 - 1), B).max() == 2 ** 31 - 1


@pytest.mark.parametrize("streams", [np.zeros(B - 1, int), np.zeros(B + 1, int), np.full(B, -1), np.full(B, 0.5),
                                     np.full(B, math.nan), np.full(B, 2 ** 31), np.zeros((0,), int)])
def test_bad_streams_are_a_value_error(streams):
    with pytest.raises(ValueError):
        nat.make_noise_streams(streams, B)
