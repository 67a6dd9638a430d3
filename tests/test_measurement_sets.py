"""CPU tier: per-controller measurement noise (lmpc_rollout_set_measurement_noise).
reference_params.MeasurementParams (zero, scaled) and the Python-side checks and packing of _native.make_measurement_sets, which
refuses whatever the library refuses."""
import ctypes as C
import math

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat
from racinglmpc_b200.reference_params import MeasurementParams

B = 32
FIELDS = ("sigma", "clip")
BASE = MeasurementParams((0.01, 0.01, 0.01, 0.005, 0.01, 0.01), (0.05, 0.05, 0.05, 0.025, 0.05, 0.05))
ODD = MeasurementParams((0.3, 0.0, 1e-3, 0.2, 7.0, 0.1), (0.1, 0.5, 0.0, 0.02, 1.0, 0.3))


def _bits(m):
    return [np.asarray(getattr(m, f), float).tobytes() for f in FIELDS]


def test_library_exports_the_call_and_the_struct_size_matches():
    syms = nat.exported_symbols()
    assert {"lmpc_rollout_set_measurement_noise", "lmpc_sizeof_measurement_params"} <= set(syms)
    L = nat.lib()                                     # asserts lmpc_sizeof_measurement_params() == sizeof(MeasurementParams)
    assert L.lmpc_sizeof_measurement_params() == C.sizeof(nat.MeasurementParams) == 96


def test_zero_and_scaled():
    z = MeasurementParams.zero()
    assert z.sigma == z.clip == (0.0,) * 6
    assert _bits(MeasurementParams.scaled(1, BASE)) == _bits(BASE)
    assert _bits(MeasurementParams.scaled(1.0, ODD)) == _bits(ODD)
    assert _bits(MeasurementParams.scaled(0, BASE)) == _bits(z)
    s = MeasurementParams.scaled(10, BASE)
    assert s.sigma == tuple(v * 10 for v in BASE.sigma) and s.clip == tuple(v * 10 for v in BASE.clip)


def test_valid_sets_pack_field_by_field():
    ms = [BASE, MeasurementParams.zero(), ODD, MeasurementParams.scaled(100, BASE)]
    idx = (7 * np.arange(B)) % 4
    packed, pidx = nat.make_measurement_sets(ms, idx, B)
    assert len(packed) == 4 and pidx.dtype == np.int32 and np.array_equal(pidx, idx)
    for k, m in enumerate(ms):
        for f in FIELDS:
            assert np.asarray(getattr(packed[k], f)).tobytes() == np.asarray(getattr(m, f), float).tobytes(), (k, f)
    # the row layout the library reads: sigma[6] then clip[6]
    raw = np.frombuffer(bytes(packed[2]), dtype=np.float64)
    assert np.array_equal(raw, np.concatenate([ODD.sigma, ODD.clip]))


@pytest.mark.parametrize("index", [np.zeros(B - 1, int), np.zeros(B + 1, int), np.full(B, 2), np.full(B, -1), np.full(B, 0.5), None])
def test_bad_index_is_a_value_error(index):
    with pytest.raises(ValueError):
        nat.make_measurement_sets([BASE] * 2, index, B)


def test_no_sets_or_more_than_batch_is_a_value_error():
    with pytest.raises(ValueError):
        nat.make_measurement_sets([], np.zeros(B, int), B)
    with pytest.raises(ValueError):
        nat.make_measurement_sets([BASE] * (B + 1), np.zeros(B, int), B)


def _with(field, j, v):
    vals = {f: list(getattr(BASE, f)) for f in FIELDS}
    vals[field][j] = v
    return MeasurementParams(**{f: tuple(t) for f, t in vals.items()})


BAD = [(f, j, v) for f in FIELDS for j in range(6) for v in (math.nan, math.inf, -1e-3)]


@pytest.mark.parametrize("field,j,v", BAD)
def test_bad_value_is_a_value_error(field, j, v):
    with pytest.raises(ValueError):
        nat.make_measurement_sets([BASE, _with(field, j, v)], np.arange(B) % 2, B)


@pytest.mark.parametrize("field,value", [("sigma", (0.01,) * 5), ("sigma", (0.01,) * 7), ("clip", (0.05,) * 3), ("clip", 0.05)])
def test_wrong_length_is_a_value_error(field, value):
    bad = MeasurementParams(**dict({f: getattr(BASE, f) for f in FIELDS}, **{field: value}))
    with pytest.raises(ValueError):
        nat.make_measurement_sets([bad], np.zeros(B, int), B)


def test_zero_values_are_allowed():
    packed, _ = nat.make_measurement_sets([MeasurementParams.zero()], np.zeros(B, int), B)
    assert list(packed[0].sigma) == [0.0] * 6 and list(packed[0].clip) == [0.0] * 6
    packed, _ = nat.make_measurement_sets([MeasurementParams((0.0, 1.0, 0.0, 2.0, 0.0, 3.0), (1.0, 0.0, 0.0, 1.0, 1.0, 0.0))],
                                          np.zeros(B, int), B)
    assert list(packed[0].clip) == [1.0, 0.0, 0.0, 1.0, 1.0, 0.0]
