"""CPU tier: per-controller vehicles (lmpc_rollout_set_vehicles).  The test-side dynModel for any vehicle (tests/support/vehicle_model.py)
against the reference's own dynModel with its vehicle constants replaced (tests/golden/vehicle_golden.npz,
tests/golden/make_vehicle_golden.py) and, on the reference car, against the oracle's; and the Python-side checks and packing of
_native.make_vehicle_sets and reference_params.VehicleParams."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import vehicle_model as vm
from oracle import vehicle as ov
from racinglmpc_b200 import _native as nat
from racinglmpc_b200.reference_params import VehicleParams

B = 32
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vehicle_golden.npz")


class Draws:
    """An rng whose standard_normal() hands out fixed draws in order (the reference consumes np.random.randn())."""

    def __init__(self, z):
        self._it = iter(np.asarray(z, float).ravel())

    def standard_normal(self):
        return next(self._it)


@pytest.fixture(scope="module")
def vg():
    return np.load(GOLD)


def test_dyn_model_equals_the_reference_on_every_vehicle(vg, track):
    assert tuple(vg["fields"]) == vm.VEHICLE_FIELDS == tuple(f for f, _ in nat.VehicleParams._fields_)
    for k, row in enumerate(vg["vehicles"]):
        veh = VehicleParams(*row)
        for i in range(vg["x"].shape[0]):
            xn, gn = vm.dyn_model(track, vg["x"][i], vg["x_glob"][i], vg["u"][i], veh, rng=Draws(vg["z"][k, i]))
            assert np.max(np.abs(xn - vg["x_next"][k, i])) == 0.0, (k, i)
            assert np.max(np.abs(gn - vg["x_glob_next"][k, i])) == 0.0, (k, i)


def test_golden_vehicles_differ_and_cover_the_track(vg, track):
    """The fixture exercises what it should: straights and curves, lateral offset, side slip and yaw rate, and vehicles whose
    next states differ from the reference car's."""
    curv = np.array([track.curvature(s) for s in vg["x"][:, 4]])
    assert (curv == 0).any() and (curv != 0).any()
    assert np.all(vg["x"][:, 5] != 0) and np.all(vg["x"][:, 1] != 0) and np.all(vg["x"][:, 2] != 0)
    for k in range(1, vg["vehicles"].shape[0]):
        assert np.abs(vg["x_next"][k] - vg["x_next"][0]).max() > 1e-4, k


def test_reference_vehicle_equals_the_oracle(vg, track):
    ref = VehicleParams.reference()
    assert np.array_equal(vg["vehicles"][0], [getattr(ref, f) for f in vm.VEHICLE_FIELDS])
    for i in range(vg["x"].shape[0]):
        a = ov.dyn_model(track, vg["x"][i], vg["x_glob"][i], vg["u"][i], rng=Draws(vg["z"][0, i]))
        b = vm.dyn_model(track, vg["x"][i], vg["x_glob"][i], vg["u"][i], ref, rng=Draws(vg["z"][0, i]))
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), i


def test_reference_vehicle_and_from_friction():
    ref = VehicleParams.reference()
    assert (ref.m, ref.lf, ref.lr, ref.Iz, ref.Cf, ref.Bf, ref.Cr, ref.Br) == (1.98, 0.125, 0.125, 0.024, 1.25, 1.0, 1.25, 1.0)
    D = 0.8 * 1.98 * 9.81 / 2.0                               # SysModel.py:65,68, bit for bit
    assert VehicleParams.from_friction(0.8).Df == D and VehicleParams.from_friction(0.8).Dr == D
    assert ref.Df == ov._DF and ref.Dr == ov._DR
    v = VehicleParams.from_friction(0.5, m=2.6, Iz=0.032)
    assert v.Df == v.Dr == 0.5 * 2.6 * 9.81 / 2.0 and v.Iz == 0.032


def test_library_exports_set_vehicles_and_the_struct_size_matches():
    assert "lmpc_rollout_set_vehicles" in nat.exported_symbols()
    L = nat.lib()                                             # asserts lmpc_sizeof_vehicle_params() == sizeof(VehicleParams)
    assert L.lmpc_sizeof_vehicle_params() == C.sizeof(nat.VehicleParams) == 80


def test_valid_sets_pack_field_by_field():
    vs = [VehicleParams.reference(), VehicleParams.from_friction(0.5), VehicleParams.from_friction(1.1, m=2.6, Iz=0.032)]
    idx = (5 * np.arange(B)) % 3
    packed, pidx = nat.make_vehicle_sets(vs, idx, B)
    assert len(packed) == 3 and pidx.dtype == np.int32 and np.array_equal(pidx, idx)
    for k, v in enumerate(vs):
        assert all(getattr(packed[k], f) == getattr(v, f) for f in vm.VEHICLE_FIELDS), k


@pytest.mark.parametrize("index", [np.zeros(B - 1, int), np.zeros(B + 1, int), np.full(B, 2), np.full(B, -1), np.full(B, 0.5), None])
def test_bad_index_is_a_value_error(index):
    with pytest.raises(ValueError):
        nat.make_vehicle_sets([VehicleParams.reference()] * 2, index, B)


def test_no_vehicles_or_more_than_batch_is_a_value_error():
    with pytest.raises(ValueError):
        nat.make_vehicle_sets([], np.zeros(B, int), B)
    with pytest.raises(ValueError):
        nat.make_vehicle_sets([VehicleParams.reference()] * (B + 1), np.zeros(B, int), B)


def _with(**kw):
    v = VehicleParams.reference()
    return VehicleParams(**{f: kw.get(f, getattr(v, f)) for f in vm.VEHICLE_FIELDS})


@pytest.mark.parametrize("bad", [dict(m=0.0), dict(m=-1.98), dict(Iz=0.0), dict(lf=0.0), dict(lr=-0.1)] +
                         [{f: v} for f in vm.VEHICLE_FIELDS for v in (math.nan, math.inf)] + [dict(Df=-math.inf)])
def test_bad_vehicle_is_a_value_error(bad):
    with pytest.raises(ValueError):
        nat.make_vehicle_sets([VehicleParams.reference(), _with(**bad)], np.arange(B) % 2, B)


def test_non_positive_friction_and_shape_are_allowed():
    """Only m, Iz, lf and lr must be positive (they divide or set the geometry); D, C, B are the user's to choose."""
    packed, _ = nat.make_vehicle_sets([_with(Df=0.0, Cr=-1.0, Br=0.0)], np.zeros(B, int), B)
    assert packed[0].Df == 0.0 and packed[0].Cr == -1.0
