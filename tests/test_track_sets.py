"""CPU tier: per-controller tracks (lmpc_set_tracks).  reference_params.TrackParams and the test-side Map for any circuit
(tests/support/track_model.py) against the reference's own Map and dynModel on the three circuits of Track.py
(tests/golden/track_golden.npz, tests/golden/make_track_golden.py); and the Python-side checks and packing of
_native.make_track_sets."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import track_model
import vehicle_model as vm
from racinglmpc_b200 import _native as nat
from racinglmpc_b200.reference_params import TrackParams, VehicleParams

B = 32
HERE = os.path.dirname(os.path.abspath(__file__))
NAMES = ("l_shaped", "goggle", "oval")
MAKE = {"l_shaped": TrackParams.l_shaped, "goggle": TrackParams.goggle, "oval": TrackParams.oval}


class Draws:
    def __init__(self, z):
        self._it = iter(np.asarray(z, float).ravel())

    def standard_normal(self):
        return next(self._it)


@pytest.fixture(scope="module")
def tg():
    return np.load(os.path.join(HERE, "golden", "track_golden.npz"))


@pytest.mark.parametrize("name", NAMES)
def test_from_spec_equals_the_reference_table(tg, name):
    t = MAKE[name]()
    assert np.array_equal(t.table6, tg[name + "_table"])
    assert t.TrackLength == float(tg[name + "_length"])
    assert np.array_equal(t.seg_table, tg[name + "_table"][:, 3:6])


def test_l_track_equals_the_reference_golden_and_workloads():
    g = np.load(os.path.join(HERE, "golden", "reference_golden.npz"))
    t = TrackParams.l_shaped()
    assert np.array_equal(t.table6, g["track_table"])
    from racinglmpc_b200 import reference_params as rp, workloads
    assert t.TrackLength == rp.TRACK_LENGTH and np.array_equal(t.seg_table, workloads.track_seg_table())


def test_circuits_as_the_issue_describes_them(tg):
    """7, 11 and 6 rows; 19.23, 19.13 and 13.0 m; the L track turns left, the oval right; the oval's closing straight is empty."""
    rows = [tg[n + "_table"].shape[0] for n in NAMES]
    assert rows == [7, 11, 6]
    assert np.allclose([float(tg[n + "_length"]) for n in NAMES], [19.2296, 19.1313, 13.0], atol=1e-4)
    assert (tg["l_shaped_table"][:, 5] > 0).sum() > (tg["l_shaped_table"][:, 5] < 0).sum()
    assert (tg["oval_table"][:, 5] <= 0).all() and (tg["oval_table"][:, 5] < 0).any()
    assert 0 < tg["oval_table"][-1, 4] < 1e-15


@pytest.mark.parametrize("name", NAMES)
def test_curvature_and_global_position_equal_the_reference(tg, name):
    t = track_model.from_table(tg[name + "_table"])
    assert t.TrackLength == float(tg[name + "_length"])
    s, ey = tg[name + "_s"], tg[name + "_ey"]
    for i in range(s.shape[0]):
        if tg[name + "_curvature_ok"][i]:
            assert t.curvature(s[i]) == tg[name + "_curvature"][i], (name, i)
        else:
            with pytest.raises(Exception):
                t.curvature(s[i])
        if tg[name + "_xy_ok"][i]:
            assert np.array_equal(np.array(t.global_position(s[i], ey[i])), tg[name + "_xy"][i]), (name, i)
        else:
            with pytest.raises(Exception):
                t.global_position(s[i], ey[i])
    assert tg[name + "_curvature_ok"].sum() < s.shape[0]          # the fixture holds points where the reference raises


def test_oval_end_point_raises(tg):
    t = track_model.from_table(tg["oval_table"])
    with pytest.raises(Exception):
        t.curvature(13.0)


@pytest.mark.parametrize("name", NAMES)
def test_dyn_model_equals_the_reference_on_every_track(tg, name):
    t = track_model.from_table(tg[name + "_table"])
    for i in range(tg[name + "_x"].shape[0]):
        xn, gn = vm.dyn_model(t, tg[name + "_x"][i], tg[name + "_x_glob"][i], tg[name + "_u"][i], VehicleParams.reference(),
                              rng=Draws(tg[name + "_z"][i]))
        assert np.array_equal(xn, tg[name + "_x_next"][i]) and np.array_equal(gn, tg[name + "_x_glob_next"][i]), (name, i)


def test_library_exports_set_tracks_and_the_struct_size_matches():
    assert "lmpc_set_tracks" in nat.exported_symbols()
    L = nat.lib()                                             # asserts lmpc_sizeof_track_params() == sizeof(TrackParams)
    assert L.lmpc_sizeof_track_params() == C.sizeof(nat.TrackParams) == 8 + 8 * 48 + 8


def test_valid_sets_pack_row_by_row():
    ts = [TrackParams.l_shaped(), TrackParams.goggle(), TrackParams.oval()]
    idx = (5 * np.arange(B)) % 3
    packed, pidx = nat.make_track_sets(ts, idx, B)
    assert len(packed) == 3 and pidx.dtype == np.int32 and np.array_equal(pidx, idx)
    for k, t in enumerate(ts):
        n = t.seg_table.shape[0]
        assert packed[k].nseg == n and packed[k].TrackLength == t.TrackLength
        seg = np.ctypeslib.as_array(packed[k].seg)
        assert np.array_equal(seg[:3 * n], t.seg_table.ravel()) and not seg[3 * n:].any()


@pytest.mark.parametrize("index", [np.zeros(B - 1, int), np.zeros(B + 1, int), np.full(B, 2), np.full(B, -1), np.full(B, 0.5), None])
def test_bad_index_is_a_value_error(index):
    with pytest.raises(ValueError):
        nat.make_track_sets([TrackParams.l_shaped()] * 2, index, B)


def test_no_tracks_or_more_than_batch_is_a_value_error():
    with pytest.raises(ValueError):
        nat.make_track_sets([], np.zeros(B, int), B)
    with pytest.raises(ValueError):
        nat.make_track_sets([TrackParams.l_shaped()] * (B + 1), np.zeros(B, int), B)


class Table:
    def __init__(self, seg, L):
        self.seg_table, self.TrackLength = np.asarray(seg, float), L


def _bad_tables():
    ok = TrackParams.oval()
    seg, L = ok.seg_table.copy(), ok.TrackLength
    out = {"no rows": (np.zeros((0, 3)), 1.0), "17 rows": (np.zeros((17, 3)), 1.0)}
    for what, v in (("nan", math.nan), ("inf", math.inf)):
        s = seg.copy(); s[2, 2] = v
        out["curvature " + what] = (s, L)
        out["TrackLength " + what] = (seg, v)
    s = seg.copy(); s[1, 1] = -s[1, 1]; out["negative length"] = (s, L)
    s = seg.copy(); s[0, 0] = 1e-12; out["first start"] = (s, L)
    s = seg.copy(); s[3, 0] = np.nextafter(s[3, 0], 0); out["gap"] = (s, L)
    out["length short"] = (seg, np.nextafter(L, 0))
    out["length long"] = (seg, np.nextafter(L, 20))
    out["zero length"] = (np.zeros((1, 3)), 0.0)
    out["wrong columns"] = (np.zeros((3, 2)), 1.0)
    return out


@pytest.mark.parametrize("what", sorted(_bad_tables()))
def test_malformed_table_is_a_value_error(what):
    seg, L = _bad_tables()[what]
    with pytest.raises(ValueError):
        nat.make_track_sets([TrackParams.l_shaped(), Table(seg, L)], np.arange(B) % 2, B)


def test_oval_with_its_empty_closing_segment_is_accepted():
    packed, _ = nat.make_track_sets([TrackParams.oval()], np.zeros(B, int), B)
    assert packed[0].nseg == 6 and packed[0].TrackLength == 13.0
