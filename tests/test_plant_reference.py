"""CPU tier: the exact plant reference (tests/support/plant_exact.py) before any GPU test relies on it.

Rounded to fp64 it meets the real reference's outputs (tests/golden/vehicle_golden.npz, track_golden.npz, reference_golden.npz)
within the bounds the GPU tests use; the fp64 NumPy restatements sit well inside those bounds on the case lists of the GPU tests
(calibration); and every bound rejects known-wrong implementations by at least 100 times (mutations)."""
import os

import numpy as np
import pytest

import plant_exact as pe
import plant_cases as pc
import vehicle_model as vm
import noise_model as nm
from racinglmpc_b200.reference_params import NoiseParams, VehicleParams

HERE = os.path.dirname(os.path.abspath(__file__))


class Draws:
    def __init__(self, z):
        self._it = iter(np.asarray(z, float).ravel())

    def standard_normal(self):
        return next(self._it)


@pytest.fixture(scope="module")
def vg():
    return np.load(os.path.join(HERE, "golden", "vehicle_golden.npz"))


@pytest.fixture(scope="module")
def tg():
    return np.load(os.path.join(HERE, "golden", "track_golden.npz"))


@pytest.fixture(scope="module")
def cases():
    return pc.sim_cases()


def test_exact_dyn_model_meets_the_vehicle_golden(vg, track):
    et = pe.ExactTrack(track.seg_table(), track.TrackLength)
    worst = 0.0
    for k, row in enumerate(vg["vehicles"]):
        veh = VehicleParams(*row)
        for i in range(vg["x"].shape[0]):
            r = pe.dyn_model(veh, et, vg["x"][i], vg["x_glob"][i], vg["u"][i], z=vg["z"][k, i])
            worst = max(worst, pe.sim_error(vg["x_next"][k, i], r["x"]), pe.sim_error(vg["x_glob_next"][k, i], r["x_glob"]))
    assert worst <= pe.SIM_BOUND / 8, worst


@pytest.mark.parametrize("name", pc.CIRCUITS)
def test_exact_dyn_model_meets_the_track_golden(tg, name):
    et = pe.ExactTrack(tg[name + "_table"][:, 3:6], float(tg[name + "_length"]))
    veh = VehicleParams.reference()
    for i in range(tg[name + "_x"].shape[0]):
        r = pe.dyn_model(veh, et, tg[name + "_x"][i], tg[name + "_x_glob"][i], tg[name + "_u"][i], z=tg[name + "_z"][i])
        assert pe.sim_error(tg[name + "_x_next"][i], r["x"]) <= pe.SIM_BOUND / 8, (name, i)
        assert pe.sim_error(tg[name + "_x_glob_next"][i], r["x_glob"]) <= pe.SIM_BOUND / 8, (name, i)


def test_exact_lookup_raises_where_the_reference_raises(tg):
    for name in pc.CIRCUITS:
        et = pe.ExactTrack(tg[name + "_table"][:, 3:6], float(tg[name + "_length"]))
        L = float(tg[name + "_length"])
        for s in (-1e-3, L, float("nan"), 65 * L):
            with pytest.raises(pe.LookupFailed):
                et.lookup(pe.mp.mpf(s))
        for s, ok, cur in zip(tg[name + "_s"], tg[name + "_curvature_ok"], tg[name + "_curvature"]):
            if ok:
                assert float(et.lookup(pe.mp.mpf(float(s)))[0]) == cur, (name, s)
            else:
                with pytest.raises(pe.LookupFailed):
                    et.lookup(pe.mp.mpf(float(s)))


def test_exact_cost_and_sysid_meet_the_reference_golden(gold):
    assert np.array_equal(pe.compute_cost(gold["pid_x"][:, 4], float(gold["track_length"])), gold["pid_Qfun"])
    ref = pe.regression(gold["pid_x"], gold["pid_u"], 1e-7)
    # the reference's own np.linalg.inv solve, measured against the exact one in the sysid bound's units
    assert pe.sysid_error(gold["lti_A"], gold["lti_B"], ref) <= pe.SYSID_C / 4
    assert 1e7 < ref["cond"] < 1e9


def test_numpy_dyn_model_calibration_on_the_case_list(cases):
    """NumPy's fp64 dynModel against the exact one on every simulator case of the GPU tests: the GPU bound leaves it a
    factor of 8 or more."""
    worst = 0.0
    for c in cases:
        r = pe.dyn_model(c.vehicle, c.exact_track, c.x, c.xg, c.u, z=c.z, noise=c.noise)
        assert c.boundary_case or r["margin"] >= 1e-9, (c.name, float(r["margin"]))
        xn, gn = nm.dyn_model(c.track_model, c.x, c.xg, c.u, c.vehicle, c.noise, rng=Draws(c.z))
        worst = max(worst, pe.sim_error(xn, r["x"]), pe.sim_error(gn, r["x_glob"]))
    assert worst <= pe.SIM_BOUND / 8, worst


def test_numpy_kernel_emulation_calibrates_the_sysid_bound():
    """The NumPy emulation of ridge_sysid_kernel's elimination stays within SYSID_C / 4 of the exact solution on every
    calibration record, so SYSID_C is at least four times what the kernel's arithmetic needs."""
    for x, u, lamb in pc.sysid_records():
        ref = pe.regression(x, u, lamb)
        A, B, flag = pe.regression_gauss_jordan(x, u, lamb)
        assert not flag
        assert pe.sysid_error(A, B, ref) <= pe.SYSID_C / 4, (x.shape[0], lamb)


MUTATIONS = ("alpha_r_lr", "curvature_at_next_s", "noise_global", "substeps_99", "substeps_101")


@pytest.mark.parametrize("variant", MUTATIONS)
def test_sim_bound_rejects_wrong_variants(cases, variant):
    """Each known-wrong dynModel misses the exact one by at least 100 SIM_BOUND on the case list (curvature_at_next_s only
    shows where a sub-step crosses a boundary and alpha_r_lr on a car with lf != lr, so they are measured on those cases)."""
    sel = {"curvature_at_next_s": [c for c in cases if c.crosses],
           "alpha_r_lr": [c for c in cases if c.vehicle.lf != c.vehicle.lr]}.get(variant, cases[::4])
    assert sel
    worst = 0.0
    for c in sel:
        r = pe.dyn_model(c.vehicle, c.exact_track, c.x, c.xg, c.u, z=c.z, noise=c.noise)
        w = pe.dyn_model(c.vehicle, c.exact_track, c.x, c.xg, c.u, z=c.z, noise=c.noise, variant=variant)
        worst = max(worst, pe.sim_error(pe.to_f64(w["x"]), r["x"]), pe.sim_error(pe.to_f64(w["x_glob"]), r["x_glob"]))
    assert worst >= 100 * pe.SIM_BOUND, (variant, worst)


@pytest.mark.parametrize("variant", ("rows_0", "no_lambda"))
def test_sysid_bound_rejects_wrong_variants(gold, variant):
    ref = pe.regression(gold["pid_x"], gold["pid_u"], 1e-7)
    w = pe.regression(gold["pid_x"], gold["pid_u"], 1e-7, variant=variant)
    assert pe.sysid_error(w["A"], w["B"], ref) >= 100 * pe.SYSID_C, variant


def test_cost_rejects_le_variant():
    """computeCost is integer-valued and checked bit for bit; a `<=` comparison changes it on a row with s == TrackLength."""
    L = 19.0
    for s, T in pc.cost_cases(L, 1024):
        if np.any(s == L):
            assert not np.array_equal(pe.compute_cost_le(s, L), pe.compute_cost(s, L)), T


def test_cost_cases_hit_the_chunk_edges():
    L = 19.0
    seen = set()
    for s, T in pc.cost_cases(L, 1024):
        q = pe.compute_cost(s, L)
        assert q[-1] == 0 and np.all(q >= 0) and np.all(q == np.round(q))
        for r in (0, 255, 256, T - 1):
            if r < T and not s[r] < L:
                seen.add(r if r != T - 1 else "last")
    assert {0, 255, 256, "last"} <= seen


def test_pid_exact_and_clip_edges():
    """PID.solve exactly: the clip edges sit where the cases say, and the fp64 form of the reference is within one ulp."""
    for c in pc.pid_cases():
        e = pe.pid_input(c.x, c.vt, c.z, c.noise.pid_sigma, c.noise.pid_clip)
        f = nm.PIDFollower(c.vt, c.noise, rng=Draws(c.z))
        f.solve(c.x)
        for j in range(2):
            assert abs(f.uPred[0, j] - float(e[j])) <= pe.ulp(e[j]) * c.ulps, (c.name, j)
