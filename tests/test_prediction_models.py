"""CPU tier: per-controller prediction models (lmpc_set_prediction_models) -- the ABI record and its packing, every refusal of
make_prediction_model_sets, the exact sensitivities of tests/support/nominal_model.py against numerical differentiation of the
exact plant, and the device bound rejecting every known-wrong variant at the test states."""
import ctypes as C
import math

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat
from racinglmpc_b200.reference_params import PredictionModelParams as P, VehicleParams as V
import nominal_model as nm

CARS = (V.reference(), V(2.5, 0.14, 0.11, 0.03, 9.0, 1.4, 1.2, 8.0, 1.3, 0.9), V(1.6, 0.11, 0.14, 0.02, 5.0, 1.2, 0.9, 5.5, 1.1, 1.1))
# (x, u): closed-loop states and edges (small vx, large slip, delta and a at their bounds)
STATES = (([1.3, 0.12, 0.6, 0.05, 3.0, 0.1], [0.2, 0.8]), ([2.5, -0.05, -0.4, 0.0, 9.0, -0.2], [-0.1, 0.3]),
          ([0.05, 0.0, 0.0, 0.0, 1.0, 0.0], [0.5, 10.0]), ([1.0, 0.8, -2.0, 0.1, 5.0, 0.2], [-0.5, -10.0]),
          ([0.2, 0.1, 1.5, -0.1, 2.0, 0.0], [0.0, 0.5]))


def test_abi_record_and_symbols():
    assert C.sizeof(nat.PredictionModelParams) == 88 == nat.lib().lmpc_sizeof_prediction_model_params()
    assert [getattr(nat.PredictionModelParams, f).offset for f in ("mode", "pad", "vehicle")] == [0, 4, 8]
    syms = nat.exported_symbols()
    for s in ("lmpc_set_prediction_models", "lmpc_sizeof_prediction_model_params"):
        assert s in syms
    assert nat.FLAG_NOMINAL_NONFINITE == 1024
    assert P.learned() == P(0, V.reference()) and P.plant().mode == 2 and P.believes(CARS[1]) == P(1, CARS[1])


def test_packing():
    rows, idx = nat.make_prediction_model_sets([P.learned(), P.believes(CARS[1]), P.plant()], [2, 0, 1, 1], 4)
    assert [r.mode for r in rows] == [0, 1, 2] and all(r.pad == 0 for r in rows)
    assert [getattr(rows[1].vehicle, f) for f in nat.VEHICLE_FIELDS] == [getattr(CARS[1], f) for f in nat.VEHICLE_FIELDS]
    assert idx.dtype == np.int32 and list(idx) == [2, 0, 1, 1]
    # modes 0 and 2 do not read the vehicle: any finite car, non-positive masses included, is accepted
    nat.make_prediction_model_sets([P(2, V(*[0.0] * 10)), P(0, V(*[-1.0] * 10))], [0, 1], 2)


def _with(field, value, mode=1):
    vals = {f: getattr(V.reference(), f) for f in nat.VEHICLE_FIELDS}
    vals[field] = value
    return P(mode, V(**vals))


@pytest.mark.parametrize("row", [P(3), P(-1), P(True), P(1.0), P("1"), _with("m", 0.0), _with("lf", -0.1), _with("lr", 0.0),
                                 _with("Iz", 0.0), _with("Df", math.nan), _with("Br", math.inf, 0), _with("Cf", -math.inf, 2),
                                 _with("m", "2.0"), _with("m", None, 2)])
def test_refused_rows(row):
    with pytest.raises(ValueError):
        nat.make_prediction_model_sets([row], np.zeros(2, int), 2)


def test_refused_indices():
    for idx in ([0, 1], [0], [0, 0, 0], [-1, 0], [0.5, 0]):
        with pytest.raises(ValueError):
            nat.make_prediction_model_sets([P.plant()], idx, 2)
    with pytest.raises(ValueError):
        nat.make_prediction_model_sets([P.plant()] * 3, [0, 1], 2)          # more rows than controllers


@pytest.mark.parametrize("car", range(len(CARS)))
def test_exact_sensitivities_equal_numerical_differentiation_of_the_plant(car):
    for x, u in STATES[:3]:
        phi, S = nm.phi_sens(CARS[car], x, u)
        phn, Sn = nm.numdiff(CARS[car], x, u)
        assert max(abs(float(a - b)) for a, b in zip(phi, phn)) < 1e-50      # the same map, evaluated to DPS digits
        err = max(abs(float(S[r][c] - Sn[r][c])) / (1 + abs(float(S[r][c]))) for r in range(3) for c in range(5))
        assert err < 1e-15, (x, u, err)


def _f64(rows):
    return [np.array([[float(q) for q in r] for r in rows[0]]), np.array([[float(q) for q in r] for r in rows[1]]),
            np.array([float(q) for q in rows[2]])]


def test_rounded_exact_rows_meet_the_bound_and_every_variant_is_rejected():
    for car in CARS:
        for x, u in STATES:
            exact = nm.rows(car, x, u)
            assert nm.deviation(_f64(exact), exact) <= 2.0 ** -52
            for v in nm.VARIANTS:
                if v == "alpha_r_lr" and car.lf == car.lr:
                    continue                            # the same model for a car with lf == lr
                assert nm.deviation(_f64(nm.rows(car, x, u, variant=v)), exact) > 1e3 * nm.NOMINAL_BOUND, (car, x, v)


def test_driver_refusals_and_start_model_rows():
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "benchmarks"))
    import rollout_mc as rmc
    ok = ([P.plant()], np.zeros(8, int))
    with pytest.raises(ValueError, match="lap_reports"):
        rmc.run(batch=8, laps=1, prediction_model_sets=ok)                 # the per-row summary needs the reports
    for bad in (([P(3)], np.zeros(8, int)), ([P(1, V(*[0.0] * 10))], np.zeros(8, int)), ([P.plant()], np.ones(8, int)),
                ([P.plant()], np.zeros(7, int)), ([_with("Df", math.nan, 2)], np.zeros(8, int))):
        with pytest.raises(ValueError):
            rmc.run(batch=8, laps=1, lap_reports=1, prediction_model_sets=bad)
    models = [P.learned(), P.believes(CARS[1])]
    packed = rmc.pack_tables(8, prediction_model_sets=(models, np.arange(8) % 2))[0]
    rows, idx = packed["prediction_model_sets"]
    assert len(idx) == 8 and rows[idx[1]].mode == 1
    assert [getattr(rows[idx[1]].vehicle, f) for f in nat.VEHICLE_FIELDS] == [getattr(CARS[1], f) for f in nat.VEHICLE_FIELDS]
    assert rmc.pack_tables(8, prediction_model_sets=None)[0] == {}
    had, none = rmc.table_rows(packed), {}
    other = rmc.table_rows(rmc.pack_tables(8, prediction_model_sets=([P.learned(), P.believes(CARS[1]), P.plant()],
                                                                      np.where(np.arange(8) == 3, 2, np.arange(8) % 2)))[0])
    for a, b in ((had, none), (none, had), (had, other)):
        with pytest.raises(ValueError, match="other prediction models"):
            rmc.check_start_tables(a, b)
    rmc.check_start_tables(had, rmc.table_rows(packed))
    rmc.check_start_tables(none, none)


def test_benchmark_prediction_error_and_table():
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "benchmarks"))
    import prediction_models as pm
    cap, N = 10, 12
    tr = {"steps": [], "x": [], "xPred": [], "lap": []}
    for t in range(2):
        x = np.zeros((cap, 6)); xp = np.zeros((cap, N + 1, 6))
        x[:, 0] = np.arange(cap)                                     # vx rises by 1 per step
        xp[:, 1, 0] = np.arange(cap) + 1 + 0.5 * t                   # predicted one step ahead, off by 0.5 for controller 1
        tr["steps"].append(cap); tr["x"].append(x); tr["xPred"].append(xp); tr["lap"].append(np.repeat([0, 1], 5).astype(np.int32))
    e = pm.prediction_error(tr, np.array([0, 1]), np.array([0, 1]), ["a", "b"], last_laps=1)
    assert e["a"]["steps"] == cap - 1 and e["a"]["rms"] == [0.0, 0.0, 0.0]
    assert e["b"]["rms"][0] == 0.5 and e["b"]["rms_last_laps"][0] == 0.5
    laps = 2
    study = {"benchmark": "t", "gpu": "g", "power_limit_w": None, "controllers_per_cell": 1, "laps": laps, "prediction_error": e,
             "cells": [{"prediction": "a", "per_lap": [{"steps_mean": 1.0, "violating_share": 0.0, "unsolved": 0}] * laps}]}
    assert "one-step prediction error" in pm.summary(study)
