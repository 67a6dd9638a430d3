"""CPU tier: per-controller regression models (lmpc_set_regression_sets).

reference_params.RegressionParams against the oracle's PredictiveModel constants, the struct and the exported symbols, every
refusal of _native.make_regression_sets, and the certified scaling range of K1's fp32 pre-filter: the knn_fixtures groups with
their scaling and bandwidth moved to both ends of the range (tests/support/regression_sets.py) reach the branches and candidates
of the unscaled groups with the same margin (>= 2^-20), and the weakened pre-filters lose selected rows there as they do at the
reference's scaling."""
import ctypes as C
import dataclasses
import math

import numpy as np
import pytest

import knn_fixtures as kf
import regression_sets as rs
from oracle import ltv_model
from racinglmpc_b200 import _native as nat
from racinglmpc_b200.reference_params import RegressionParams

B = 32
REF = RegressionParams.reference()
SCALED_GROUPS = ("default_N12", "k1_h50_ridge", "k3_h0.5", "negative_scaling")


def test_reference_equals_the_oracle_constants():
    for tr in (1, 4):
        m = ltv_model.LocalLTVModel(6, 2, None, tr)
        r = RegressionParams.reference(tr)
        assert r.trToUse == len(m.usedIt) == tr
        assert r.MaxNumPoint == m.MaxNumPoint and r.h == m.h and r.lamb == m.lamb
        assert np.array_equal(np.diag(r.scaling), m.scaling)
    assert REF.trToUse == 4                       # LMPC's PredictiveModel (main.py:102)


def test_library_exports_the_call_and_the_struct_size_matches():
    syms = nat.exported_symbols()
    assert {"lmpc_set_regression_sets", "lmpc_sizeof_regression_params"} <= set(syms)
    L = nat.lib()                                 # asserts lmpc_sizeof_regression_params() == sizeof(RegressionParams)
    assert L.lmpc_sizeof_regression_params() == C.sizeof(nat.RegressionParams) == 64


def test_valid_sets_pack_field_by_field():
    regs = [REF, RegressionParams(1, 1, 0.5, 1e-6, (-0.1, 2.0 ** 32, 0.0, 2.0 ** -32, 1.0)), RegressionParams.reference(2)]
    idx = (5 * np.arange(B)) % 3
    packed, pidx = nat.make_regression_sets(regs, idx, B, trToUse=4)
    assert len(packed) == 3 and pidx.dtype == np.int32 and np.array_equal(pidx, idx)
    for k, r in enumerate(regs):
        assert (packed[k].trToUse, packed[k].MaxNumPoint, packed[k].h, packed[k].lamb) == (r.trToUse, r.MaxNumPoint, r.h, r.lamb)
        assert list(packed[k].scaling) == list(r.scaling)


@pytest.mark.parametrize("index", [np.zeros(B - 1, int), np.zeros(B + 1, int), np.full(B, 2), np.full(B, -1), np.full(B, 0.5), None])
def test_bad_index_is_a_value_error(index):
    with pytest.raises(ValueError):
        nat.make_regression_sets([REF] * 2, index, B, trToUse=4)


def test_no_sets_or_more_than_batch_is_a_value_error():
    with pytest.raises(ValueError):
        nat.make_regression_sets([], np.zeros(B, int), B, trToUse=4)
    with pytest.raises(ValueError):
        nat.make_regression_sets([REF] * (B + 1), np.zeros(B, int), B, trToUse=4)


def _scal(j, v):
    s = list(REF.scaling)
    s[j] = v
    return tuple(s)


BAD = ([("trToUse", v) for v in (0, -1, 5, 2.0, True)] + [("MaxNumPoint", v) for v in (0, 8, -3, 7.0)] +
       [("h", v) for v in (0.0, -5.0, math.nan, math.inf, 2.0 ** -1023, 5e-324, 2.0 ** 1023)] +
       [("lamb", v) for v in (-1e-12, math.nan, math.inf)] +
       [("scaling", _scal(j, v)) for j in (0, 4) for v in (math.nan, math.inf, -math.inf, 2.0 ** 33, -(2.0 ** 32) * 1.000001,
                                                          2.0 ** -33, 1e-300, 5e-324)] +
       [("scaling", (0.1, 1.0, 1.0, 1.0)), ("scaling", (0.1, 1.0, 1.0, 1.0, 1.0, 1.0))])


@pytest.mark.parametrize("field,value", BAD, ids=["%s=%r" % fv for fv in BAD])
def test_bad_value_is_a_value_error(field, value):
    with pytest.raises(ValueError):
        nat.make_regression_sets([REF, dataclasses.replace(REF, **{field: value})], np.arange(B) % 2, B, trToUse=4)


def test_range_ends_and_zero_scaling_are_admitted():
    ok = [RegressionParams(4, 7, 2.0 ** -1022, 0.0, (2.0 ** -32, -(2.0 ** 32), 0.0, -0.0, 1.0)),
          RegressionParams(1, 1, 2.0 ** 1022, 1e300, (0.0,) * 5)]
    packed, _ = nat.make_regression_sets(ok, np.arange(B) % 2, B, trToUse=4)
    assert packed[0].scaling[1] == -(2.0 ** 32)   # packed as given: the library takes |s|
    with pytest.raises(ValueError):
        nat.make_regression_sets(ok, np.arange(B) % 2, B, trToUse=3)     # trToUse above the store's


# ---- the certified range: the fixtures with their scaling and bandwidth at both ends of it
def _groups():
    return {g.name: g for g in kf.groups()}


def test_scaled_fixture_sets_are_at_the_ends_of_the_admitted_range():
    gs = _groups()
    lo = [rs.set_of(rs.scaled(gs[n], rs.LOW)) for n in SCALED_GROUPS]
    hi = [rs.set_of(rs.scaled(gs[n], rs.HIGH)) for n in SCALED_GROUPS]
    nat.make_regression_sets(lo + hi, np.arange(B) % (2 * len(SCALED_GROUPS)), B, trToUse=8)
    a_lo = np.abs(np.array([r.scaling for r in lo]))
    a_hi = np.abs(np.array([r.scaling for r in hi]))
    assert a_lo[a_lo > 0].min() < 2 * 2.0 ** -32 and a_hi.max() == 2.0 ** 32
    kk = {r.MaxNumPoint for r in lo} | {r.MaxNumPoint for r in hi}
    assert {1, 7} <= kk                            # both ends of MaxNumPoint, h from 0.5 to 50 times 2^k
    assert {r.h for r in hi} >= {0.5 * 2.0 ** 32, 50.0 * 2.0 ** 32}


CASES = [(n, k, fi) for n in SCALED_GROUPS for k in (rs.LOW, rs.HIGH) for fi in range(len(_groups()[n].fixtures))]


@pytest.mark.parametrize("case", CASES, ids=["%s/2^%d/%s" % (n, k, _groups()[n].fixtures[fi].name) for n, k, fi in CASES])
def test_scaled_fixture_reaches_the_same_branch_with_margin(case):
    """Same candidates, same branch (a lap shorter than k rows: `open` at the reference's scaling, the padding key as G below
    it -- both admit every stored row), every decision >= 2^-20 from flipping."""
    n, k, fi = case
    g = _groups()[n]
    sg = rs.scaled(g, k)
    fx = g.fixtures[fi]
    worst = np.inf
    for i in range(g.N):
        q5 = kf.query(fx, i)
        for x, u in kf.used_laps(fx, g.trToUse):
            p0 = kf.prefilter(x, u, q5, g.consts)
            p1 = kf.prefilter(x, u, q5, sg.consts)
            assert p1.branch == p0.branch or (p0.branch == "open" and p1.branch == "fast"), (fx.name, i, p0.branch, p1.branch)
            assert p1.nc == p0.nc and np.array_equal(p1.cand, p0.cand), (fx.name, i)
            assert kf.min_margin(p1) >= kf.MARGIN, (fx.name, i, p1.margins)
            worst = min(worst, kf.min_margin(p1))
    print("%-40s 2^%d margin %.2e" % (fx.name, k, worst))


def _lost(group, names, mutation):
    out = {}
    for fx in group.fixtures:
        if fx.name not in names:
            continue
        n = 0
        for i in range(group.N):
            m = kf.exact_model(fx, group, exact=False)
            m.model(fx.xLin[i], fx.uLin[i])
            for c, (x, u) in enumerate(kf.used_laps(fx, group.trToUse)):
                p = kf.prefilter(x, u, kf.query(fx, i), group.consts, **mutation)
                n += not set(np.atleast_1d(m.last_indices[c]).tolist()) <= set(p.cand.tolist())
        out[fx.name] = n
    return out


@pytest.mark.parametrize("k", [rs.LOW, rs.HIGH])
@pytest.mark.parametrize("mutation, must_catch", [(dict(c_abs=0.0), "magnitude_margin"), (dict(recollect=False), "lane_packing")],
                         ids=["no_rounding_term", "no_recollect"])
def test_a_weakened_prefilter_loses_selected_rows_at_the_range_ends(k, mutation, must_catch):
    sg = rs.scaled(_groups()["default_N12"], k)
    lost = _lost(sg, {must_catch}, mutation)
    print("2^%d weakened %s loses selected rows: %s" % (k, mutation, lost))
    assert lost[must_catch] > 0
    assert _lost(sg, {must_catch}, {})[must_catch] == 0
