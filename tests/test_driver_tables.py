"""CPU tier: the table arguments of rollout_mc.run as one list (rollout_mc.TABLES).

For every table: a bad index is refused before any device work; start refuses a capture taken without the table, a run without
the table, and other rows, and accepts the same rows; run()'s table keywords are exactly the list's; and the per-row statistics
(rollout_mc.table_stats) carry each table's row fields on synthetic books and reports, with the entries that join tables."""
import inspect
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat, reference_params as rp, sharding
from racinglmpc_b200.controller import BatchedController
from racinglmpc_b200.reference_params import (LaneMarginParams as G, LaneRuleParams as R, LapWindowParams as W,
                                              MeasurementParams as Ms, NoiseParams as Ns, PredictionModelParams as P,
                                              RegressionParams as Rg, SurfaceParams as S, TrackParams as T, VehicleParams as V)

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "benchmarks"))
try:
    import rollout_mc as rmc
finally:
    sys.path.pop(0)                                 # benchmarks/ holds module names that tests/support also uses

B = 8
IDX = np.arange(B) % 2


def _par(width):
    p = rp.lmpc_params(12)[5]
    return SimpleNamespace(**{**vars(p), "bx": np.array([width, width])})


# keyword: (two rows, the same table with one row changed); every pair installs together (the statistics test packs them all)
ROWS = {
    "param_sets": (([_par(0.4), _par(0.3)], IDX, None), ([_par(0.4), _par(0.35)], IDX, None)),
    "vehicle_sets": (([V.reference(), V.from_friction(0.6)], IDX), ([V.reference(), V.from_friction(0.5)], IDX)),
    "noise_sets": (([Ns.reference(), Ns.scaled(2.0)], IDX), ([Ns.reference(), Ns.scaled(3.0)], IDX)),
    "noise_streams": (np.arange(B) // 2, np.arange(B)),
    "measurement_sets": (([Ms.zero(), Ms((0.01,) * 6, (0.05,) * 6)], IDX), ([Ms.zero(), Ms((0.02,) * 6, (0.05,) * 6)], IDX)),
    "regression_sets": (([Rg.reference(), Rg.reference(2)], IDX), ([Rg.reference(), Rg.reference(3)], IDX)),
    "track_sets": (([T.l_shaped(), T.oval()], IDX), ([T.l_shaped(), T.goggle()], IDX)),
    "pool_groups": ((IDX, 2), (1 - IDX, 2)),
    "shape_sets": (([(12, 48), (6, 48)], IDX), ([(12, 48), (8, 48)], IDX)),
    "ss_laps_sets": (([4, 2], IDX), ([4, 1], IDX)),
    "lap_window_sets": (([W(0, 0), W(4, 4)], IDX), ([W(0, 0), W(5, 4)], IDX)),
    "lane_rule_sets": (([R(0, 0.0), R(1, 0.05)], IDX), ([R(0, 0.0), R(1, 0.1)], IDX)),
    "lane_margin_sets": (([G(1, 0.1, 0.1), G(2, 0.0, 0.1, 0.01, 0.0)], IDX), ([G(1, 0.2, 0.2), G(2, 0.0, 0.1, 0.01, 0.0)], IDX)),
    "prediction_model_sets": (([P.learned(), P.plant()], IDX), ([P.learned(), P.believes(V.from_friction(0.6))], IDX)),
    "surface_sets": (([S.dry(), S.from_zones([(0.0, 1.0, 0.5, 0.5)])], IDX), ([S.dry(), S.from_zones([(0.0, 1.0, 0.6, 0.5)])], IDX)),
}
KEYWORDS = [t.keyword for t in rmc.TABLES]
NAME = {t.keyword: t.name for t in rmc.TABLES}
# run()'s arguments that are not tables
NOT_TABLES = {"batch", "laps", "mode", "share", "tpad", "ship_after", "poll", "max_steps", "seed", "local", "warm", "final", "books",
              "readiness", "capture", "start", "lap_budget", "lap_reports", "lap_schedules", "trace"}


def _bad_index(kw):
    """The table of ROWS with an index one controller short."""
    good = ROWS[kw][0]
    if kw == "noise_streams":
        return good[:-1]
    if kw == "pool_groups":
        return good[0][:-1], good[1]
    return (good[0], good[1][:-1]) + tuple(good[2:])


def _no_device(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(rmc.torch.cuda, "set_device", no_device)
    monkeypatch.setattr(rmc, "BatchedController", no_device)


def _rows(**tables):
    return rmc.table_rows(rmc.pack_tables(B, **tables)[0])


def _start(**tables):
    s = {k: 0 for k in sharding.ExchangeSchedule.FIELDS}
    s.update(records=np.zeros((B, 16), np.uint8), clock=0, batch=B, laps=1, mode="independent", readiness="batch", poll=8,
             warm=False, pool_groups=int(tables["pool_groups"][1]) if "pool_groups" in tables else 1,
             layout=dict(rmc.layout(lap_reports=2), bytes=16), tables=_rows(**tables))
    return s


@pytest.mark.parametrize("kw", KEYWORDS)
def test_a_bad_index_is_refused_before_any_device_work(kw, monkeypatch):
    _no_device(monkeypatch)
    with pytest.raises(ValueError):
        rmc.run(batch=B, laps=1, mode="independent", lap_reports=1, **{kw: _bad_index(kw)})
    with pytest.raises(AssertionError, match="device work"):                  # the same table with its index goes on
        rmc.run(batch=B, laps=1, mode="independent", lap_reports=1, **{kw: ROWS[kw][0]})


@pytest.mark.parametrize("kw", KEYWORDS)
def test_start_refuses_other_tables_and_accepts_the_same_rows(kw, monkeypatch):
    rows, other = ROWS[kw]
    mine, none = _rows(**{kw: rows}), _rows()
    assert none == {} and list(mine) == [kw] and _rows(**{kw: other})[kw] != mine[kw]
    for had, now in ((none, mine), (mine, none), (mine, _rows(**{kw: other}))):
        with pytest.raises(ValueError, match="start was captured with other %s" % NAME[kw]):
            rmc.check_start_tables(had, now)
    rmc.check_start_tables(mine, _rows(**{kw: rows}))
    # the same rules in run(), before any device work
    _no_device(monkeypatch)
    for had, now in (({}, {kw: rows}), ({kw: rows}, {}), ({kw: rows}, {kw: other})):
        start = _start(**had)
        if kw == "pool_groups":
            start["pool_groups"] = now[kw][1] if now else 1                   # the group count has its own refusal
        with pytest.raises(ValueError, match="other %s" % NAME[kw]):
            rmc.run(batch=B, laps=2, mode="independent", lap_reports=2, start=start, **now)
    with pytest.raises(AssertionError, match="device work"):
        rmc.run(batch=B, laps=2, mode="independent", lap_reports=2, start=_start(**{kw: rows}), **{kw: rows})


def test_the_tables_of_run_are_the_list():
    params = set(inspect.signature(rmc.run).parameters)
    assert params - NOT_TABLES == set(KEYWORDS) and len(KEYWORDS) == len(set(KEYWORDS)) == 15 == len(ROWS)
    assert KEYWORDS.index("param_sets") < KEYWORDS.index("lane_margin_sets")      # margins read the parameter rows' lanes
    assert KEYWORDS.index("ss_laps_sets") < KEYWORDS.index("lap_window_sets")     # windows read the lap counts
    for t in rmc.TABLES:
        assert callable(getattr(BatchedController, t.install)), t.install
    keys = [t.key for t in rmc.TABLES if t.key is not None]
    assert len(keys) == len(set(keys)) == 13


def _synthetic(laps=3, seed=5):
    rng = np.random.default_rng(seed)
    L = 4
    ss_time = rng.integers(100, 300, (B, 7)).astype(np.int32)
    ss_time[rng.random((B, 7)) < 0.3] += nat.LANE_UNSAFE_KEY
    bk = dict(lap_hist=rng.integers(150, 250, (B, 16)).astype(np.int32), lap_n=rng.integers(0, laps + 1, B).astype(np.int32),
              ss_time=ss_time, sel=rng.integers(0, 7, (B, 4)).astype(np.int32), it=rng.integers(4, 12, B).astype(np.int32),
              flags_or=np.where(rng.random(B) < 0.3, 64, 0).astype(np.int32), unsolved=rng.integers(0, 3, B).astype(np.int32),
              lane_margins=rng.random(B) * 0.1)
    reps = dict(n=rng.integers(0, laps + 1, B).astype(np.int32), steps=rng.integers(150, 250, (B, L)).astype(np.int32),
                flags=np.where(rng.random((B, L)) < 0.4, nat.REPORT_LANE_UNSAFE, 0).astype(np.int32),
                unsolved=rng.integers(0, 2, (B, L)).astype(np.int32), viol_steps=rng.integers(0, 3, (B, L)).astype(np.int32),
                viol_max=rng.random((B, L)), ipm_iters=rng.integers(1000, 3000, (B, L)).astype(np.int32))
    bk["lap_reports"] = reps
    return bk, reps, rng.random(B) * 40.0


# keyword: the row fields of its per-row entries today, by row, and whether they carry the sampled iterations
FIELDS = {
    "shape_sets": ([dict(N=12, numSS_Points=48), dict(N=6, numSS_Points=48)], True),
    "ss_laps_sets": ([dict(numSS_it=4), dict(numSS_it=2)], True),
    "lap_window_sets": ([dict(ss_window=0, model_window=0), dict(ss_window=4, model_window=4)], True),
    "lane_rule_sets": ([dict(mode=0, lane_tol=0.0), dict(mode=1, lane_tol=0.05)], True),
    "lane_margin_sets": ([dict(mode=1, margin0=0.1, margin_max=0.1, step_up=0.0, step_down=0.0),
                          dict(mode=2, margin0=0.0, margin_max=0.1, step_up=0.01, step_down=0.0)], True),
    "prediction_model_sets": ([dict(mode=0), dict(mode=2)], False),
}


@pytest.mark.parametrize("with_reports", [True, False])
def test_statistics_carry_each_tables_row_fields(with_reports):
    laps, it_n = 3, 5
    bk, reps, it_ctrl = _synthetic(laps)
    if not with_reports:
        del bk["lap_reports"]
        reps = None
    packed, ctx = rmc.pack_tables(B, **{kw: rows for kw, (rows, _) in ROWS.items()})
    out = rmc.table_stats(packed, ctx, bk, it_ctrl, it_n, laps)
    for t in rmc.TABLES:
        if t.key is None:
            assert t.keyword in ("noise_streams", "pool_groups")
            continue
        fields, ipm = FIELDS.get(t.keyword, ([{}, {}], False))
        assert len(out[t.key]) == 2
        for k, s in enumerate(out[t.key]):
            sel = IDX == k
            want = rmc._set_stats(bk, bk["flags_or"], bk["unsolved"], sel, laps, reps)
            want.update(fields[k])
            if ipm:
                want["ipm_iters_mean_sampled"] = float(it_ctrl[sel].mean() / it_n)
            if t.keyword == "lane_rule_sets" and reps is not None:
                for r, row in enumerate(want["reports"]):
                    m = sel & (reps["n"] > r)
                    row["lane_unsafe_share"] = float(((reps["flags"][m, r] & nat.REPORT_LANE_UNSAFE) != 0).mean()) if m.any() else 0.0
            assert s == want, (t.keyword, k)
            assert all(type(s[f]) is type(v) for f, v in fields[k].items())
    # the entries that join tables
    assert out["handle_shape"] == [12, 48]
    cells = out["per_shape_ss_laps_rank0"]
    assert [(c["N"], c["numSS_Points"], c["numSS_it"]) for c in cells] == [(12, 48, 4), (6, 48, 2)]
    for k, c in enumerate(cells):
        assert c["controllers"] == int((IDX == k).sum()) and c["ipm_iters_mean_sampled"] == float(it_ctrl[IDX == k].mean() / it_n)
    nit = np.where(IDX == 0, 4, 2)
    unsafe = bk["ss_time"] >= nat.LANE_UNSAFE_KEY
    held = [unsafe[b, bk["sel"][b, :nit[b]]].any() for b in range(B)]
    assert out["lane_unsafe_selected_share_rank0"] == float(np.mean(held))
    if reps is not None:
        everyone = rmc.lap_report_summary(reps, np.ones(B, bool), laps)
        assert [{k: v for k, v in r.items() if k != "lane_unsafe_share"} for r in out["lap_reports_rank0"]] == everyone
        for r, row in enumerate(out["lap_reports_rank0"]):
            m = reps["n"] > r
            assert row["lane_unsafe_share"] == (float(((reps["flags"][m, r] & nat.REPORT_LANE_UNSAFE) != 0).mean()) if m.any() else 0.0)
    else:
        assert "lap_reports_rank0" not in out
    for k, f in enumerate(out["lane_margin_final_rank0"]):
        m = bk["lane_margins"][IDX == k]
        assert f == {"row": k, "n": m.size, "min": float(m.min()), "mean": float(m.mean()), "max": float(m.max())}
    assert rmc.table_stats({}, ctx, bk, it_ctrl, it_n, laps) == {}
