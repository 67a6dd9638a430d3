"""CPU tier: lap schedules of the device closed loop (lmpc_rollout_set_lap_schedule).

The ABI (constants, symbol, prototype), every refusal of _native.make_lap_schedule, the both-order refusals of BatchedController
before any native call, the refusals of rollout_mc.run(lap_schedules=...) before any device work, the host restatement of which row
a controller reads (tests/support/lap_schedule.py) on synthetic lap_n sequences, and the driver's per-lap-row summary against
hand-built reports."""
import importlib.util
import os
import re
import sys

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat
from racinglmpc_b200 import reference_params as rp, sharding
from racinglmpc_b200.controller import BatchedController
from racinglmpc_b200.reference_params import VehicleParams, NoiseParams, MeasurementParams

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# tests/support/lap_schedule.py by its path: benchmarks/lap_schedule.py has the same module name and other test modules put
# benchmarks/ on sys.path
_spec = importlib.util.spec_from_file_location("lap_schedule_restatement", os.path.join(ROOT, "tests", "support", "lap_schedule.py"))
ls = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(ls)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
try:
    import rollout_mc  # noqa: E402
finally:
    sys.path.pop(0)          # benchmarks/ also holds modules named like tests/support's (lap_reports, lap_schedule)


def test_abi_constants_symbol_and_prototype():
    txt = re.sub(r"\s+", " ", open(os.path.join(ROOT, "include", "lmpc_b200.h")).read())
    assert "int lmpc_rollout_set_lap_schedule(lmpc_handle* h, int table, int nlaps, const int* row_of_lap);" in txt
    for name, v in (("VEHICLE", 0), ("NOISE", 1), ("MEASUREMENT", 2)):
        assert re.search(r"#define LMPC_SCHEDULE_%s %d\b" % (name, v), txt), name
        assert nat.LAP_SCHEDULE_TABLES[name.lower()] == v
    assert "lmpc_rollout_set_lap_schedule" in nat.exported_symbols()
    assert hasattr(nat.lib(), "lmpc_rollout_set_lap_schedule")
    assert nat.MAX_LAP_SCHEDULE == 1024


def test_make_lap_schedule_broadcasts_and_packs():
    s = nat.make_lap_schedule([0, 1, 1], 4, 2)
    assert s.dtype == np.int32 and s.flags["C_CONTIGUOUS"] and s.shape == (4, 3)
    assert np.array_equal(s, np.tile([0, 1, 1], (4, 1)))
    full = np.arange(8).reshape(4, 2) % 3
    assert np.array_equal(nat.make_lap_schedule(full, 4, 3), full)
    assert np.array_equal(nat.make_lap_schedule(np.array([2.0]), 4, 3), np.full((4, 1), 2))
    assert nat.make_lap_schedule(np.zeros(1024, np.int64), 2, 1).shape == (2, 1024)


@pytest.mark.parametrize("rows, nsets, what", [
    ([], 2, "L >= 1"), (np.zeros((4, 0), int), 2, "L >= 1"), (np.zeros(1025, int), 2, "1 .. 1024"),
    (np.zeros((3, 2), int), 2, "needs 4 rows"), (np.zeros((5, 2), int), 2, "needs 4 rows"), (np.zeros((4, 2, 1), int), 2, r"\[L\]"),
    ([0, 2], 2, "out of range"), ([-1, 0], 2, "out of range"), ([0, 0], 0, "out of range"),
    ([0.5, 1], 2, "integer"), ([np.nan], 2, "integer"), ([True, False], 2, "integer"), (["0"], 2, "integer"), (0, 2, r"\[L\]")])
def test_make_lap_schedule_refusals(rows, nsets, what):
    with pytest.raises(ValueError, match=what):
        nat.make_lap_schedule(rows, 4, nsets)


class _Recorder:
    """A stand-in library: records every lmpc_* call and returns LMPC_OK."""
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("lmpc_"):
            raise AttributeError(name)
        return lambda *a: self.calls.append(name) or 0


@pytest.fixture
def host(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(nat, "lib", lambda: rec)
    _, _, _, _, Qts, par = rp.lmpc_params(12)
    c = BatchedController(par, 4, np.array([[0.0, 19.3, 0.0]]), 19.3, trToUse=4, numSS_Points=48, numSS_it=4, QterminalSlack=Qts,
                          Tmax=64, ss_cap=6, model_cap=5)
    c.enable_rollout(Tcl=64)
    rec.calls.clear()
    return c, rec


V2 = [VehicleParams.reference(), VehicleParams.from_friction(0.6)]
N2 = [NoiseParams.reference(), NoiseParams.scaled(2, 1)]
M2 = [MeasurementParams.zero(), MeasurementParams.zero()]


def test_controller_installs_and_reports_its_schedules(host):
    c, rec = host
    assert c.lap_schedule_of("vehicle") is None
    c.set_vehicles(V2, [0, 1, 0, 1])
    c.set_lap_schedule("vehicle", [0, 1])
    assert rec.calls[-1] == "lmpc_rollout_set_lap_schedule"
    assert np.array_equal(c.lap_schedule_of("vehicle"), np.tile([0, 1], (4, 1)))
    c.set_lap_schedule("vehicle", None)
    assert c.lap_schedule_of("vehicle") is None and rec.calls[-1] == "lmpc_rollout_set_lap_schedule"


def test_controller_refusals_before_any_native_call(host):
    c, rec = host
    with pytest.raises(ValueError, match="kind"):
        c.set_lap_schedule("track", [0])
    with pytest.raises(ValueError, match="out of range"):
        c.set_lap_schedule("vehicle", [0, 1])                   # the reference vehicle is one row
    with pytest.raises(ValueError, match="measurement table"):
        c.set_lap_schedule("measurement", [0])
    with pytest.raises(ValueError, match="kind"):
        c.lap_schedule_of("params")
    fresh = object.__new__(BatchedController)
    fresh._lib = None
    with pytest.raises(ValueError, match="enable_rollout"):
        fresh.set_lap_schedule("noise", [0])
    assert rec.calls == []


@pytest.mark.parametrize("kind, install, two", [("vehicle", "set_vehicles", V2), ("noise", "set_noise", N2),
                                                ("measurement", "set_measurement_noise", M2)])
def test_both_install_orders_are_refused_before_any_native_call(host, kind, install, two):
    c, rec = host
    getattr(c, install)(two, [0, 1, 1, 0])
    c.set_lap_schedule(kind, [[0, 1]] * 4)
    rec.calls.clear()
    with pytest.raises(ValueError, match="names row 1"):
        getattr(c, install)(two[:1], [0, 0, 0, 0])               # one row does not cover entry 1
    with pytest.raises(ValueError, match="names row 1"):
        getattr(c, install)(None)                                 # the revert leaves one row (or none: measurement)
    assert rec.calls == []
    getattr(c, install)(two + two[:1], [0, 1, 2, 0])              # three rows cover it
    c.set_lap_schedule(kind, [0])                                 # a schedule inside row 0 ...
    getattr(c, install)(two[:1], [0, 0, 0, 0])                    # ... lets one row in
    if kind != "measurement":
        getattr(c, install)(None)
    else:
        with pytest.raises(ValueError, match="names row 0"):
            c.set_measurement_noise(None)                         # no table has no row 0
        c.set_lap_schedule(kind, None)
        c.set_measurement_noise(None)


def _no_device(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(rollout_mc.torch.cuda, "set_device", no_device)
    monkeypatch.setattr(rollout_mc, "BatchedController", no_device)


VS = (V2, np.zeros(8, np.int32))


@pytest.mark.parametrize("kw, what", [
    (dict(lap_schedules={"vehicle": [0, 1]}, lap_reports=3), "needs vehicle_sets"),
    (dict(lap_schedules={"noise": [0]}, vehicle_sets=VS, lap_reports=3), "needs noise_sets"),
    (dict(lap_schedules={"measurement": [0]}, lap_reports=3), "needs measurement_sets"),
    (dict(lap_schedules={"vehicle": [0, 1]}, vehicle_sets=VS), "lap_reports"),
    (dict(lap_schedules={"vehicle": [0, 1]}, vehicle_sets=VS, lap_reports=2), "fewer rows"),
    (dict(lap_schedules={"vehicle": [0, 2]}, vehicle_sets=VS, lap_reports=3), "out of range"),
    (dict(lap_schedules={"track": [0]}, lap_reports=3), "kind"),
    (dict(lap_schedules=[0, 1], vehicle_sets=VS, lap_reports=3), "dict")])
def test_run_refusals_before_device_work(kw, what, monkeypatch):
    _no_device(monkeypatch)
    with pytest.raises(ValueError, match=what):
        rollout_mc.run(batch=8, laps=3, **kw)


def _start(scheds):
    s = {k: 0 for k in sharding.ExchangeSchedule.FIELDS}
    s.update(records=np.zeros((8, 16), np.uint8), clock=0, batch=8, laps=3, mode="pooled", readiness="batch", poll=8, warm=False,
             pool_groups=1, layout=dict(rollout_mc.layout(lap_reports=8), bytes=16), lap_schedules=scheds,
             tables=rollout_mc.table_rows(rollout_mc.pack_tables(8, vehicle_sets=VS)[0]))
    return s


@pytest.mark.parametrize("captured, now", [({"vehicle": [[0, 1]] * 8}, None), ({}, {"vehicle": [0, 1]}),
                                           ({"vehicle": [[0, 1]] * 8}, {"vehicle": [1, 0]}),
                                           ({"vehicle": [[0, 1]] * 8}, {"vehicle": [0, 1, 1]})])
def test_run_start_refuses_other_schedules(captured, now, monkeypatch):
    _no_device(monkeypatch)
    with pytest.raises(ValueError, match="lap_schedules"):
        rollout_mc.run(batch=8, laps=5, start=_start(captured), lap_reports=8, vehicle_sets=VS, lap_schedules=now)


# ---- the restatement on synthetic lap_n sequences ------------------------------------------------------------------------------
def test_rows_follow_lap_n_and_the_last_entry_holds():
    lap_n = np.array([[0, 0, 3], [0, 1, 4], [1, 2, 9], [2, 2, 1000]])
    sched = np.array([[5, 6, 7], [1, 2, 3], [0, 4, 8]])
    got = ls.rows_read(lap_n, own=[9, 9, 9], schedule=sched)
    assert got.tolist() == [[5, 1, 8], [5, 2, 8], [6, 3, 8], [7, 3, 8]]
    assert ls.rows_read(lap_n, own=[4, 5, 6]).tolist() == [[4, 5, 6]] * 4
    assert ls.host_switch_index(lap_n[3], sched).tolist() == [7, 3, 8]


def test_pid_steps_read_the_own_index_and_retired_controllers_read_nothing():
    lap_n = np.array([[0, 0], [0, 0], [1, 0], [2, 1], [2, 1]])
    sched = np.array([[1, 2, 3], [3, 2, 1]])
    pid = [True, False, False, False, False]
    got = ls.rows_read(lap_n, own=[0, 0], schedule=sched, budget=[2, 16], pid=pid)
    assert got.tolist() == [[0, 0], [1, 3], [2, 3], [ls.RETIRED, 2], [ls.RETIRED, 2]]
    # raising the budget revives a controller at the entry its lap_n names
    assert ls.rows_read(lap_n[3:], own=[0, 0], schedule=sched, budget=[3, 16]).tolist() == [[3, 2], [3, 2]]


def _reports(n, steps, viol, unsolved):
    return {"n": np.asarray(n), "steps": np.asarray(steps), "viol_steps": np.asarray(viol), "unsolved": np.asarray(unsolved)}


def test_per_lap_row_summary_against_hand_built_reports():
    reps = _reports(n=[2, 3, 1, 3],
                    steps=[[100, 110, 0], [90, 95, 97], [120, 0, 0], [80, 85, 86]],
                    viol=[[0, 2, 0], [1, 0, 0], [0, 0, 0], [0, 0, 3]],
                    unsolved=[[0, 1, 0], [2, 0, 0], [0, 0, 0], [0, 0, 5]])
    sched = {"vehicle": np.array([[0, 1], [0, 1], [1, 1], [1, 0]])}
    got = rollout_mc.lap_row_summary(reps, sched, 3)["vehicle"]
    want = [(1, 0, 2, 95.0, 0.5, 2), (1, 1, 2, 100.0, 0.0, 0),
            (2, 0, 1, 85.0, 0.0, 0), (2, 1, 2, 102.5, 0.5, 1),        # controller 2 filed no lap 2
            (3, 0, 1, 86.0, 1.0, 5), (3, 1, 1, 97.0, 0.0, 0)]         # lap 3 is past L = 2: the last entry holds
    assert [(r["lap"], r["row"], r["controllers"], r["steps_mean"], r["violating_share"], r["unsolved"]) for r in got] == want
