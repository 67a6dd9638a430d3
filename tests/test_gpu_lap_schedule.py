"""GPU tier: lap schedules of the device-resident closed loop (lmpc_rollout_set_lap_schedule).

Every check is bit for bit.  A schedule whose every entry is the controller's own table index is the closed loop without one; a
scheduled batch equals a second handle of the same batch on which the host re-installs the plain table whenever a controller's
entry changes (lap_n read after every hand-over); the PID lap ignores schedules; a controller that retires mid-schedule stays put and
revives at the entry its lap_n names; a snapshot resumes at its entry; refused calls leave the handle as it was."""
import ctypes as C
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                # noqa: E402
from racinglmpc_b200 import _native as nat                        # noqa: E402
from racinglmpc_b200.controller import BatchedController          # noqa: E402
from racinglmpc_b200.export import RolloutTrace                   # noqa: E402
from racinglmpc_b200.reference_params import TrackParams, VehicleParams, NoiseParams, MeasurementParams   # noqa: E402
from closed_loop import N, X0                                     # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# tests/support/lap_schedule.py by its path: benchmarks/lap_schedule.py has the same module name and other test modules put
# benchmarks/ on sys.path
_spec = importlib.util.spec_from_file_location("lap_schedule_restatement", os.path.join(ROOT, "tests", "support", "lap_schedule.py"))
ls = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(ls)
LMPC_E_INVALID, LMPC_E_STATE = -1, -4
INT32_MAX = 2 ** 31 - 1
THREE = [TrackParams.l_shaped(), TrackParams.goggle(), TrackParams.oval()]
B = 24
TIDX = (np.arange(B) % 3).astype(np.int32)
SEED = 1234
KIND = nat.LAP_SCHEDULE_TABLES
# the plant-side tables: three cars, two noise models, two sensors; own index of every controller
TABLES = {"vehicle": ([VehicleParams.from_friction(mu) for mu in (0.8, 0.6, 1.0)], (np.arange(B) // 3) % 3),
          "noise": ([NoiseParams.reference(), NoiseParams.scaled(3, 1)], (np.arange(B) // 2) % 2),
          "measurement": ([MeasurementParams.zero(), MeasurementParams((0.01, 0.005, 0.005, 0.002, 0.005, 0.005), (0.05,) * 6)],
                          (np.arange(B) // 4) % 2)}
INSTALL = {"vehicle": "set_vehicles", "noise": "set_noise", "measurement": "set_measurement_noise"}


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _rollout_mc():
    sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
    try:
        import rollout_mc
    finally:
        sys.path.pop(0)
    return rollout_mc


def _handle(kinds, sched=None, reports=16, trace=None, budget=None):
    """A controller per circuit of THREE with the tables of `kinds` at their own index, reports on, optionally traced; `sched`
    ({kind: [B, L]}) is installed before the PID lap.  PID lap and seeding done."""
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    t0 = TrackParams.l_shaped()
    c = BatchedController(par, B, t0.seg_table, t0.TrackLength, trToUse=4, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=1280, ss_cap=7, model_cap=5)
    c.set_tracks(THREE, TIDX)
    c.enable_rollout(Tcl=1024)
    for k in kinds:
        getattr(c, INSTALL[k])(*TABLES[k])
    if reports:
        c.enable_lap_reports(reports)
    for k, s in (sched or {}).items():
        c.set_lap_schedule(k, s)
    if budget is not None:
        c.set_lap_budget(budget)
    tr = RolloutTrace(c, trace, cap_steps=2000) if trace is not None else None
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    return c, tr


def _records(c):
    return c.snapshot().cpu().numpy()


def _everything(c):
    """Books, end state, health, the last step's solver report and the lap reports."""
    flags, unsolved = c.rollout_health()
    out = dict(c.books(), flags=flags, unsolved=unsolved, **c.rollout_state(), **{"r_" + k: v for k, v in c.step_results().items()})
    if getattr(c, "lap_report_cap", 0):
        out.update({"rep_" + k: v for k, v in c.lap_reports().items()})
    return out


def _same(a, b, what=""):
    assert sorted(a) == sorted(b), what
    for k in a:
        assert np.array_equal(a[k], b[k]), (what, k)


class _HostSwitch:
    """The host-driven equivalent of a schedule: after every hand-over, read lap_n and re-install the plain tables with
    set_of_instance = row_of_lap[b][min(lap_n[b], L - 1)] whenever some controller's entry changed."""
    def __init__(self, c, sched):
        self.c, self.sched, self.cur = c, sched, {}
        self.update()

    def update(self):
        lap_n = self.c.books()["lap_n"]
        for k, s in self.sched.items():
            idx = ls.host_switch_index(lap_n, s)
            if k not in self.cur or not np.array_equal(idx, self.cur[k]):
                getattr(self.c, INSTALL[k])(TABLES[k][0], idx)
                self.cur[k] = idx


def _lockstep(a, b, host, n=None, laps=None, every=True, cap=2400):
    """Step a (scheduled) and b (host switch) alike, `n` steps or until every controller of a has `laps` laps or has retired (laps
    None with n None), polled every 8 steps; with `every`, books and end states agree after every step.  Returns the steps."""
    for t in range(1, cap + 1):
        for c in (a, b):
            c.rollout_step(seed=SEED)
            c.rollout_commit_laps_dev()
        host.update()
        if every:
            _same(dict(a.books(), **a.rollout_state()), dict(b.books(), **b.rollout_state()), "step %d" % t)
        if n is not None:
            if t == n:
                return t
        elif t % 8 == 0:
            lap_min = a.rollout_stats()[0]
            if (lap_min == INT32_MAX) if laps is None else lap_min >= laps:
                return t
    pytest.fail("the closed loop did not get there in %d steps" % cap)


def _steps(c, n, mode=None):
    for _ in range(n):
        c.rollout_step(seed=SEED, mode=mode)
        c.rollout_commit_laps_dev()


def _until(c, laps, cap=2400):
    for n in range(8, cap + 1, 8):
        _steps(c, 8)
        if c.rollout_stats()[0] >= laps:
            return n
    pytest.fail("the closed loop did not get there in %d steps" % cap)


def _identity(k, L=3):
    return np.repeat(np.asarray(TABLES[k][1], np.int32)[:, None], L, axis=1)


@pytest.mark.parametrize("kind", ["vehicle", "noise", "measurement"])
def test_identity_schedule_is_the_closed_loop_without_one(kind):
    """PID lap, seeding, three LMPC laps, then 16 mode-0 and, after sysid, 16 mode-2 steps: a schedule whose every entry is the
    controller's own index equals no schedule (books, end states, health, step results, lap reports, snapshot records)."""
    _need_gpu()
    outs = []
    for sched in (None, {kind: _identity(kind)}):
        c, _ = _handle([kind], sched=sched)
        _until(c, 3)
        _steps(c, 16, mode=0)
        c.rollout_sysid()
        _steps(c, 16, mode=2)
        outs.append((_everything(c), _records(c)))
        c.close()
    assert outs[0][0]["lap_n"].min() >= 3
    _same(outs[0][0], outs[1][0], kind)
    assert np.array_equal(outs[0][1], outs[1][1]), kind


def _switching(kinds, L, seed):
    """Per-controller schedules with switches at entries 0, 1 and 2: entry 0 differs from the own index for a third of the batch."""
    rng = np.random.default_rng(seed)
    out = {}
    for k in kinds:
        nrows = len(TABLES[k][0])
        s = rng.integers(0, nrows, size=(B, L)).astype(np.int32)
        s[::3, 0] = (np.asarray(TABLES[k][1])[::3] + 1) % nrows
        out[k] = s
    return out


@pytest.mark.parametrize("kinds", [("vehicle",), ("noise",), ("measurement",), ("vehicle", "noise")])
def test_device_switch_equals_host_switch(kinds):
    """A scheduled batch against the same batch whose host re-installs the plain tables at every change of entry (same streams
    and seed, lock step): books and end states after every step, then health, lap reports, trace rows and records.  L = 3 and
    four LMPC laps driven, so the last entry holds for lap 4."""
    _need_gpu()
    sched = _switching(kinds, 3, 7 + len(kinds))
    traced = [0, 1, 2, 9]
    a, tra = _handle(kinds, sched=sched, trace=traced)
    b, trb = _handle(kinds, trace=traced)
    host = _HostSwitch(b, sched)
    _lockstep(a, b, host, laps=4)
    assert a.books()["lap_n"].min() >= 4
    assert len(host.cur) == len(kinds)
    _same(_everything(a), _everything(b), kinds)
    for j in range(len(traced)):
        ta, tb = tra.get(j), trb.get(j)
        assert all(np.array_equal(ta[k], tb[k]) for k in ta), traced[j]
    assert np.array_equal(_records(a), _records(b))
    for k in kinds:
        assert np.array_equal(a.lap_schedule_of(k), sched[k])
    a.close(); b.close()


def test_the_pid_lap_ignores_the_schedule():
    """Schedules of all three tables whose entries all differ from the own index, installed before the PID lap: the seeded stores
    equal those of a handle without schedules, byte for byte."""
    _need_gpu()
    kinds = ("vehicle", "noise", "measurement")
    other = {k: np.repeat(((np.asarray(TABLES[k][1]) + 1) % len(TABLES[k][0])).astype(np.int32)[:, None], 2, axis=1) for k in kinds}
    a, _ = _handle(kinds, sched=other)
    b, _ = _handle(kinds)
    assert np.array_equal(_records(a), _records(b))
    _steps(a, 1); _steps(b, 1)
    assert not np.array_equal(_records(a), _records(b)), "the first LMPC step reads entry 0"
    a.close(); b.close()


def test_a_retired_controller_stays_put_and_revives_at_its_entry():
    """Budget 2 against a vehicle + noise schedule of L = 4: once everybody has retired, 20 more steps change no byte of any
    record; the budget raised to 4 revives every controller at entry 2, and all of it equals the host-switch arm in lock step."""
    _need_gpu()
    kinds = ("vehicle", "noise")
    sched = _switching(kinds, 4, 3)
    a, _ = _handle(kinds, sched=sched, budget=2)
    b, _ = _handle(kinds, budget=2)
    host = _HostSwitch(b, sched)
    _lockstep(a, b, host, every=False)
    assert np.all(a.books()["lap_n"] == 2)
    rec = _records(a)
    _lockstep(a, b, host, n=20, every=False)
    assert np.array_equal(rec, _records(a)), "a retired controller moved"
    for c in (a, b):
        c.set_lap_budget(4)
    assert a.rollout_stats()[0] == 2
    _lockstep(a, b, host, every=False)
    assert np.all(a.books()["lap_n"] == 4)
    _same(_everything(a), _everything(b), "revived")
    assert np.array_equal(_records(a), _records(b))
    a.close(); b.close()


def test_snapshot_resumes_at_its_entry():
    """rollout_mc.run to LMPC lap 2, captured, restored into a fresh handle with the same tables and schedule and run to lap 5,
    equals a straight 5-lap run: books, health, lap reports and records; a schedule other than the captured one is refused."""
    _need_gpu()
    mc = _rollout_mc()
    Bp = 48
    veh = ([VehicleParams.from_friction(mu) for mu in (0.8, 0.65)], np.zeros(Bp, np.int32))
    sched = {"vehicle": np.tile([0, 0, 1, 1, 0], (Bp, 1))}
    sched["vehicle"][::2] = [1, 0, 0, 1, 1]
    kw = dict(batch=Bp, mode="independent", local=0, vehicle_sets=veh, lap_reports=8, lap_schedules=sched)
    cap2, cap5, bk_resumed, bk_straight, end = {}, {}, {}, {}, {}
    mc.run(laps=2, capture=cap2, **kw)
    assert np.array_equal(np.asarray(cap2["lap_schedules"]["vehicle"]), sched["vehicle"])
    with pytest.raises(ValueError, match="lap_schedules"):
        mc.run(laps=5, start=cap2, **dict(kw, lap_schedules={"vehicle": [0, 1]}))
    o_r = mc.run(laps=5, start=cap2, books=bk_resumed, capture=end, **kw)
    o_s = mc.run(laps=5, books=bk_straight, capture=cap5, **kw)
    assert o_r["resume_exact"]
    assert np.all(bk_straight["lap_n"] >= 5)
    for k in bk_straight:
        if k == "lap_reports":
            _same(bk_straight[k], bk_resumed[k], k)
        else:
            assert np.array_equal(bk_straight[k], bk_resumed[k]), k
    assert torch.equal(end["records"], cap5["records"])
    assert o_r["per_lap_row_rank0"] == o_s["per_lap_row_rank0"]
    rows = o_s["per_lap_row_rank0"]["vehicle"]
    assert sum(r["controllers"] for r in rows if r["lap"] == 1) == Bp


def test_refused_calls_leave_the_handle_as_it_was():
    _need_gpu()
    L = nat.lib()
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    one = np.zeros(B, np.int32)
    # no store (the lap books hold lap_n), then no rollout
    p = nat.make_params(par, numSS_Points, numSS_it, Qts)
    h = C.c_void_p()
    nat.check(L.lmpc_create(C.byref(p), B, 0, C.byref(h)))
    assert L.lmpc_rollout_set_lap_schedule(h, 0, 1, nat.ptr(one)) == LMPC_E_STATE
    L.lmpc_destroy(h)
    t0 = TrackParams.l_shaped()
    c = BatchedController(par, B, t0.seg_table, t0.TrackLength, trToUse=4, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=1280, ss_cap=7, model_cap=5)
    assert L.lmpc_rollout_set_lap_schedule(c._h, 0, 1, nat.ptr(one)) == LMPC_E_STATE
    c.close()
    kinds = ("vehicle", "noise")
    sched = _switching(kinds, 3, 11)
    a, _ = _handle(kinds, sched=sched)
    b, _ = _handle(kinds, sched=sched)
    _steps(a, 100); _steps(b, 100)
    rec = _records(a)
    s2 = np.ascontiguousarray(np.zeros((B, 2), np.int32))
    bad = np.ascontiguousarray(np.full((B, 2), 3, np.int32))            # three cars: row 3 does not exist
    neg = s2.copy(); neg[5, 1] = -1
    big = np.zeros((B, 1025), np.int32)
    refusals = [(LMPC_E_STATE, (KIND["measurement"], 2, nat.ptr(s2))),            # no measurement table
                (LMPC_E_INVALID, (3, 2, nat.ptr(s2))), (LMPC_E_INVALID, (-1, 2, nat.ptr(s2))),
                (LMPC_E_INVALID, (0, 1025, nat.ptr(big))), (LMPC_E_INVALID, (0, -1, nat.ptr(s2))),
                (LMPC_E_INVALID, (0, 0, nat.ptr(s2))), (LMPC_E_INVALID, (0, 2, None)),
                (LMPC_E_INVALID, (0, 2, nat.ptr(bad))), (LMPC_E_INVALID, (0, 2, nat.ptr(neg))),
                (LMPC_E_INVALID, (1, 2, nat.ptr(np.ascontiguousarray(np.full((B, 2), 2, np.int32)))))]
    for rc, args in refusals:
        assert L.lmpc_rollout_set_lap_schedule(a._h, *args) == rc, args
    # both install orders, past the Python checks: tables that do not cover the installed schedules
    vmax, nmax = int(sched["vehicle"].max()), int(sched["noise"].max())
    assert vmax >= 1 and nmax >= 1
    v1 = (nat.VehicleParams * 1)(nat.make_vehicle_sets(TABLES["vehicle"][0][:1], one, B)[0][0])
    assert L.lmpc_rollout_set_vehicles(a._h, v1, 1, nat.ptr(one)) == LMPC_E_INVALID
    assert L.lmpc_rollout_set_vehicles(a._h, None, 0, None) == LMPC_E_INVALID
    assert L.lmpc_rollout_set_noise(a._h, None, 0, None) == LMPC_E_INVALID
    with pytest.raises(ValueError):
        a.set_vehicles(TABLES["vehicle"][0][:1], one)
    # a measurement schedule, then removing the measurement table
    a.set_measurement_noise(*TABLES["measurement"]); b.set_measurement_noise(*TABLES["measurement"])
    ms = np.ascontiguousarray(np.ones((B, 1), np.int32))
    assert L.lmpc_rollout_set_lap_schedule(a._h, KIND["measurement"], 1, nat.ptr(ms)) == 0
    assert L.lmpc_rollout_set_measurement_noise(a._h, None, 0, None) == LMPC_E_INVALID
    assert L.lmpc_rollout_set_lap_schedule(a._h, KIND["measurement"], 0, None) == 0
    assert np.array_equal(rec, _records(a))
    assert np.array_equal(a.lap_schedule_of("vehicle"), sched["vehicle"])
    _steps(a, 60); _steps(b, 60)
    _same(_everything(a), _everything(b), "after the refusals")
    assert np.array_equal(_records(a), _records(b))
    a.close(); b.close()
