"""CPU tier: per-lap reports of the device closed loop (lmpc_rollout_enable_lap_reports).

The ABI (symbols, prototypes, the 32-byte row), every refusal of BatchedController.enable_lap_reports and of
rollout_mc.run(lap_reports=...) before any device work, the host restatement of the accumulation rule (tests/support/lap_reports.py)
on synthetic step sequences, the driver's per-lap summary against hand-built tables, and the snapshot header's report sections."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat
from racinglmpc_b200.controller import BatchedController
import lap_reports as lr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
import rollout_mc  # noqa: E402
from racinglmpc_b200 import sharding  # noqa: E402

LANE = np.array([[0., 0., 0., 0., 0., 1.], [0., 0., 0., 0., 0., -1.]])


def _header():
    return open(os.path.join(ROOT, "include", "lmpc_b200.h")).read()


def test_abi_symbols_prototypes_and_row_size():
    names = nat.exported_symbols()
    for s in ("lmpc_rollout_enable_lap_reports", "lmpc_rollout_get_lap_reports", "lmpc_sizeof_lap_report"):
        assert s in names
        assert hasattr(nat.lib(), s), s
    txt = re.sub(r"\s+", " ", _header())
    assert "int lmpc_rollout_enable_lap_reports(lmpc_handle* h, int max_laps);" in txt
    assert "int lmpc_rollout_get_lap_reports(lmpc_handle* h, lmpc_lap_report* rows, int* n);" in txt
    assert C.sizeof(nat.LapReport) == 32
    assert nat.lib().lmpc_sizeof_lap_report() == 32
    assert nat.LAP_REPORT_DTYPE.itemsize == 32
    assert [f for f, _ in nat.LapReport._fields_] == list(lr.FIELDS)
    assert nat.LapReport.viol_max.offset == 24


@pytest.mark.parametrize("bad", [-1, 1025, 2.0, True, "8", None])
def test_enable_refusals_before_native_call(bad):
    c = object.__new__(BatchedController)          # no handle: a refusal must come before any native call
    c._lib = None
    with pytest.raises(ValueError):
        c.enable_lap_reports(bad)
    with pytest.raises(ValueError):
        nat.check_lap_reports(bad)


def test_enable_needs_rollout_and_reading_needs_reports():
    c = object.__new__(BatchedController)
    c._lib = None
    with pytest.raises(ValueError, match="enable_rollout"):
        c.enable_lap_reports(4)
    with pytest.raises(ValueError, match="not enabled"):
        c.lap_reports()
    assert nat.check_lap_reports(0) == 0 and nat.check_lap_reports(1024) == 1024 and nat.check_lap_reports(np.int32(3)) == 3


@pytest.mark.parametrize("kw", [dict(laps=17), dict(laps=20, lap_reports=None), dict(laps=3, lap_reports=2),
                                dict(laps=3, lap_reports=0), dict(laps=3, lap_reports=1025), dict(laps=3, lap_reports=3.0)])
def test_run_refusals_before_device_work(kw, monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(rollout_mc.torch.cuda, "set_device", no_device)
    monkeypatch.setattr(rollout_mc, "BatchedController", no_device)
    with pytest.raises(ValueError):
        rollout_mc.run(batch=8, **kw)


def _start(L):
    s = {k: 0 for k in sharding.ExchangeSchedule.FIELDS}
    s.update(records=np.zeros((8, 16), np.uint8), clock=0, batch=8, laps=3, mode="pooled", readiness="batch", poll=8, warm=False,
             pool_groups=1, layout=dict(rollout_mc.layout(lap_reports=L), bytes=16), tables={})
    return s


@pytest.mark.parametrize("captured, now", [(8, None), (0, 8), (8, 10)])
def test_run_start_refuses_another_report_capacity(captured, now, monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(rollout_mc.torch.cuda, "set_device", no_device)
    monkeypatch.setattr(rollout_mc, "BatchedController", no_device)
    with pytest.raises(ValueError, match="lap_reports"):
        rollout_mc.run(batch=8, laps=5, start=_start(captured), lap_reports=now)


def test_layout_has_the_report_key_only_with_reports():
    assert "lap_reports" not in rollout_mc.layout()
    assert rollout_mc.layout(lap_reports=24)["lap_reports"] == 24
    assert rollout_mc.check_lap_reports(None, 16) == 0 and rollout_mc.check_lap_reports(20, 20) == 20


# ---- the restatement on synthetic step sequences ------------------------------------------------------------------------------
def _x(ey, s=1.0):
    return np.array([1.0, 0.0, 0.0, 0.0, s, ey])


def test_restatement_accumulates_and_files_at_record_restarts():
    bk = lr.LapReportBook(2, 4)
    bk.step(0, _x(0.1), LANE, [0.4, 0.4], 0, status=1, iters=7)
    bk.step(0, _x(0.5), LANE, [0.4, 0.4], 2, status=0, iters=40)       # violates row 0 by 0.1
    bk.step(0, _x(-0.2), LANE, [0.4, 0.4], 0, status=1, iters=9)
    bk.file(0)
    bk.step(0, _x(0.0), LANE, [0.4, 0.4], 0, status=1, iters=5)         # the next lap's running row
    t = bk.table()
    assert t["n"].tolist() == [1, 0]
    assert (t["steps"][0, 0], t["flags"][0, 0], t["unsolved"][0, 0], t["viol_steps"][0, 0]) == (3, 2, 1, 1)
    assert (t["ipm_iters"][0, 0], t["ipm_iters_max"][0, 0]) == (56, 40)
    assert t["viol_max"][0, 0] == (0.5 - 0.4)
    assert bk.run[0]["steps"] == 1 and bk.run[0]["viol_max"] == -0.4
    assert t["steps"][1].tolist() == [0] * 4 and t["viol_max"][0, 1] == 0.0
    bk.file(1)                                                           # a lap without steps: viol_max stays -inf
    assert bk.table()["viol_max"][1, 0] == -np.inf


def test_restatement_full_record_pid_steps_and_seeding():
    bk = lr.LapReportBook(1, 3)
    for _ in range(3):
        bk.step(0, _x(0.0), LANE, [2.0, 2.0], 0)                         # PID: no QP status, no iterations
    bk.step(0, _x(0.0), LANE, [2.0, 2.0], 256)                           # a step that found the record full still counts
    assert bk.run[0] == dict(steps=4, flags=256, unsolved=0, viol_steps=0, ipm_iters=0, ipm_iters_max=0, viol_max=-2.0)
    bk.file(0)
    bk.restart(0)                                                        # the seeding starts the table afresh
    assert bk.table()["n"].tolist() == [0] and bk.run[0]["steps"] == 0


def test_restatement_retirement_and_capacity_overflow():
    bk = lr.LapReportBook(2, 2)
    for lap in range(5):
        for k in range(lap + 1):
            bk.step(0, _x(0.0), LANE, [2.0, 2.0], 0, status=1, iters=1)
        bk.file(0)
        if lap < 2:                                                      # controller 1 retires after two laps: nothing more is fed
            bk.step(1, _x(0.0), LANE, [2.0, 2.0], 0, status=1, iters=1)
            bk.file(1)
    t = bk.table()
    assert t["n"].tolist() == [5, 2]
    assert t["steps"][0].tolist() == [1, 2] and t["steps"][1].tolist() == [1, 1]


def test_restatement_multi_row_fx_and_order_of_summation():
    Fx = np.array([[0.3, 0.1, 0.0, 0.2, 0.0, 1.0], [0.0, 0.0, 0.0, -1.0, 0.0, -1.0]])
    x = np.array([0.1, 0.2, 0.0, 0.3, 5.0, 0.7])
    d = lr.lane_margins(Fx, [0.9, 0.5], x)
    s0 = 0.3 * 0.1
    for a, b in ((0.1, 0.2), (0.0, 0.0), (0.2, 0.3), (0.0, 5.0), (1.0, 0.7)):
        s0 = s0 + a * b
    s1 = 0.0 * 0.1
    for a, b in ((0.0, 0.2), (0.0, 0.0), (-1.0, 0.3), (0.0, 5.0), (-1.0, 0.7)):
        s1 = s1 + a * b
    assert d == [s0 - 0.9, s1 - 0.5]
    bk = lr.LapReportBook(1, 1)
    bk.step(0, x, Fx, [0.9, 0.5], 0, status=1, iters=3)
    bk.file(0)
    assert bk.table()["viol_steps"][0, 0] == (1 if max(d) > 0 else 0)
    assert bk.table()["viol_max"][0, 0] == max(d)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_restatement_non_finite_state_is_a_violation(bad):
    bk = lr.LapReportBook(1, 1)
    bk.step(0, _x(0.0), LANE, [2.0, 2.0], 0, status=1, iters=3)
    x = _x(0.0)
    x[2] = bad
    bk.step(0, x, LANE, [2.0, 2.0], 0, status=2, iters=40)
    bk.step(0, _x(0.0), LANE, [2.0, 2.0], 0, status=1, iters=3)       # a later finite step does not lower +inf
    bk.file(0)
    t = bk.table()
    assert t["viol_steps"][0, 0] == 1 and t["viol_max"][0, 0] == np.inf and t["unsolved"][0, 0] == 1


# ---- the driver's summary -----------------------------------------------------------------------------------------------------
def test_summary_against_hand_built_reports():
    B, L = 4, 3
    z = lambda dt=np.int32: np.zeros((B, L), dt)
    reps = {"n": np.array([3, 2, 1, 0], np.int32), "steps": z(), "flags": z(), "unsolved": z(), "viol_steps": z(), "ipm_iters": z(),
            "ipm_iters_max": z(), "viol_max": z(np.float64)}
    reps["steps"][:3, 0] = [200, 210, 190]
    reps["steps"][:2, 1] = [180, 170]
    reps["steps"][0, 2] = 160
    reps["viol_steps"][1, 0] = 4
    reps["viol_max"][:3, 0] = [-0.1, 0.05, -0.2]
    reps["viol_max"][:2, 1] = [-0.3, -0.25]
    reps["viol_max"][0, 2] = np.inf
    reps["unsolved"][2, 0] = 3
    reps["ipm_iters"][:3, 0] = [2000, 2100, 1900]
    out = rollout_mc.lap_report_summary(reps, np.ones(B, bool), 3)
    assert out[0] == {"lap": 1, "controllers": 3, "steps_mean": 200.0, "steps_min": 190, "steps_max": 210, "violating": 1,
                      "viol_steps_mean": 4 / 3, "viol_max_max": 0.05, "viol_max_mean": (-0.1 + 0.05 - 0.2) / 3, "unsolved": 3,
                      "ipm_iters_per_step": 6000 / 600}
    assert out[1]["controllers"] == 2 and out[1]["steps_mean"] == 175.0 and out[1]["violating"] == 0
    assert out[2]["viol_max_max"] == np.inf and out[2]["controllers"] == 1
    sub = rollout_mc.lap_report_summary(reps, np.array([False, True, False, True]), 3)
    assert sub[0]["controllers"] == 1 and sub[0]["violating"] == 1 and sub[1]["steps_max"] == 170 and sub[2]["controllers"] == 0
    st = rollout_mc._set_stats({}, np.zeros(B, np.int32), np.zeros(B, np.int32), np.ones(B, bool), 3, reps)
    assert [l["mean"] for l in st["laps"]] == [200.0, 175.0, 160.0] and st["reports"] == out


# ---- snapshot header ----------------------------------------------------------------------------------------------------------
def _raw_header(L):
    h = nat.SnapshotHeader()
    h.magic, h.version, h.nsect = nat.SNAPSHOT_MAGIC, nat.SNAPSHOT_VERSION, nat.SNAPSHOT_SECTIONS
    names = nat.SNAPSHOT_SECTIONS_NAMES
    off = 1024
    for k in range(names.index("lap_reports")):
        h.sect_off[k], h.sect_bytes[k] = off, 16
        off += 16
    if L:
        k = names.index("lap_reports")
        h.sect_off[k], h.sect_bytes[k] = off, 32 * L
        h.sect_off[k + 1], h.sect_bytes[k + 1] = off + 32 * L, 48
        off += 32 * L + 48
    h.bytes = off
    return bytes(h)


def test_header_lists_report_sections_and_names_a_mismatch():
    assert nat.SNAPSHOT_SECTIONS_NAMES[-2:] == ("lap_reports", "lap_report_run") and len(nat.SNAPSHOT_SECTIONS_NAMES) <= 40
    d = nat.decode_snapshot_header(_raw_header(24))
    assert d["sections"]["lap_reports"][1] == 24 * 32 and d["sections"]["lap_report_run"][1] == 48
    assert nat.snapshot_lap_reports(d) == 24
    d0 = nat.decode_snapshot_header(_raw_header(0))
    assert "lap_reports" not in d0["sections"] and nat.snapshot_lap_reports(d0) == 0
    mine = {f: int(d[f]) for f in nat.SNAPSHOT_LAYOUT}
    assert nat.snapshot_layout_mismatch(d, dict(mine, bytes=d["bytes"], lap_reports=24)) is None
    for have, rec in ((dict(mine, bytes=d0["bytes"]), d), (dict(mine, bytes=d["bytes"], lap_reports=24), d0),
                      (dict(mine, bytes=d["bytes"], lap_reports=8), d)):
        msg = nat.snapshot_layout_mismatch(rec, have)
        assert msg is not None and "lap_reports" in msg
