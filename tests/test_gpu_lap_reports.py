"""GPU tier: per-lap reports of the device closed loop (lmpc_rollout_enable_lap_reports).

Every report equals, bit for bit, the host restatement (tests/support/lap_reports.py) fed with the plant state, the step results
and the lane constants read at every step, through the device-book and the host-slot hand-over, in modes 1, 0 and 2 with tightened
lanes, a low-friction car and measurement noise; reports change nothing else; steps agree with lap_hist; a 20-lap run reports every
lap; retired controllers and imported laps file nothing; snapshots carry the reports and refuse a mismatched layout."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                # noqa: E402
from racinglmpc_b200 import _native as nat                        # noqa: E402
from racinglmpc_b200.reference_params import MeasurementParams, VehicleParams   # noqa: E402
import closed_loop as cl                                          # noqa: E402
import lap_reports as lr                                          # noqa: E402
from closed_loop import N, X0                                     # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
import rollout_mc                                                 # noqa: E402

LMPC_E_STATE = -4
MEAS = MeasurementParams((0.01, 0.01, 0.01, 0.005, 0.01, 0.01), (0.05, 0.05, 0.05, 0.025, 0.05, 0.05))


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _lanes(B, widths=(0.4, 0.25, 0.1)):
    """Parameter sets with the reference's lane (0.4) and tightened ones, and every controller's (Fx, bx)."""
    base = rp.lmpc_params(N)[5]
    sets = []
    for w in widths:
        q = copy.copy(base)
        q.bx = np.array([w, w])
        sets.append(q)
    idx = np.arange(B, dtype=np.int32) % len(widths)
    Fx = [np.asarray(sets[k].Fx, float).reshape(2, 6) for k in idx]
    bx = [np.asarray(sets[k].bx, float).reshape(2) for k in idx]
    return sets, idx, Fx, bx


def _setup(B, L, Tcl=1024):
    """A controller with tightened lanes, a low-friction car on every fourth controller and measurement noise on the odd ones,
    reports of capacity L enabled before the PID lap; returns (controller, book, Fx, bx)."""
    c = cl.controller(B)
    sets, idx, Fx, bx = _lanes(B)
    c.set_param_sets(sets, idx)
    c.set_vehicles([VehicleParams.reference(), VehicleParams.from_friction(0.5)], (np.arange(B) % 4 == 3).astype(np.int32))
    c.enable_rollout(Tcl=Tcl)
    c.set_measurement_noise([MeasurementParams.zero(), MEAS], (np.arange(B) % 2).astype(np.int32))
    c.enable_lap_reports(L)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    return c, lr.LapReportBook(B, L), Fx, bx


def _lookup_failed(c):
    return (c.rollout_health()[0] & 128) != 0


def _sim_bits(c, st, before, after, b):
    """The simulator's bits of the step just driven: 256 from the record length before it; 128 (a failed curvature lookup) where
    the health counter gained it, which shows its first occurrence only (_compare accounts for the later ones)."""
    return (256 if st["cl_len"][b] >= c.Tcl else 0) | (128 if after[b] and not before[b] else 0)


def _pid_lap(c, book, Fx, bx):
    for _ in range(1000):
        st, before = c.rollout_state(), _lookup_failed(c)
        c.rollout_pid_step(0.8, seed=4321)
        after = _lookup_failed(c)
        for b in range(c.B):
            book.step(b, st["x"][b], Fx[b], bx[b], _sim_bits(c, st, before, after, b))


def _drive(c, book, Fx, bx, laps, mode=None, host_slot=False, budget=None, cap=450):
    """Host-stepped closed loop until every live controller has driven `laps` more laps (at most cap * laps steps), feeding the
    restatement with the plant state, step results and simulator bits of every step and every hand-over."""
    start = None
    for _ in range(cap * laps):
        st, before = c.rollout_state(), _lookup_failed(c)
        lap_n = book.n.copy()                     # hand-overs since the seeding: lap_n of the device books
        if start is None:
            start = lap_n.copy()
        retired = (lap_n >= budget) if budget is not None else np.zeros(c.B, bool)
        if np.all((lap_n - start >= laps) | retired):
            return
        c.rollout_step(seed=1234, mode=mode)
        res = c.step_results()
        done, n = c.rollout_done()
        after = _lookup_failed(c)
        for b in range(c.B):
            if not retired[b]:
                sim = _sim_bits(c, st, before, after, b)
                book.step(b, st["x"][b], Fx[b], bx[b], int(res["flags"][b]) | sim, int(res["status"][b]), int(res["iters"][b]))
        if host_slot:
            if done.any():
                c.rollout_finish_laps(done, n)
            fin = done != 0
        else:
            c.rollout_commit_laps_dev()
            fin = (done != 0) & ~retired
        for b in np.nonzero(fin)[0]:
            book.file(b)


def _compare(c, got, want, what):
    """Reports against the restatement: every field bit for bit, flags too except bit 128 after its first occurrence, which the
    host sees only through the health counter: there a report may hold 128 where the restatement has none, and only on a
    controller whose health holds it."""
    gf, wf = got["flags"], want["flags"]
    assert np.array_equal(gf & ~128, wf & ~128), what
    assert ((wf & 128) <= (gf & 128)).all(), what
    assert not (gf[~_lookup_failed(c)] & 128).any(), what
    lr.assert_equal_tables(dict(got, flags=wf), want, what)


def test_reports_equal_the_restatement_with_device_books():
    """PID lap, device seeding, 3 LMPC laps, one LTV-MPC lap and one LTI-MPC lap through the device hand-over."""
    _need_gpu()
    B = 48
    c, book, Fx, bx = _setup(B, 8)
    try:
        _pid_lap(c, book, Fx, bx)
        c.rollout_seed_from_record_dev(copies=4)
        for b in range(B):
            book.restart(b)
        c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
        _drive(c, book, Fx, bx, 3, mode=1)
        _drive(c, book, Fx, bx, 1, mode=0)
        c.rollout_sysid()
        _drive(c, book, Fx, bx, 1, mode=2)
        got = c.lap_reports()
        _compare(c, got, book.table(), "device books")
        assert (got["n"] >= 1).all() and got["viol_steps"].sum() > 0 and got["ipm_iters"].sum() > 0, got["n"]
        bk = c.books()
        assert np.array_equal(got["n"], bk["lap_n"])
        clean = ((got["flags"] & 256) == 0) & (np.arange(8)[None, :] < got["n"][:, None])
        assert np.array_equal(got["steps"][clean], bk["lap_hist"][:, :8][clean])
    finally:
        c.close()


def test_reports_equal_the_restatement_with_host_slots():
    """PID lap, host seeding, 2 LMPC laps through the host-slot hand-over (rollout_finish_laps)."""
    _need_gpu()
    B = 24
    c, book, Fx, bx = _setup(B, 4)
    try:
        _pid_lap(c, book, Fx, bx)
        _, n = c.rollout_done()
        c.rollout_seed_from_record(n, copies=4)
        for b in range(B):
            book.restart(b)
        c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
        _drive(c, book, Fx, bx, 2, mode=1, host_slot=True)
        got = c.lap_reports()
        _compare(c, got, book.table(), "host slots")
        assert (got["n"] >= 1).all() and got["viol_steps"].sum() > 0
    finally:
        c.close()


def _reports_then(L):
    def hook(c):
        enable = c.enable_rollout

        def enable_then_report(Tcl=512):
            enable(Tcl)
            c.enable_lap_reports(L)
        c.enable_rollout = enable_then_report
    return hook


def test_reports_change_nothing_else():
    """Books, stored laps, end states and health of a run with reports equal those of the same run without, bit for bit."""
    _need_gpu()
    B = 64
    sets, idx, _, _ = _lanes(B)
    plain = cl.run(B, psets=(sets, idx, None))
    rep = cl.run(B, psets=(sets, idx, None), hook=_reports_then(4))
    assert plain[0] == rep[0]
    cl.same(plain[1:], rep[1:], np.ones(B, bool), "reports on")


def _loop(c, until_laps, seed=1234):
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))
    for k in range(300 * until_laps):
        c.rollout_step(seed=seed)
        c.rollout_commit_laps_dev()
        if k % 8 == 7 and c.rollout_stats()[0] >= until_laps:
            break


def test_capacity_overflow_keeps_counting():
    """20 laps with 8 rows: 8 stored, n = lap_n >= 20, the stored rows agree with lap_hist."""
    _need_gpu()
    B = 32
    c = cl.controller(B)
    try:
        c.enable_rollout(Tcl=1024)
        c.enable_lap_reports(8)
        _loop(c, 20)
        got, bk = c.lap_reports(), c.books()
        assert (got["n"] >= 20).all() and np.array_equal(got["n"], bk["lap_n"])
        clean = (got["flags"] & 256) == 0
        assert np.array_equal(got["steps"][clean], bk["lap_hist"][:, :8][clean])
        assert (got["steps"] > 0).all()
    finally:
        c.close()


def test_driver_reports_twenty_laps_and_keeps_lap_stats():
    """rollout_mc.run(laps=20, lap_reports=24) with parameter sets installed: every lap reported, its summaries equal those computed
    from the reports, and lap_stats_rank0 of laps < 16 equals a run without reports."""
    _need_gpu()
    B = 64
    sets, idx, _, _ = _lanes(B, (0.4, 0.3))
    got = {}
    out = rollout_mc.run(batch=B, laps=20, mode="independent", lap_reports=24, books=got, param_sets=(sets, idx, None))
    reps = got["lap_reports"]
    assert (reps["n"] >= 20).all() and len(out["lap_stats_rank0"]) == 20 and out["lap_reports"] == 24
    assert out["lap_reports_rank0"] == rollout_mc.lap_report_summary(reps, np.ones(B, bool), 20)
    for k, s in enumerate(out["per_set_rank0"]):
        assert s["reports"] == rollout_mc.lap_report_summary(reps, idx == k, 20)
    base = rollout_mc.run(batch=B, laps=16, mode="independent", param_sets=(sets, idx, None))
    assert "lap_reports_rank0" not in base
    clean = ((reps["flags"][:, :16] & 256) == 0).all()
    assert clean, "a lap found the record full"
    assert out["lap_stats_rank0"][:16] == base["lap_stats_rank0"]


def test_retired_controllers_and_imports_file_nothing():
    """A retired controller's reports equal its rows in a run without budgets; a pooled run files only driven laps."""
    _need_gpu()
    B = 32
    budget = np.where(np.arange(B) % 2 == 0, 1, 100).astype(np.int32)
    outs = []
    for bud in (budget, None):
        c = cl.controller(B)
        try:
            c.enable_rollout(Tcl=1024)
            c.enable_lap_reports(4)
            c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
            for _ in range(1000):
                c.rollout_pid_step(0.8, seed=4321)
            c.rollout_seed_from_record_dev(copies=4)
            if bud is not None:
                c.set_lap_budget(bud)
            c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
            for k in range(900):
                c.rollout_step(seed=1234)
                c.rollout_commit_laps_dev()
            outs.append(c.lap_reports())
        finally:
            c.close()
    a, b = outs
    ret = np.arange(B) % 2 == 0
    assert (a["n"][ret] == 1).all() and (b["n"] >= 3).all()
    for f in lr.FIELDS:
        assert np.array_equal(a[f][ret, :1], b[f][ret, :1]), f
        assert (a[f][ret, 1:] == 0).all(), f
        assert np.array_equal(a[f][~ret], b[f][~ret]), f
    got = {}
    out = rollout_mc.run(batch=64, laps=3, mode="pooled", lap_reports=4, books=got)
    reps = got["lap_reports"]
    assert out["laps_filed_rank0"] > 0
    assert np.array_equal(reps["n"], got["lap_n"])
    clean = ((reps["flags"][:, :3] & 256) == 0) & (np.arange(3)[None, :] < reps["n"][:, None])
    assert np.array_equal(reps["steps"][:, :3][clean], got["lap_hist"][:, :3][clean])


def test_snapshot_resume_and_refusals():
    _need_gpu()
    B = 32
    cap, b3 = {}, {}
    rollout_mc.run(batch=B, laps=3, mode="pooled", lap_reports=8, capture=cap, books=b3)
    assert cap["layout"]["lap_reports"] == 8
    resumed, straight = {}, {}
    rollout_mc.run(batch=B, laps=5, mode="pooled", lap_reports=8, start=cap, books=resumed)
    rollout_mc.run(batch=B, laps=5, mode="pooled", lap_reports=8, books=straight)
    lr.assert_equal_tables(resumed["lap_reports"], straight["lap_reports"], "resumed")
    assert (straight["lap_reports"]["n"] >= 5).all()
    with pytest.raises(ValueError, match="lap_reports"):
        rollout_mc.run(batch=B, laps=5, mode="pooled", start=cap)
    # a handle with another capacity, or without reports, refuses the records and keeps its own
    recs = cap["records"]
    for L in (0, 4):
        c = cl.controller(B)
        try:
            c.enable_rollout(Tcl=rollout_mc.TCL)
            if L:
                c.enable_lap_reports(L)
            _loop(c, 1)
            with pytest.raises(ValueError):
                c.restore(recs)
            mine = c.snapshot().cpu().numpy()
            if recs.shape[1] == mine.shape[1]:
                continue
            # the library's own check names the reports too (the Python checks bypassed: same record size needed, so only
            # the header of a record of this handle's size with foreign report sections is tried)
            fake = torch.from_numpy(mine.copy()).to(recs.device)
            hdr = bytearray(fake[0, :nat.C.sizeof(nat.SnapshotHeader)].cpu().numpy().tobytes())
            h = nat.SnapshotHeader.from_buffer_copy(bytes(hdr))
            k = nat.SNAPSHOT_SECTIONS_NAMES.index("lap_reports")
            h.sect_bytes[k] = 32 * 8
            fake[:, :nat.C.sizeof(nat.SnapshotHeader)] = torch.frombuffer(bytearray(bytes(h)), dtype=torch.uint8).to(recs.device)
            dst = np.arange(B, dtype=np.int32)
            torch.cuda.synchronize()
            rc = nat.lib().lmpc_snapshot_unpack_dev(c._h, nat.ptr(fake), B, B, nat.ptr(dst), None)
            assert rc != 0 and b"lap report layout" in nat.lib().lmpc_last_error()
            assert np.array_equal(c.snapshot().cpu().numpy(), mine), "a refused restore changed the handle"
        finally:
            c.close()


def test_handle_without_reports_keeps_its_records():
    """Records of a handle without reports list no report section, and turning reports on and off again leaves records as they were;
    enabling while a record holds rows is refused and changes nothing."""
    _need_gpu()
    B = 16
    recs = []
    for toggle in (False, True):
        c = cl.controller(B)
        try:
            c.enable_rollout(Tcl=1024)
            if toggle:
                c.enable_lap_reports(6)
                c.enable_lap_reports(0)
            c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
            for _ in range(20):
                c.rollout_pid_step(0.8, seed=4321)
            rc = nat.lib().lmpc_rollout_enable_lap_reports(c._h, 4)
            assert rc == LMPC_E_STATE and b"holds rows" in nat.lib().lmpc_last_error()
            c.rollout_seed_from_record_dev(copies=4)
            recs.append(c.snapshot().cpu().numpy())
            head = nat.decode_snapshot_header(recs[-1][0])
            assert "lap_reports" not in head["sections"] and "lap_report_run" not in head["sections"]
            assert set(head["sections"]) <= set(nat.SNAPSHOT_SECTIONS_NAMES[:37])
        finally:
            c.close()
    assert np.array_equal(recs[0], recs[1])
