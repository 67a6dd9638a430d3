"""GPU tier: lap budgets of the device-resident closed loop (lmpc_rollout_set_lap_budget).

No budget, and a budget that is never reached, are the closed loop without the call.  A controller that reached its budget is
frozen: further steps change no byte of its snapshot record, no health counter and no trace row, in every mode of the step and
with the uniform, the per-controller-parameter and the warm-started QP kernel, while the live controllers beside it equal those of
a handle without budgets.  Up to its retirement a controller drives what it drives without a budget; a batch of mixed budgets is
one handle per budget; raising the budget revives a controller where it stopped; the progress numbers leave retired controllers
out; a uniform budget equal to `laps` leaves the pooled exchange as it is; refused calls leave the handle as it was."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp, sharding     # noqa: E402
from racinglmpc_b200 import _native as nat                       # noqa: E402
from racinglmpc_b200.controller import BatchedController         # noqa: E402
from racinglmpc_b200.export import RolloutTrace                  # noqa: E402
from racinglmpc_b200.reference_params import TrackParams, NoiseParams      # noqa: E402
from closed_loop import N, X0                                    # noqa: E402
import lap_budget as lb                                          # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LMPC_E_INVALID, LMPC_E_STATE = -1, -4
INT32_MAX = 2 ** 31 - 1
THREE = [TrackParams.l_shaped(), TrackParams.goggle(), TrackParams.oval()]
B = 24
TIDX = (np.arange(B) % 3).astype(np.int32)
SEED = 1234


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


def _seeded(batch=B, tracks=True, warm=False, psets=False, quiet=False, trace=None):
    """A controller per circuit of THREE (track = b mod 3), PID lap and seeding done: ready for LMPC steps.  psets: two parameter
    sets interleaved (the per-controller-parameter QP kernel); quiet: no simulator noise; trace: controllers to trace."""
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    t0 = TrackParams.l_shaped()
    c = BatchedController(par, batch, t0.seg_table, t0.TrackLength, trToUse=4, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=1280, ss_cap=7, model_cap=5, warm_start=warm)
    if tracks:
        c.set_tracks(THREE, (np.arange(batch) % 3).astype(np.int32))
    if psets:
        other = rp.lmpc_params(N)[5]
        other.dR = 1.5 * np.asarray(other.dR)
        c.set_param_sets([par, other], (np.arange(batch) // 3) % 2)
    if quiet:
        c.set_noise([NoiseParams.scaled(0, 1)], np.zeros(batch, np.int32))      # the PID lap keeps its noise: it excites the model
    c.enable_rollout(Tcl=1024)
    tr = RolloutTrace(c, trace, cap_steps=1400) if trace is not None else None
    c.rollout_set_state(np.tile(X0, (batch, 1)), np.tile(X0, (batch, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (batch, 1)), np.tile(X0, (batch, 1)))
    return (c, tr) if trace is not None else c


def _steps(c, n, mode=None):
    for _ in range(n):
        c.rollout_step(seed=SEED, mode=mode)
        c.rollout_commit_laps_dev()


def _until(c, laps=None, cap=1600):
    """Step until every controller has retired (laps None) or has driven `laps` laps, polled every 8 steps.  Returns the steps."""
    for n in range(8, cap + 1, 8):
        _steps(c, 8)
        lap_min = c.rollout_stats()[0]
        if lap_min == INT32_MAX if laps is None else lap_min >= laps:
            return n
    pytest.fail("the closed loop did not get there in %d steps (lap_min %d)" % (cap, lap_min))


def _records(c):
    return c.snapshot().cpu().numpy()


def _everything(c):
    """What a run leaves behind besides the records: books, end state, health and the last step's solver report."""
    flags, unsolved = c.rollout_health()
    return dict(c.books(), flags=flags, unsolved=unsolved, **c.rollout_state(), **{"r_" + k: v for k, v in c.step_results().items()})


def _same(a, b, sel=slice(None), what=""):
    for k in a:
        assert np.array_equal(a[k][sel], b[k][sel]), (what, k)


def test_no_budget_and_a_budget_never_reached_are_the_closed_loop_without_the_call():
    """PID lap, seeding and 160 LMPC steps (the oval controllers hand laps over) on three handles: no call, a budget of 16
    installed before the PID lap, and a budget of 1 installed, then removed again after the seeding."""
    _need_gpu()
    outs = []
    for arm in ("none", "never", "reverted"):
        numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
        t0 = TrackParams.l_shaped()
        c = BatchedController(par, B, t0.seg_table, t0.TrackLength, trToUse=4, numSS_Points=numSS_Points, numSS_it=numSS_it,
                              QterminalSlack=Qts, Tmax=1280, ss_cap=7, model_cap=5)
        c.set_tracks(THREE, TIDX)
        c.enable_rollout(Tcl=1024)
        if arm == "never":
            c.set_lap_budget(16)
        c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
        for _ in range(1000):
            c.rollout_pid_step(0.8, seed=4321)
        c.rollout_seed_from_record_dev(copies=4)
        c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
        if arm == "reverted":
            c.set_lap_budget(1)
            c.set_lap_budget(None)
        _steps(c, 160)
        outs.append((_everything(c), _records(c), c.rollout_stats()))
        c.close()
    assert outs[0][0]["lap_n"].max() >= 1 and outs[0][0]["lap_n"].min() == 0, "the run should be caught with laps under way"
    for name, o in zip(("never", "reverted"), outs[1:]):
        _same(outs[0][0], o[0], what=name)
        assert np.array_equal(outs[0][1], o[1]), name
        assert outs[0][2] == o[2], name


@pytest.mark.parametrize("mode,psets,warm", [(1, False, False), (0, False, False), (2, False, False), (1, True, False),
                                             (0, True, False), (1, False, True)])
def test_retired_controllers_freeze_and_their_neighbours_do_not_notice(mode, psets, warm):
    """Two handles driven alike for 160 steps (every controller has a lap or not: the oval ones do).  Then handle A retires every
    controller that has a lap (budget = 1) and 40 steps follow on both in `mode` (0: the kernel without a safe set, 2: the LTI
    model) -- with two parameter sets, and with warm starts (a retired warp must leave its warm record alone).  The retired
    controllers of A keep their records byte for byte, their health and their trace; the live ones equal handle B's."""
    _need_gpu()
    traced = [0, 1, 2, 5]
    pairs = [_seeded(psets=psets, warm=warm, trace=traced) for _ in range(2)]
    before = None
    for i, (c, tr) in enumerate(pairs):
        _steps(c, 160)
        if mode == 2:
            c.rollout_sysid()
        if i == 0:
            lap_n = c.books()["lap_n"]
            gone = lap_n >= 1
            assert gone.any() and not gone.all(), lap_n
            before = (_records(c), c.rollout_health(), [tr.get(j) for j in range(len(traced))])
            c.set_lap_budget(np.where(gone, 1, 16))
            assert c.rollout_stats()[0] == 0 and c.rollout_stats()[1] == lap_n.max()
        _steps(c, 40, mode=mode)
    (a, tra), (b, trb) = pairs
    ra, rb = _records(a), _records(b)
    assert np.array_equal(ra[gone], before[0][gone]), "a retired controller's record changed"
    assert np.array_equal(ra[~gone], rb[~gone]), "a live controller noticed its retired neighbours"
    assert not np.array_equal(rb[gone], before[0][gone]), "the controllers without a budget should have driven on"
    for h0, h1 in zip(before[1], a.rollout_health()):
        assert np.array_equal(h0[gone], h1[gone])
    for j, inst in enumerate(traced):
        t0, t1, t2 = before[2][j], tra.get(j), trb.get(j)
        if gone[inst]:
            assert all(np.array_equal(t0[k], t1[k]) for k in t0), inst
        else:
            keys = [k for k in t1 if mode == 1 or k != "SS_sel"]          # a step without a safe set traces no selected points
            assert len(t1["lap"]) == len(t0["lap"]) + 40 and all(np.array_equal(t1[k], t2[k]) for k in keys), inst
    # the progress numbers leave the retired controllers out, and equal the host restatement
    st = a.rollout_state()
    want = lb.group_stats(a.books()["lap_n"], st["cl_len"], a.rollout_health()[0], np.zeros(B, int), 1, np.where(gone, 1, 16))
    assert list(a.rollout_stats()) == want[0].tolist()
    a.set_pool_groups(TIDX, 3)
    want = lb.group_stats(a.books()["lap_n"], st["cl_len"], a.rollout_health()[0], TIDX, 3, np.where(gone, 1, 16))
    assert np.array_equal(a.rollout_group_stats(), want)
    a.close(); b.close()


def test_retirement_freezes_everything_and_reports_the_empty_row():
    """Budget 2 on three circuits: once every controller has retired, twenty more steps and hand-overs change no byte of any
    record, no health counter and no trace row, and the progress row is the empty-group row with lap_max = 2."""
    _need_gpu()
    c, tr = _seeded(trace=[0, 1, 2])
    c.set_lap_budget(2)
    n = _until(c)
    bk = c.books()
    assert np.all(bk["lap_n"] == 2) and np.all(c.rollout_state()["cl_len"] == 0) and np.all(c.rollout_state()["done"] == 0)
    rec, health, rows = _records(c), c.rollout_health(), [tr.get(j) for j in range(3)]
    clock = c.rollout_clock
    _steps(c, 20)
    assert c.rollout_clock == clock + 20, "the simulator clock counts for the whole handle"
    assert np.array_equal(rec, _records(c))
    assert all(np.array_equal(p, q) for p, q in zip(health, c.rollout_health()))
    for j in range(3):
        now = tr.get(j)
        assert all(np.array_equal(rows[j][k], now[k]) for k in now)
        assert len(now["lap"]) == int(bk["lap_hist"][j, :2].sum()) and len(now["lap"]) < n
    stats = c.rollout_stats()
    assert stats[0] == INT32_MAX and stats[1] == 2 and stats[2] == INT32_MAX
    assert sharding.ready_groups([stats], 1, 2, 40)[0] and stats[0] >= 2
    c.close()


def test_up_to_its_retirement_a_controller_drives_what_it_drives_without_a_budget():
    """Three circuits, budget 3 against no budget, same seed, both traced: the first three laps are as long, and every traced
    controller's rows up to its retirement are the first rows of its trace without a budget, bit for bit."""
    _need_gpu()
    traced = [0, 1, 2, 10]
    a, tra = _seeded(trace=traced)
    b, trb = _seeded(trace=traced)
    a.set_lap_budget(3)
    na, nb = _until(a), _until(b, laps=3)
    ha, hb = a.books(), b.books()
    assert np.array_equal(ha["lap_hist"][:, :3], hb["lap_hist"][:, :3])
    assert np.all(ha["lap_n"] == 3) and hb["lap_n"].max() > 3, "without a budget the oval controllers drive surplus laps"
    for j, inst in enumerate(traced):
        ta, tb = tra.get(j), trb.get(j)
        rows = len(ta["lap"])
        assert rows == int(ha["lap_hist"][inst, :3].sum()) and len(tb["lap"]) == min(nb, 1400)
        assert all(np.array_equal(ta[k], tb[k][:rows]) for k in ta), inst
    a.close(); b.close()


@pytest.mark.parametrize("psets,warm", [(False, False), (True, False), (False, True)])
def test_a_batch_of_mixed_budgets_is_one_handle_per_budget(psets, warm):
    """Budgets 2 and 3 interleaved against a uniform-2 and a uniform-3 handle (same seed and streams), run until everyone has
    retired: every controller's final record equals that of its uniform handle, byte for byte -- also with two parameter sets
    and with warm starts."""
    _need_gpu()
    budget = 2 + (np.arange(B) // 3 + np.arange(B)) % 2
    recs = {}
    for name, bud in (("mixed", budget), (2, 2), (3, 3)):
        c = _seeded(psets=psets, warm=warm)
        c.set_lap_budget(bud)
        _until(c)
        assert np.array_equal(c.books()["lap_n"], np.broadcast_to(bud, (B,)))
        recs[name] = _records(c)
        c.close()
    for k in (2, 3):
        assert (budget == k).any() and np.array_equal(recs["mixed"][budget == k], recs[k][budget == k]), k
    assert not np.array_equal(recs[2], recs[3])


def test_raising_the_budget_revives_a_controller_where_it_stopped():
    """Without simulator noise the clock does not matter: budget 2 until everyone has retired, then budget 4 and on, equals a
    straight budget-4 run, records byte for byte."""
    _need_gpu()
    a, b = _seeded(quiet=True), _seeded(quiet=True)
    a.set_lap_budget(2)
    _until(a)
    a.set_lap_budget(4)
    assert a.rollout_stats()[0] == 2, "revived"
    _until(a)
    b.set_lap_budget(4)
    _until(b)
    assert np.all(a.books()["lap_n"] == 4) and np.array_equal(_records(a), _records(b))
    a.close(); b.close()


def test_resume_through_the_driver_with_a_raised_budget():
    """A budget-3 run captured and resumed with budget 5 finishes five laps per controller, and its first three laps are the
    captured ones.  Equality with a straight budget-5 run is not claimed: the clock counts for the whole handle, so a revived
    controller meets later noise draws than it would have met driving on."""
    _need_gpu()
    mc = _rollout_mc()
    cap, bk3, bk5 = {}, {}, {}
    o3 = mc.run(batch=48, laps=3, mode="independent", local=0, capture=cap, books=bk3, lap_budget=3)
    assert cap["lap_budget"] == [3] * 48 and np.all(bk3["lap_n"] == 3)
    assert o3["driven_controller_steps_rank0"] == int(bk3["lap_hist"][:, :3].sum()) < 48 * o3["closed_loop_steps"]
    with pytest.raises(ValueError, match="lap_budget is below"):
        mc.run(batch=48, laps=5, mode="independent", local=0, start=cap, lap_budget=2)
    o5 = mc.run(batch=48, laps=5, mode="independent", local=0, start=cap, books=bk5, lap_budget=5)
    assert np.all(bk5["lap_n"] == 5) and np.array_equal(bk5["lap_hist"][:, :3], bk3["lap_hist"][:, :3])
    assert o5["driven_controller_steps_rank0"] == int(bk5["lap_hist"][:, 3:5].sum())


def test_pooled_mode_with_a_uniform_budget_exchanges_as_without_one():
    """lap_budget = laps: the exchanges happen at the same steps and the laps are as long as without a budget, (a) on one circuit
    under batch readiness and (b) on three circuits grouped per circuit under group readiness; nobody had retired before its
    group's last exchange."""
    _need_gpu()
    mc = _rollout_mc()
    Bp, laps = 48, 3
    tidx = (np.arange(Bp) % 3).astype(np.int32)
    for kw in (dict(readiness="batch"), dict(readiness="group", track_sets=(THREE, tidx), pool_groups=(tidx, 3))):
        b0, b1 = {}, {}
        o0 = mc.run(batch=Bp, laps=laps, mode="pooled", local=0, books=b0, **kw)
        o1 = mc.run(batch=Bp, laps=laps, mode="pooled", local=0, books=b1, lap_budget=laps, **kw)
        assert o1["closed_loop_steps"] == o0["closed_loop_steps"], kw
        assert o1["exchanges"] == o0["exchanges"] >= laps - 1 and o1["laps_filed_rank0"] == o0["laps_filed_rank0"], kw
        if "pool_groups" in kw:
            assert o1["exchange_steps_per_group_rank0"] == o0["exchange_steps_per_group_rank0"]
        assert np.array_equal(b1["lap_hist"][:, :laps], b0["lap_hist"][:, :laps]), kw["readiness"]
        assert np.all(b1["lap_n"] == laps) and not any(o1["retired_before_last_exchange_rank0"])
        assert "retired_before_last_exchange_rank0" not in o0 and "driven_steps_per_s" not in o0
        assert o1["driven_controller_steps_rank0"] == int(b1["lap_hist"][:, :laps].sum())


def test_pooled_mode_with_mixed_budgets_is_not_held_back_by_the_retired():
    """Budgets 2 and 4 in one pool: rounds 2 and 3 still happen after the budget-2 controllers retired (the progress numbers
    leave them out) and the budget-4 controllers finish four laps."""
    _need_gpu()
    mc = _rollout_mc()
    Bp = 48
    budget = np.where(np.arange(Bp) % 2 == 0, 2, 4)
    bk = {}
    o = mc.run(batch=Bp, laps=4, mode="pooled", local=0, books=bk, lap_budget=budget)
    assert np.array_equal(bk["lap_n"], budget)
    assert o["exchanges"] >= 3 and o["retired_before_last_exchange_rank0"] == [True]
    assert o["lap_budget"] == "per controller, 2 .. 4"


def test_refused_calls_leave_the_handle_as_it_was():
    _need_gpu()
    L = nat.lib()
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    t0 = TrackParams.l_shaped()
    c = BatchedController(par, B, t0.seg_table, t0.TrackLength, trToUse=4, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=1280, ss_cap=7, model_cap=5)
    good = np.full(B, 2, np.int32)
    assert L.lmpc_rollout_set_lap_budget(c._h, nat.ptr(good)) == LMPC_E_STATE          # before lmpc_rollout_create
    with pytest.raises(nat.NativeError):
        c.set_lap_budget(2)
    c.close()
    c = _seeded()
    c.set_lap_budget(np.where(np.arange(B) % 3 == 2, 1, 16))                             # the oval controllers retire after a lap
    _steps(c, 200)
    rec = _records(c)
    for bad in (0, -1):
        arr = good.copy()
        arr[B // 2] = bad
        assert L.lmpc_rollout_set_lap_budget(c._h, nat.ptr(arr)) == LMPC_E_INVALID
        assert b"below 1" in L.lmpc_last_error()
    for bad in (np.ones(B - 1, int), np.ones(B + 1, int), 0, 1.5):
        with pytest.raises(ValueError):
            c.set_lap_budget(bad)
    assert np.array_equal(rec, _records(c))
    # the installed budget still holds: the retired oval controllers stay where they are, the others drive on
    _steps(c, 16)
    now = _records(c)
    gone = c.books()["lap_n"] >= np.where(np.arange(B) % 3 == 2, 1, 16)
    assert gone.any() and np.array_equal(now[gone], rec[gone]) and not np.array_equal(now[~gone], rec[~gone])
    c.close()
