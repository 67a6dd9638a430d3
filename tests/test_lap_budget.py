"""CPU tier: lap budgets (lmpc_rollout_set_lap_budget): packing and refusals of _native.make_lap_budget, the ABI symbol and its
prototype, the driver's refusals before any device work, and the progress numbers with retired controllers (tests/support/
lap_budget.py) against sharding.ready_groups: a group whose controllers have all retired reads as ready and as done, and a retired
controller does not hold its group back."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat, sharding
import group_stats as gs
import lap_budget as lb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
import rollout_mc                                                  # noqa: E402

B = 12
INT32_MAX = 2 ** 31 - 1


def test_budget_packs_and_none_means_no_budget():
    assert nat.make_lap_budget(None, B) is None
    u = nat.make_lap_budget(3, B)
    assert u.dtype == np.int32 and u.flags["C_CONTIGUOUS"] and np.array_equal(u, np.full(B, 3))
    assert np.array_equal(nat.make_lap_budget(np.int64(2), B), np.full(B, 2))
    m = nat.make_lap_budget(2 + np.arange(B) % 2, B)
    assert m.dtype == np.int32 and np.array_equal(m, 2 + np.arange(B) % 2)
    assert nat.make_lap_budget([1] * B, B).min() == 1
    assert nat.make_lap_budget(np.full(B, 2 ** 31 - 1), B).max() == 2 ** 31 - 1


@pytest.mark.parametrize("budget", [0, -1, 2.5, math.nan, 2 ** 31, np.zeros(B, int), np.full(B, -1), np.full(B, 1.5),
                                    np.ones(B - 1, int), np.ones(B + 1, int), np.zeros((0,), int),
                                    np.where(np.arange(B) == 5, 0, 3)])
def test_bad_budgets_are_a_value_error(budget):
    with pytest.raises(ValueError):
        nat.make_lap_budget(budget, B)


def test_streams_and_budgets_share_their_rules_but_not_their_floor():
    assert np.array_equal(nat.make_noise_streams(np.zeros(B, int), B), np.zeros(B))      # stream 0 exists, budget 0 does not
    with pytest.raises(ValueError):
        nat.make_lap_budget(np.zeros(B, int), B)


def test_symbol_and_prototype():
    L = nat.lib()
    assert "lmpc_rollout_set_lap_budget" in nat.exported_symbols()
    assert L.lmpc_rollout_set_lap_budget.argtypes == [C.c_void_p, C.c_void_p]
    assert L.lmpc_rollout_set_lap_budget(None, None) != 0 and b"null handle" in L.lmpc_last_error()


def test_driver_refuses_bad_budgets_before_any_device_work():
    for bad in (0, [1, 2], np.full(B, 0.5)):
        with pytest.raises(ValueError):
            rollout_mc.run(batch=B, lap_budget=bad)
    start = dict(records=np.zeros((B, 1)), clock=0, steps=8, next_round=1, next_rounds=None, exchanged=[False], exchange_steps=[[]],
                 diverged_step=None, batch=B, laps=3, mode="independent", readiness="batch", poll=8, warm=False, pool_groups=1,
                 layout=rollout_mc.layout(), lap_budget=[3] * B, tables={})
    with pytest.raises(ValueError, match="lap_budget is below"):
        rollout_mc.run(batch=B, laps=5, mode="independent", start=start, lap_budget=np.where(np.arange(B) == 4, 2, 5))


def test_driven_steps_counts_filed_laps_and_the_lap_under_way():
    hist = np.full((3, 16), -1, np.int32)
    hist[0, :2] = (180, 170)
    hist[1, :1] = (200,)
    bk = dict(lap_n=np.array([2, 1, 0], np.int32), lap_hist=hist)
    assert rollout_mc._driven_steps(bk, dict(cl_len=np.array([0, 17, 90], np.int32))) == 180 + 170 + 200 + 17 + 90


def test_stats_without_a_budget_are_the_existing_ones():
    rng = np.random.default_rng(3)
    lap_n, cl_len, fl, grp = rng.integers(0, 4, 40), rng.integers(0, 200, 40), rng.integers(0, 2, 40), rng.integers(0, 5, 40)
    grp[grp == 3] = 2                                    # group 3 stays empty
    assert np.array_equal(lb.group_stats(lap_n, cl_len, fl, grp, 5), gs.group_stats(lap_n, cl_len, fl, grp, 5))
    never = np.full(40, 16)
    assert np.array_equal(lb.group_stats(lap_n, cl_len, fl, grp, 5, never), gs.group_stats(lap_n, cl_len, fl, grp, 5))


def test_all_retired_is_the_empty_group_row_and_reads_ready_and_done():
    lap_n, cl_len, fl = np.array([3, 3, 2, 2]), np.zeros(4, int), np.array([0, 8, 0, 0])
    grp, budget = np.array([0, 0, 1, 1]), np.array([3, 3, 2, 2])
    s = lb.group_stats(lap_n, cl_len, fl, grp, 2, budget)
    assert s.tolist() == [[INT32_MAX, 3, INT32_MAX, 1], [INT32_MAX, 2, INT32_MAX, 0]]
    laps = 3
    assert s[:, 0].min() >= laps                                               # the driver's `done`
    assert sharding.ready_groups(s, np.array([1, 2]), laps, 40).all()          # like a group without controllers
    assert not sharding.ready_groups(s, np.array([3, 3]), laps, 40).any()      # no round beyond the last
    one = lb.group_stats(lap_n, cl_len, fl, np.zeros(4, int), 1, budget)
    assert one.tolist() == [[INT32_MAX, 3, INT32_MAX, 1]]


def test_a_retired_controller_does_not_hold_its_group_back():
    # budgets 2 and 4 in one group: the budget-2 controllers retired at 2 laps, the others are 50 steps into lap 4
    lap_n, cl_len = np.array([2, 3, 2, 3]), np.array([0, 50, 0, 61])
    grp, budget = np.zeros(4, int), np.array([2, 4, 2, 4])
    held = gs.group_stats(lap_n, cl_len, np.zeros(4, int), grp, 1)
    free = lb.group_stats(lap_n, cl_len, np.zeros(4, int), grp, 1, budget)
    assert held.tolist() == [[2, 3, 0, 0]] and free.tolist() == [[3, 3, 50, 0]]
    assert not sharding.ready_groups(held, 3, 4, 40)[0] and sharding.ready_groups(free, 3, 4, 40)[0]
    assert free[0, 0] < 4                                                      # not done: the live ones have a lap to go
