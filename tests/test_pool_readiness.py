"""CPU tier: per-group readiness of the pooled exchange (rollout_mc.run(readiness="group")).

``sharding.ready_groups`` with one row is the batch rule rollout_mc applied inline; with G rows each row is that rule on its
group alone; applied per rank and ANDed over the ranks (``agree_groups``: one MIN all-reduce) it equals the rule on the union
of the ranks' controllers, empty groups included.  Over gloo with two ranks the agreed vector is the same on both.  The Python
argument checks come before any device work."""
import itertools
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from racinglmpc_b200 import sharding
from racinglmpc_b200.controller import BatchedController
from group_stats import INT32_MAX, group_stats, inline_rule

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIP = 40


def test_one_row_equals_the_inline_batch_rule():
    for lap_min, since, r, laps in itertools.product(list(range(6)) + [INT32_MAX], list(range(0, 90, 3)) + [SHIP - 1, SHIP, INT32_MAX],
                                                     range(6), range(1, 6)):
        got = sharding.ready_groups([(lap_min, 7, since, 3)], r, laps, SHIP)
        assert got.shape == (1,) and got.dtype == bool
        assert bool(got[0]) == inline_rule(lap_min, since, r, laps, SHIP), (lap_min, since, r, laps)


def test_each_row_is_the_rule_on_its_group_alone():
    rng = np.random.default_rng(5)
    for _ in range(200):
        G, laps = int(rng.integers(1, 65)), int(rng.integers(1, 5))
        stats = np.stack([rng.integers(0, 5, G), rng.integers(0, 6, G), rng.integers(0, 80, G), rng.integers(0, 4, G)], axis=1)
        stats[rng.random(G) < 0.1] = (INT32_MAX, 0, INT32_MAX, 0)
        r = rng.integers(0, 5, G)
        got = sharding.ready_groups(stats, r, laps, SHIP)
        assert got.tolist() == [inline_rule(stats[g, 0], stats[g, 2], r[g], laps, SHIP) for g in range(G)]
        # a scalar round applies to every row
        assert sharding.ready_groups(stats, 2, laps, SHIP).tolist() == [inline_rule(s[0], s[2], 2, laps, SHIP) for s in stats]


def test_rule_per_rank_anded_equals_the_rule_on_the_union():
    """Random populations (laps driven, steps into the lap, group) split over 1-4 ranks; groups may be empty on a rank or on
    every rank.  AND over ranks of the per-rank rule == the rule on the union's statistics."""
    rng = np.random.default_rng(17)
    checked_empty = 0
    for trial in range(400):
        B, G, world = int(rng.integers(1, 40)), int(rng.integers(1, 9)), int(rng.integers(1, 5))
        laps = int(rng.integers(1, 5))
        lap_n = rng.integers(0, 4, B)
        cl_len = rng.integers(0, 2 * SHIP, B)
        flags = (rng.random(B) < 0.2).astype(np.int32)
        grp = rng.integers(0, G, B)
        rank_of = rng.integers(0, world, B)
        r = rng.integers(0, 4, G)
        union = sharding.ready_groups(group_stats(lap_n, cl_len, flags, grp, G), r, laps, SHIP)
        anded = np.ones(G, bool)
        for k in range(world):
            m = rank_of == k
            st = group_stats(lap_n[m], cl_len[m], flags[m], grp[m], G)
            checked_empty += int((st[:, 0] == INT32_MAX).sum())
            anded &= sharding.ready_groups(st, r, laps, SHIP)
        # a group empty on every rank is ready for every existing round: the rule leaves it to the caller (rollout_mc never
        # exchanges such a group)
        empty = np.bincount(grp, minlength=G) == 0
        assert np.array_equal(anded[~empty], union[~empty]), trial
        assert np.array_equal(anded[empty], r[empty] < laps), trial
        # the batch values: done from the minimum of the rows, flagged from their sum
        st = group_stats(lap_n, cl_len, flags, grp, G)
        assert st[:, 0].min() == lap_n.min() and st[:, 3].sum() == int((flags != 0).sum())
    assert checked_empty > 100


def test_group_stats_of_one_group_are_the_batch_numbers():
    rng = np.random.default_rng(2)
    lap_n, cl_len, flags = rng.integers(0, 4, 50), rng.integers(0, 200, 50), rng.integers(0, 3, 50)
    st = group_stats(lap_n, cl_len, flags, np.zeros(50, int), 1)
    mn = lap_n.min()
    assert st.tolist() == [[mn, lap_n.max(), cl_len[lap_n == mn].min(), int((flags != 0).sum())]]


def test_agree_groups_without_a_process_group_is_the_local_vector():
    ready, done = sharding.agree_groups(np.array([True, False, True]), False, torch.device("cpu"))
    assert ready.tolist() == [True, False, True] and done is False
    assert sharding.sum_over_ranks([3, 0, 1], torch.device("cpu")).tolist() == [3, 0, 1]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        cpu = torch.device("cpu")
        mine = [np.array([1, 1, 0, 1, 0], bool), np.array([1, 0, 0, 1, 1], bool)][rank]
        ready, done = sharding.agree_groups(mine, rank == 0, cpu)
        ready2, done2 = sharding.agree_groups(np.ones(5, bool), True, cpu)
        counts = sharding.sum_over_ranks([2, 0, rank, 0], cpu)
        q.put((rank, ready.tolist(), done, ready2.tolist(), done2, counts.tolist()))
    finally:
        dist.destroy_process_group()


def test_agree_groups_world2_gives_both_ranks_the_same_vector():
    world = 2
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    want = ([True, False, False, True, False], False, [True] * 5, True, [4, 0, 1, 0])
    assert res == [(0,) + want, (1,) + want]


def _rollout_mc():
    sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
    try:
        import rollout_mc
    finally:
        sys.path.pop(0)
    return rollout_mc


def test_group_readiness_needs_the_pooled_mode_before_any_device_work(monkeypatch):
    rm = _rollout_mc()

    def boom(*a, **k):
        raise AssertionError("device work before the argument check")
    monkeypatch.setattr(torch.cuda, "set_device", boom)
    monkeypatch.setattr(rm, "BatchedController", boom)
    with pytest.raises(ValueError, match="pooled"):
        rm.run(batch=12, mode="independent", readiness="group")
    with pytest.raises(ValueError, match="readiness"):
        rm.run(batch=12, mode="pooled", readiness="slowest")
    with pytest.raises(AssertionError, match="device work"):
        rm.run(batch=12, mode="pooled", readiness="group")


class _NoLib:
    def __getattr__(self, name):
        raise AssertionError("library call before the argument check: %s" % name)


@pytest.mark.parametrize("mask", [np.ones(2, bool), np.ones(4, bool), [1, 0], np.ones((1, 2)), [0, 1, 2], [1, -1, 0]])
def test_export_mask_of_the_wrong_length_or_values_is_a_value_error(mask):
    c = BatchedController.__new__(BatchedController)          # no device handle: the checks come before the library
    c._lib, c._h, c._pool_groups = _NoLib(), None, 3
    with pytest.raises(ValueError):
        c.pool_export(3, 288, 0, 0, 0, groups=mask)
