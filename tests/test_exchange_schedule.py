"""CPU tier: the schedule of the pooled exchange (sharding.ExchangeSchedule) on a fleet without a device.

Every controller of the fleet drives laps of a fixed length: after t closed-loop steps it has driven t // L laps and is t % L
steps into the next one, and a lap budget stops it at its budget.  The NumPy references of the progress numbers
(tests/support/group_stats.py, tests/support/lap_budget.py) turn that into the rows rollout_stats / rollout_group_stats report,
and `drive` polls them the way rollout_mc.run does.  Batch readiness is one row that decides for every group, group readiness
one row per group; a capture taken at a poll or between polls and resumed to more laps makes the decisions of a straight run;
diverged_step flags the captures that cannot; the independent mode never exchanges; groups empty on every rank never exchange;
and over two gloo ranks both ranks decide alike, with one MIN all-reduce of two int32 per poll under batch readiness."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from racinglmpc_b200 import sharding
import group_stats as gs
import lap_budget as lb

POLL, SHIP, CPU = 8, 40, torch.device("cpu")


class Fleet:
    """Controllers with fixed lap lengths `lap_len` in pool groups `grp` (G groups), with an optional lap budget."""

    def __init__(self, lap_len, grp, G, budget=None):
        self.lap_len, self.grp, self.G, self.budget = np.asarray(lap_len), np.asarray(grp), G, budget

    def rows(self, t, grouped):
        """The progress rows after t steps: [G, 4] under group readiness, the one row of the whole batch under batch readiness."""
        lap_n = t // self.lap_len if self.budget is None else np.minimum(t // self.lap_len, self.budget)
        grp, G = (self.grp, self.G) if grouped else (np.zeros_like(self.grp), 1)
        if self.budget is None:
            return gs.group_stats(lap_n, t % self.lap_len, np.zeros_like(lap_n), grp, G)
        return lb.group_stats(lap_n, t % self.lap_len, np.zeros_like(lap_n), grp, G, self.budget)

    def live(self):
        return np.bincount(self.grp, minlength=self.G) > 0

    def part(self, sel):
        return Fleet(self.lap_len[sel], self.grp[sel], self.G, None if self.budget is None else np.asarray(self.budget)[sel])


def drive(fleet, laps, readiness="batch", pooled=True, live=None, capture=False, start=None, max_steps=0):
    """rollout_mc.run's loop without the device: the polls [(step, groups exchanged, done)], the schedule and the last step."""
    s = sharding.ExchangeSchedule(fleet.G, laps, SHIP, POLL, readiness, pooled, live, capture, start)
    steps, max_steps, polls = s.start_step, max_steps or 300 * laps, []
    while steps < max_steps or s.repeat:
        if not s.repeat:
            steps += 1
            if steps % POLL:
                continue
        ready, done = s.poll(steps, fleet.rows(steps, readiness == "group"), CPU)
        assert ready.dtype == bool and ready.shape == (fleet.G,)
        polls.append((steps, ready.tolist(), bool(done)))
        if done:
            break
    return polls, s, steps


def _grouped(per_group, n=4, rng=None):
    """A fleet of len(per_group) groups of n controllers; group g laps in per_group[g] steps or a few less."""
    rng = rng or np.random.default_rng(0)
    lap_len = np.concatenate([L - rng.integers(0, 5, n) for L in per_group])
    lap_len[::n] = per_group                             # the slowest of every group laps in exactly per_group[g]
    return lap_len, np.repeat(np.arange(len(per_group)), n)


NARROW = Fleet(*_grouped([104, 101, 103]), 3)            # every group's lap `laps` ends before any is ready for round `laps`
WIDE = Fleet(*_grouped([80, 100, 130]), 3)               # the fast group is ready for round `laps` while the slow one drives


def test_batch_decides_every_group_where_one_group_row_over_the_batch_does():
    for fleet in (NARROW, WIDE, Fleet(WIDE.lap_len, WIDE.grp, 3, budget=np.where(WIDE.grp == 2, 2, 3))):
        polls, s, _ = drive(fleet, 3)
        one = Fleet(fleet.lap_len, np.zeros_like(fleet.grp), 1, fleet.budget)
        polls1, s1, _ = drive(one, 3, "group", live=one.live())
        assert all(r == [r[0]] * 3 for _, r, _ in polls)
        assert [(t, r[0], d) for t, r, d in polls] == [(t, r[0], d) for t, r, d in polls1]
        assert s.exchange_steps == s1.exchange_steps * 3 and len(s.exchange_steps[0]) == 2     # rounds 1 and 2 of 3 laps
        # the same steps by the readiness expression rollout_mc applied inline on the batch row
        r, want = 1, []
        for t, _, _ in polls:
            lap_min, _, since, _ = fleet.rows(t, False)[0]
            if gs.inline_rule(lap_min, since, r, 3, SHIP):
                r, want = r + 1, want + [t]
        assert s.exchange_steps[0] == want
        # group readiness with one group is batch readiness, step for step
        polls2, s2, end = drive(one, 3, "batch")
        assert polls2 == polls1
        assert {k: v for k, v in s2.state(end).items() if k != "next_rounds"} == \
            {k: v for k, v in s1.state(end).items() if k != "next_rounds"}
        assert s2.state(end)["next_rounds"] is None and s1.state(end)["next_rounds"] == [s1.next_round]


def _merged(*runs):
    """{step: groups exchanged} over the polls of several runs, each group at most once per step."""
    out = {}
    for polls in runs:
        for t, r, _ in polls:
            prev = out.get(t, [False] * len(r))
            assert not any(a and b for a, b in zip(prev, r)), t          # a group exchanged at a poll is not exchanged again
            out[t] = [a or b for a, b in zip(prev, r)]
    return {t: r for t, r in out.items() if any(r)}


# controller 0 retires after one lap at step 100; controller 1 has 3 laps by then, so at poll 104 group 0 is ready for rounds 1
# and 2: a capture at 104 must not exchange the group again when the resumed run decides that poll anew
JUMP = Fleet([100, 30, 101, 98], [0, 0, 1, 1], 2, budget=[1, 9, 9, 9])


def test_capture_and_resume_equal_a_straight_run():
    for fleet in (NARROW, JUMP):
        for readiness in ("batch", "group"):
            live = fleet.live() if readiness == "group" else None
            straight, s5, end5 = drive(fleet, 5, readiness, live=live)
            done3 = drive(fleet, 3, readiness, live=live)[2]
            repeated = 0
            for cap in [t + dt for t in range(POLL, done3 + 1, POLL) for dt in (0, 3) if t + dt <= done3]:
                first, s3, end = drive(fleet, 3, readiness, live=live, capture=True, max_steps=cap)
                st = s3.state(end)
                assert end == cap and set(st) == set(sharding.ExchangeSchedule.FIELDS)
                if st["diverged_step"] is not None:       # JUMP's group 0 is ready for round 3 from step 120 on
                    assert fleet is JUMP and readiness == "group" and cap >= 120
                    continue
                assert st["exchanged"] == (first[-1][1] if first and first[-1][0] == cap else [False] * fleet.G)
                repeated += any(st["exchanged"])
                rest, sr, endr = drive(fleet, 5, readiness, live=live, start=st)
                assert rest[0][0] == (cap if cap % POLL == 0 else cap - cap % POLL + POLL)      # a poll is decided again, in time
                assert _merged(first, rest) == _merged(straight) and endr == end5 and rest[-1][2]
                assert sr.state(endr) == s5.state(end5)
            assert repeated >= 2                          # some captures were taken at a poll that exchanged


def _first_late_poll(fleet, polls, laps):
    """The first poll, not done, at which a group of `fleet` with controllers had been ready for round `laps` (its slowest
    controller `SHIP` steps into lap laps + 1): by the fixed lap lengths, without the schedule."""
    slowest = [fleet.lap_len[fleet.grp == g].max() for g in range(fleet.G) if (fleet.grp == g).any()]
    return next((t for t, _, d in polls if not d and any(t >= laps * L + SHIP for L in slowest)), None)


def test_diverged_step_marks_exactly_the_captures_a_longer_run_overtakes():
    seen = set()
    for per_group in ([104, 101, 103], [80, 100, 130], [100, 60, 100], [90, 90], [130, 70, 100, 95]):
        # the last group is empty: its sentinel row reads as ready for every round, but it is not live
        fleet = Fleet(*_grouped(per_group), len(per_group) + 1)
        for laps in (2, 3):
            polls, s, end = drive(fleet, laps, "group", live=fleet.live(), capture=True)
            # each group on its own counter: round r at the first poll once its slowest controller is SHIP steps into lap r + 1
            assert s.exchange_steps == [[-(-(r * L + SHIP) // POLL) * POLL for r in range(1, laps)] for L in per_group] + [[]]
            want = _first_late_poll(fleet, polls, laps)
            assert s.state(end)["diverged_step"] == want, (per_group, laps)
            seen.add(want is None)
            assert drive(fleet, laps, "group", live=fleet.live())[1].diverged_step is None       # only with a capture
            assert drive(fleet, laps, "batch", capture=True)[1].state(end)["diverged_step"] is None
            # a run resumed from it equals the straight run exactly when nothing was flagged
            more = drive(fleet, laps + 2, "group", live=fleet.live())[0]
            rest = drive(fleet, laps + 2, "group", live=fleet.live(), start=s.state(end))[0]
            assert (_merged(polls, rest) == _merged(more)) == (want is None), (per_group, laps)
    assert seen == {True, False}


def test_the_independent_mode_never_exchanges_but_stops():
    for fleet in (NARROW, WIDE):
        polls, s, end = drive(fleet, 3, pooled=False)
        assert not any(any(r) for _, r, _ in polls) and polls[-1][2] and end == drive(fleet, 3)[2]
        assert s.exchange_steps == [[]] * 3 and s.state(end)["next_round"] == 1
        assert [d for _, _, d in polls] == [d for _, _, d in drive(fleet, 3)[0]]


def test_groups_empty_on_every_rank_never_exchange():
    lap_len, grp = _grouped([104, 101, 103])
    fleet = Fleet(lap_len, np.where(grp == 1, 3, grp), 4)          # group 1 of four holds no controller
    assert fleet.live().tolist() == [True, False, True, True]
    polls, s, _ = drive(fleet, 3, "group", live=fleet.live())
    assert s.exchange_steps[1] == [] and not any(r[1] for _, r, _ in polls)
    assert all(len(s.exchange_steps[g]) == 2 for g in (0, 2, 3))
    # without the mask its sentinel row would be exchanged at the first poll
    assert drive(fleet, 3, "group")[0][0][1][1]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


FLEET2 = Fleet(*_grouped([104, 70, 150, 100]), 5)     # group 4 is empty everywhere
# rank 0 holds groups 1 and 3, rank 1 group 2, and group 0 is split over both.  Rank 0 alone has its 3 laps from step 312 on, so
# it is ready for a round >= laps under batch readiness long before the agreed `done`: that is no divergence
RANK_OF = np.where(FLEET2.grp == 0, np.arange(len(FLEET2.grp)) % 2, (FLEET2.grp == 2).astype(int))


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    calls, all_reduce = [], dist.all_reduce

    def counted(t, *a, **k):
        calls.append((tuple(t.shape), str(t.dtype), str(k.get("op"))))
        return all_reduce(t, *a, **k)
    dist.all_reduce = counted
    try:
        mine = FLEET2.part(RANK_OF == rank)
        out = {}
        for readiness in ("batch", "group"):
            del calls[:]
            live = sharding.sum_over_ranks(np.bincount(mine.grp, minlength=mine.G), CPU) > 0 if readiness == "group" else None
            polls, s, end = drive(mine, 3, readiness, live=live, capture=readiness == "batch")
            out[readiness] = (polls, s.state(end), list(calls))
        q.put((rank, out))
    finally:
        dist.destroy_process_group()


def test_two_ranks_decide_alike_with_one_all_reduce_per_poll():
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    assert res[0] == res[1]
    MIN, SUM = str(dist.ReduceOp.MIN), str(dist.ReduceOp.SUM)
    for readiness, rows in (("batch", 1), ("group", FLEET2.G)):
        polls, state, calls = res[0][readiness]
        # the ranks' decisions are those of one rank holding the whole fleet
        whole = drive(FLEET2, 3, readiness, live=FLEET2.live() if readiness == "group" else None)
        assert polls == whole[0] and state == whole[1].state(whole[2])
        live = [] if readiness == "batch" else [((FLEET2.G,), "torch.int64", SUM)]
        assert calls == live + [((rows + 1,), "torch.int32", MIN)] * len(polls)
    assert res[0]["batch"][1]["diverged_step"] is None and res[0]["batch"][0][-1][0] >= 450
    assert res[0]["batch"][1]["exchange_steps"][0] and not res[0]["group"][1]["exchange_steps"][4]
