"""Multi-GPU plumbing: batch sharding and the per-lap safe-set exchange (SURVEY §8e).

The hot path shards over independent controller instances: rank r owns the contiguous range
``shard_range(B, r, world)`` and no collective sits inside solve()/addPoint().  The only exchange is the
optional *pooled safe-set* mode: once per lap, after LMPC.addTrajectory (PredictiveControllers.py:418-445),
every rank all-gathers the laps its instances just finished so that all ranks can rank laps by LapTime
(PC.py:395) over the pooled set.  torch.distributed is plumbing here (NCCL on GPUs, gloo in the CPU tests).
"""
import numpy as np
import torch
import torch.distributed as dist


def shard_range(batch, rank, world):
    """Contiguous instance range [lo, hi) of `rank`; sizes differ by at most one."""
    base, rem = divmod(int(batch), int(world))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def pack_laps(xs, us, Tmax):
    """Lists of laps (x[T,6], u[T,2]) -> padded rows [n, Tmax, 8] and lengths [n] (int32)."""
    n = len(xs)
    rows = np.zeros((n, Tmax, 8))
    lens = np.zeros(n, np.int32)
    for i, (x, u) in enumerate(zip(xs, us)):
        T = x.shape[0]
        if T > Tmax:
            raise ValueError("lap longer than Tmax")
        rows[i, :T, 0:6] = x
        rows[i, :T, 6:8] = u
        lens[i] = T
    return rows, lens


def allgather_laps(rows, lens, group=None):
    """All-gather padded laps over the process group.

    rows: tensor [n_local, Tmax, 8] (CUDA for NCCL, CPU for gloo), lens: int32 tensor [n_local];
    n_local must be equal on all ranks (pad with zero-length laps).  Returns (rows_all [world*n_local, Tmax, 8],
    lens_all [world*n_local]) in rank order, i.e. global instance order under `shard_range`."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return rows, lens
    out_rows = torch.empty((world * rows.shape[0],) + tuple(rows.shape[1:]), dtype=rows.dtype, device=rows.device)
    out_lens = torch.empty(world * lens.shape[0], dtype=lens.dtype, device=lens.device)
    dist.all_gather_into_tensor(out_rows, rows.contiguous(), group=group)
    dist.all_gather_into_tensor(out_lens, lens.contiguous(), group=group)
    return out_rows, out_lens


def allgather_vec(v, group=None):
    """All-gather a 1-D tensor of equal length on every rank, in rank order."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return v
    out = torch.empty(world * v.shape[0], dtype=v.dtype, device=v.device)
    dist.all_gather_into_tensor(out, v.contiguous(), group=group)
    return out


def pooled_fastest(lens_all, k, valid_min=2, groups=None):
    """Indices (into the gathered order) of the k fastest finished laps, ties to the lower global index —
    the stable counterpart of np.argsort(LapTime)[:k] (PC.py:395,402).
    groups: None, or the pool group of every gathered lap; then a list whose entry g holds the k fastest laps of group g, for
    g in 0 .. max(groups) (laps of a negative group are never ranked) — the host counterpart of the grouped exchange."""
    lens_np = lens_all.cpu().numpy() if torch.is_tensor(lens_all) else np.asarray(lens_all)
    if groups is not None:
        groups = np.asarray(groups).reshape(-1)
        return [np.nonzero(groups == g)[0][pooled_fastest(lens_np[groups == g], k, valid_min)] for g in range(int(groups.max()) + 1)]
    idx = np.where(lens_np >= valid_min)[0]
    order = idx[np.argsort(lens_np[idx], kind="stable")]
    return order[:k]


def design_groups(*indices):
    """Pool groups of a crossed design: every distinct combination of the per-controller indices (e.g. track, vehicle and
    parameter-set index) is one group, numbered 0 .. G-1 in order of first appearance.  Returns (group index int32 [batch], G)."""
    cols = np.stack([np.asarray(i).reshape(-1) for i in indices], axis=1)
    seen, out = {}, np.empty(cols.shape[0], np.int32)
    for b, key in enumerate(map(tuple, cols.tolist())):
        out[b] = seen.setdefault(key, len(seen))
    return out, len(seen)


def ready_groups(stats, next_round, laps, ship_after):
    """The readiness rule of the pooled exchange, per row of ``stats`` [G, 4] (rollout_group_stats, or the one row of
    rollout_stats for the whole batch): row g is ready for round next_round[g] (a scalar applies to every row) once the round
    exists (r < laps), every controller of the row has driven r laps, and either every one has driven more than r laps or the
    slowest are ``ship_after`` steps into lap r + 1.  Returns bool [G].
    Applied per rank and combined with AND (agree_groups), it equals the rule on the union of the ranks' controllers: the union's
    minimum is the smallest rank minimum, and its steps-into-lap is the smallest among the ranks at that minimum.  A row without
    controllers (INT32_MAX, 0, INT32_MAX, 0) is ready for every round below ``laps`` and so leaves the decision to the others."""
    s = np.asarray(stats).reshape(-1, 4)
    r = np.asarray(next_round)
    lap_min, since = s[:, 0], s[:, 2]
    return (r < laps) & (lap_min >= r) & ((lap_min > r) | (since >= ship_after))


def agree_groups(ready, done, device, group=None):
    """One MIN all-reduce of [ready_0 .. ready_{G-1}, done] (int32): a group exchanges only if it is ready on every rank, and the
    batch stops only once every rank is done.  Returns (ready bool [G], done bool), the same on every rank."""
    ready, done = np.asarray(ready, bool).reshape(-1), bool(done)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        t = torch.from_numpy(np.append(ready, done).astype(np.int32)).to(device)
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
        v = t.cpu().numpy()
        return v[:-1] != 0, bool(v[-1])
    return ready, done


class ExchangeSchedule:
    """When the pooled exchange runs, and what a resumed run needs: one row for the whole batch (readiness="batch"; it decides for
    every pool group) or one per group ("group"), each with a round counter.  A poll agrees over the ranks `done` and the rows that
    ready_groups finds ready, less the independent mode, rows not `live` and what a repeated poll already exchanged.  With
    `capture`, group readiness records the first poll, not done, at which a live group was ready for a round >= laps."""
    FIELDS = ("steps", "next_round", "next_rounds", "exchanged", "exchange_steps", "diverged_step")

    def __init__(self, groups, laps, ship_after, poll, readiness="batch", pooled=True, live=None, capture=False, start=None):
        self.G, self.grouped, self.laps, self.ship_after = int(groups), readiness == "group", laps, ship_after
        n = self.G if self.grouped else 1
        self.live = (np.ones(n, bool) if live is None else np.asarray(live, bool).reshape(n)) & bool(pooled)
        self.watch, self.diverged_step, self.last_poll = bool(capture) and self.grouped, None, -1
        self.start_step, self.next_round = (0, 1) if start is None else (int(start["steps"]), int(start["next_round"]))
        self.rounds = np.array(start["next_rounds"] if start is not None and self.grouped else [self.next_round] * n, np.int64)
        self.exchange_steps = [[] for _ in range(self.G)] if start is None else [list(v) for v in start["exchange_steps"]]
        self.exchanged = np.zeros(self.G, bool) if start is None else np.asarray(start["exchanged"], bool).reshape(self.G)
        self.repeat = start is not None and self.start_step % poll == 0     # captured at a poll: decide it again, under new laps

    def poll(self, steps, prog, device):
        """The poll at closed-loop step `steps` on the progress rows prog [rows, 4] -> (bool [G]: groups to exchange now, done)."""
        ok = self.live & ~self.exchanged[:len(self.rounds)] if self.repeat else self.live     # row r's first group is group r
        ready, done = agree_groups(ready_groups(prog, self.rounds, self.laps, self.ship_after) & ok, prog[:, 0].min() >= self.laps, device)
        if self.watch and self.diverged_step is None and not done and \
                (ready_groups(prog, self.rounds, np.iinfo(np.int32).max, self.ship_after) & self.live & ~ready).any():
            self.diverged_step = steps
        self.exchanged, self.last_poll, self.repeat = ready if self.grouped else ready.repeat(self.G), steps, False
        if ready.any():
            self.next_round += 1
            self.rounds += ready
            for g in np.nonzero(self.exchanged)[0]:
                self.exchange_steps[g].append(steps)
        return self.exchanged, done

    def state(self, steps):
        """The FIELDS of a capture taken at closed-loop step `steps` (next_rounds is None under batch readiness)."""
        return dict(steps=steps, next_round=self.next_round, next_rounds=self.rounds.tolist() if self.grouped else None,
                    exchanged=(self.exchanged if self.last_poll == steps else np.zeros(self.G, bool)).tolist(),
                    exchange_steps=self.exchange_steps, diverged_step=self.diverged_step)


def sum_over_ranks(values, device, group=None):
    """Element-wise sum of an integer vector over the ranks (int64 numpy array)."""
    v = np.asarray(values, np.int64).reshape(-1)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        t = torch.from_numpy(v.copy()).to(device)
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
        v = t.cpu().numpy()
    return v


def max_over_ranks(value, device, group=None):
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return float(t.item())
