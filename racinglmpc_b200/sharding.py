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
    v = np.append(np.asarray(ready, bool).reshape(-1), bool(done)).astype(np.int32)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        t = torch.from_numpy(v).to(device)
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
        v = t.cpu().numpy()
    return v[:-1] != 0, bool(v[-1])


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
