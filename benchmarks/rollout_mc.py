#!/usr/bin/env python
"""BASELINE.json configs[3]: LMPC Monte-Carlo rollouts sharded over the GPUs of one node, with the once-per-lap NCCL
all-gather of finished laps (pooled-safe-set exchange, SURVEY §8e).

Every instance is an independent LMPC controller + vehicle (its own 1000-step PID lap as initial safe set, Philox process
noise), advanced entirely on the device: K1 regression -> K2 selection -> QP -> shift -> addPoint -> dynModel per step, lap
hand-over and lap bookkeeping included (csrc/lapbooks.cuh).  The host launches kernels and, every `poll` steps, reads four
integers of progress; ranks agree on exchanging / stopping through one tiny all-reduce at those polls, so no rank can enter
a collective the others skip.

  --mode independent   reference semantics: no data-path collective (replicas).
  --mode pooled        once every controller of every rank is `--ship-after` steps into lap r+1, each rank packs its
                       `share + 1` fastest laps r on the device (only the globally fastest laps are ever selected, PC.py:395, so
                       a rank's candidates are its own fastest few: ~60 KB per rank instead of every lap), all ranks all-gather
                       them over NCCL, rank them by (lap time, global id) and every controller files the `share` fastest laps
                       it does not own as additional stored laps (safe set + regression model).

  python benchmarks/rollout_mc.py --batch 8192 --laps 3            (1 GPU)
  python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 benchmarks/rollout_mc.py --batch 8192
Prints one JSON line (rank 0): closed-loop steps/s over all GPUs (device events, max over ranks), lap-length statistics per
LMPC lap, exchange time and bytes."""
import argparse
import json
import os
import sys
import time
import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from racinglmpc_b200 import workloads, sharding, reference_params as rp      # noqa: E402
from racinglmpc_b200.controller import BatchedController                      # noqa: E402


def run(batch=8192, laps=3, mode="pooled", share=2, tpad=288, ship_after=40, poll=8, max_steps=0, seed=1234, local=None, warm=False,
        final=None, param_sets=None, vehicle_sets=None, books=None, track_sets=None):
    """One Monte-Carlo run on this rank's GPU (torch.distributed may or may not be initialised).  Returns a dict (all ranks).
    final: None, or a dict that receives the closed loop's end state (rollout_state) and the last step's solver report (step_results).
    books: None, or a dict that receives the lap books (books) and the health counters (flags_or, unsolved).
    param_sets: None, or (params, index, QterminalSlack) handed to BatchedController.set_param_sets after construction (a
    parameter sweep over the batch; the result then holds per-set lap statistics under "per_set_rank0").
    vehicle_sets: None, or (vehicles, index) handed to BatchedController.set_vehicles (a sweep over the plant, PID lap included; the
    result then holds per-vehicle lap statistics under "per_vehicle_rank0").  The pooled mode still exchanges laps between
    controllers whatever their car, so plant sweeps run in the independent mode.
    track_sets: None, or (tracks, index) handed to BatchedController.set_tracks (several circuits in one batch; the result then
    holds per-track lap statistics under "per_track_rank0").  A lap of another circuit is not a trajectory of this one, so more
    than one track runs in the independent mode only (ValueError otherwise, raised before any collective)."""
    if track_sets is not None and mode == "pooled" and len(track_sets[0]) > 1:
        raise ValueError("the pooled mode exchanges laps between controllers: it needs one track, got %d" % len(track_sets[0]))
    rank = dist.get_rank() if dist.is_initialized() else 0
    world = dist.get_world_size() if dist.is_initialized() else 1
    local = int(os.environ.get("LOCAL_RANK", 0)) if local is None else local
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    B, N = int(batch), 12
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, B, workloads.track_seg_table(), rp.TRACK_LENGTH, trToUse=4, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=Qts, device=local, Tmax=1280, ss_cap=7, model_cap=5, warm_start=warm)
    if param_sets is not None:
        c.set_param_sets(*param_sets)
    if vehicle_sets is not None:
        c.set_vehicles(*vehicle_sets)
    if track_sets is not None:
        c.set_tracks(*track_sets)
    stream = torch.cuda.ExternalStream(c.stream, device=dev)
    x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (B, 1))
    # ---- main.py:65-66 + 99-110 on the device: every controller drives its OWN PID lap (the full 100 s) and is seeded with it
    t0 = time.perf_counter()
    c.enable_rollout(Tcl=1024)
    c.rollout_set_state(x0, x0)
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321 + rank)
    c.rollout_seed_from_record_dev(copies=4)
    c.sync()
    pid_s = time.perf_counter() - t0
    c.rollout_set_state(x0, x0)
    kbest = share + 1
    rows = torch.zeros(kbest, tpad, 9, dtype=torch.float64, device=dev)
    meta = torch.zeros(kbest, 4, dtype=torch.int32, device=dev)
    rows_all = torch.zeros(world * kbest, tpad, 9, dtype=torch.float64, device=dev)
    meta_all = torch.zeros(world * kbest, 4, dtype=torch.int32, device=dev)
    agree = torch.zeros(2, dtype=torch.int32, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    max_steps = int(max_steps) or 300 * laps
    steps, next_round, n_xchg, xchg_s, took_total = 0, 1, 0, 0.0, 0
    it_sum, it_n, it_max = 0.0, 0, 0                     # interior-point iterations, sampled at the polls
    l0 = c.kernel_launches
    e0.record(stream)
    while steps < max_steps:
        c.rollout_step(seed=seed + rank)
        c.rollout_commit_laps_dev()                       # every controller whose lap just ended hands it over, on the device
        steps += 1
        if steps % poll:
            continue
        # ---- poll: four integers of progress; ranks agree on what happens next (same decision everywhere, no deadlock)
        lap_min, lap_max, since, flagged = c.rollout_stats()
        its = c.step_results()["iters"]
        it_sum += float(its.mean()); it_n += 1; it_max = max(it_max, int(its.max()))
        ready = int(mode == "pooled" and next_round < laps and lap_min >= next_round and (lap_min > next_round or since >= ship_after))
        done = int(lap_min >= laps)
        if world > 1:
            agree[0], agree[1] = ready, done
            dist.all_reduce(agree, op=dist.ReduceOp.MIN)
            ready, done = int(agree[0].item()), int(agree[1].item())
        if ready:
            tx = time.perf_counter()
            with torch.cuda.stream(stream):
                c.pool_export(kbest, tpad, rank * B, rows, meta)
                if world > 1:
                    dist.all_gather_into_tensor(rows_all, rows)
                    dist.all_gather_into_tensor(meta_all, meta)
                    took_total += c.pool_import(world * kbest, share, tpad, rank * B, rows_all, meta_all, count=True)
                else:
                    took_total += c.pool_import(kbest, share, tpad, 0, rows, meta, count=True)
            xchg_s += time.perf_counter() - tx
            n_xchg += 1
            next_round += 1
        if done:
            break
    e1.record(stream)
    c.sync()
    torch.cuda.synchronize()
    ms = sharding.max_over_ranks(e0.elapsed_time(e1), dev)
    bk = c.books()
    flags_or, unsolved = c.rollout_health()
    stats = []
    for r in range(laps):
        a = bk["lap_hist"][bk["lap_n"] > r, r]
        a = a if a.size else np.array([0])
        stats.append({"lap": r + 1, "n": int((bk["lap_n"] > r).sum()), "mean": float(a.mean()), "min": int(a.min()), "max": int(a.max())})
    out = {"benchmark": "configs[3] LMPC Monte-Carlo rollouts", "mode": mode, "n_gpus": world, "batch_per_gpu": B,
           "closed_loop_steps": steps, "ms_total": ms, "controller_steps_per_s": B * world * steps / (ms * 1e-3),
           "kernel_launches_rank0": int(c.kernel_launches - l0), "lap_stats_rank0": stats, "device_pid_laps_s": pid_s,
           "exchanges": n_xchg, "exchange_s_total": xchg_s, "exchange_ms_each": 1e3 * xchg_s / max(n_xchg, 1),
           "allgather_bytes_per_rank": int(rows.numel() * 8 + meta.numel() * 4), "laps_filed_rank0": took_total,
           "share": share, "ship_after": ship_after, "poll_every": poll, "warm_start": bool(warm),
           "ipm_iters_mean_sampled": it_sum / max(it_n, 1), "ipm_iters_max_sampled": it_max,
           "instances_with_flags_rank0": int((flags_or != 0).sum()), "flag_bits_rank0": int(np.bitwise_or.reduce(flags_or)),
           "unsolved_steps_rank0": int(unsolved.sum()), "late_accepts_rank0": c.late_accepts}
    if param_sets is not None:
        idx = np.asarray(param_sets[1]).reshape(B)
        out["per_set_rank0"] = [_set_stats(bk, flags_or, unsolved, idx == k, laps) for k in range(len(param_sets[0]))]
    if vehicle_sets is not None:
        idx = np.asarray(vehicle_sets[1]).reshape(B)
        out["per_vehicle_rank0"] = [_set_stats(bk, flags_or, unsolved, idx == k, laps) for k in range(len(vehicle_sets[0]))]
    if track_sets is not None:
        idx = np.asarray(track_sets[1]).reshape(B)
        out["per_track_rank0"] = [_set_stats(bk, flags_or, unsolved, idx == k, laps) for k in range(len(track_sets[0]))]
    if final is not None:
        final.update(c.rollout_state())
        final.update(c.step_results())
    if books is not None:
        books.update(bk, flags_or=flags_or, unsolved=unsolved)
    c.close()
    return out


def _set_stats(bk, flags_or, unsolved, sel, laps):
    """Lap lengths (mean / min per LMPC lap), unsolved steps and flagged controllers of the controllers `sel` of one parameter set or vehicle."""
    laps_out = []
    for r in range(laps):
        m = sel & (bk["lap_n"] > r)
        a = bk["lap_hist"][m, r]
        laps_out.append({"lap": r + 1, "n": int(m.sum()), "mean": float(a.mean()) if a.size else 0.0, "min": int(a.min()) if a.size else 0})
    return {"controllers": int(sel.sum()), "laps": laps_out, "unsolved_steps": int(unsolved[sel].sum()),
            "instances_with_flags": int((flags_or[sel] != 0).sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8192, help="instances per GPU")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps every instance has to finish")
    ap.add_argument("--max-steps", type=int, default=0, help="0 = 300 per lap")
    ap.add_argument("--mode", choices=["independent", "pooled"], default="pooled")
    ap.add_argument("--share", type=int, default=2, help="pooled mode: globally fastest laps handed to every instance per exchange")
    ap.add_argument("--tpad", type=int, default=288, help="rows per exchanged lap (lap + addPoint overrun)")
    ap.add_argument("--ship-after", type=int, default=40, help="pooled mode: steps into the next lap before a lap is shipped")
    ap.add_argument("--poll", type=int, default=8, help="closed-loop steps between progress polls")
    ap.add_argument("--warm", action="store_true", help="warm-started interior-point solves (lmpc_params.warm_start)")
    args = ap.parse_args()
    world, local = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    out = run(args.batch, args.laps, args.mode, args.share, args.tpad, args.ship_after, args.poll, args.max_steps, local=local, warm=args.warm)
    if (dist.get_rank() if dist.is_initialized() else 0) == 0:
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
