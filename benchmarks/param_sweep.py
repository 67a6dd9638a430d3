#!/usr/bin/env python
"""Parameter sweeps in one batch (lmpc_set_param_sets): what per-controller QP parameters cost, and a closed-loop tuning grid.

Leg 1, QP throughput: the configs[1] workload (4096 LTV-MPC QPs, N = 12) solved through the device entry point by three handles,
timed in alternating rounds in the same process (CUDA events, L2 flushed between timed launches as in bench.py):
  uniform   the handle's own parameters (ftocp_kernel<..., false>: parameters in the constant bank);
  one_set   the same parameters installed as the only set (ftocp_kernel<..., true>: the pure cost of the variant);
  sweep16   16 sets varying Qslack, dR, xRef[0] and the lane bound bx, interleaved over the batch.  The tunings take different
            numbers of interior-point iterations, so this arm is not a pure overhead figure.
Leg 2, closed-loop sweep: benchmarks/rollout_mc.run in independent mode with a 4 Qslack x 4 dR grid of LMPC tunings over the batch
(set = controller mod 16): per set, mean / minimum length of every LMPC lap, unsolved steps and controllers with health flags.

  python benchmarks/param_sweep.py [--rounds 3 --steps 20] [--batch2 8192 --laps 3] [--out FILE]
Prints one JSON line per leg (card name and power limit read in the same run); --out appends them to FILE as well."""
import argparse
import copy
import json
import os
import subprocess
import sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "benchmarks")):
    if p not in sys.path:
        sys.path.insert(0, p)
from racinglmpc_b200 import BatchedFTOCP, workloads, reference_params as rp      # noqa: E402
import rollout_mc                                                                  # noqa: E402


def card(dev):
    """Card name and enforced power limit (W) of the device, read now (every stated timing names its power limit)."""
    name, watts = torch.cuda.get_device_name(dev), None
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        watts = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return {"gpu": name, "power_limit_w": watts}


def mpc_sweep_sets(N, K=16):
    """K configs[1] tunings: lane-slack weight, input-rate weight, target speed and lane half-width on a 4 x 4 grid."""
    base = rp.mpc_params(N)
    sets = []
    for k in range(K):
        p = copy.deepcopy(base)
        p.Qslack = np.array([0.0, (25.0, 50.0, 100.0, 200.0)[k % 4]])
        p.dR = (0.0, 0.5, 1.0, 2.0)[(k // 4) % 4] * np.array([1.0, 10.0])
        p.xRef = np.array([(0.7, 0.8, 0.9, 1.0)[(k // 4) % 4], 0, 0, 0, 0, 0.0])
        p.bx = np.full(2, (1.6, 1.8, 2.0, 2.2)[k % 4])
        sets.append(p)
    return sets


def leg_qp(rounds, steps, warmup, dev):
    B, N = 4096, 12
    x0, uold, abc = workloads.ltv_mpc_batch(B, N=N)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_x0, d_u, d_abc = t(x0), t(uold), t(abc)
    sweep = mpc_sweep_sets(N)
    arms = {"uniform": None, "one_set": ([rp.mpc_params(N)], np.zeros(B, np.int32)),
            "sweep16": (sweep, np.arange(B) % len(sweep))}
    solvers, outs = {}, {}
    for name, ps in arms.items():
        s = BatchedFTOCP(rp.mpc_params(N), batch=B, device=dev)
        if ps is not None:
            s.set_param_sets(*ps)
        solvers[name] = s
        outs[name] = dict(xP=torch.zeros(B, N + 1, 6, dtype=torch.float64, device=dev), uP=torch.zeros(B, N, 2, dtype=torch.float64, device=dev),
                          st=torch.zeros(B, dtype=torch.int32, device=dev), it=torch.zeros(B, dtype=torch.int32, device=dev),
                          rs=torch.zeros(B, 3, dtype=torch.float64, device=dev))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)     # > 50 MB L2 of the H100

    def launch(name):
        o = outs[name]
        solvers[name].solve_dev(d_x0, d_u, d_abc, N * 54, 54, o["xP"], o["uP"], o["st"], o["it"], o["rs"])

    for name in arms:
        for _ in range(warmup):
            launch(name)
        solvers[name].sync()
    ms = {name: [] for name in arms}                  # per round: median ms per launch
    for _ in range(rounds):
        for name in arms:
            stream = torch.cuda.ExternalStream(solvers[name].stream, device=dev)
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
            with torch.cuda.stream(stream):
                for i in range(steps):
                    flush.zero_()
                    ev[i][0].record(stream)
                    launch(name)
                    ev[i][1].record(stream)
            solvers[name].sync()
            torch.cuda.synchronize()
            ms[name].append(float(np.median([a.elapsed_time(b) for a, b in ev])))
    res = {"benchmark": "param_sweep leg 1: configs[1] QP throughput, uniform vs per-controller parameters", **card(dev),
           "batch": B, "N": N, "rounds": rounds, "steps_per_round": steps, "l2": "flushed between timed launches (256 MiB memset)",
           "note": "sweep16 tunings take different interior-point iteration counts: not a pure overhead figure", "arms": {}}
    for name in arms:
        o, s = outs[name], solvers[name]
        its = o["it"].cpu().numpy()
        m = np.array(ms[name])
        res["arms"][name] = {"ms_per_launch_rounds": m.tolist(), "ms_per_launch_mean": float(m.mean()),
                             "solves_per_s": float(B / (m.mean() * 1e-3)), "ipm_iters_mean": float(its.mean()),
                             "ipm_iters_max": int(its.max()), "all_solved": bool((o["st"].cpu().numpy() == 1).all()),
                             "late_accepts": s.late_accepts, "kernel_launches": s.kernel_launches}
    ov = 100.0 * (np.array(ms["one_set"]) / np.array(ms["uniform"]) - 1.0)
    res["one_set_over_uniform_pct_rounds"] = ov.tolist()
    res["one_set_over_uniform_pct"] = {"mean": float(ov.mean()), "min": float(ov.min()), "max": float(ov.max())}
    for s in solvers.values():
        s.close()
    return res


def lmpc_grid(N=12):
    """4 x 4 LMPC tunings around the reference's (initControllerParameters.py:28-58): Qslack and dR scaled by 0.5 .. 4."""
    _, _, _, _, _, base = rp.lmpc_params(N)
    sets, labels = [], []
    for qs in (0.5, 1.0, 2.0, 4.0):
        for dr in (0.5, 1.0, 2.0, 4.0):
            p = copy.deepcopy(base)
            p.Qslack = qs * np.asarray(base.Qslack, float)
            p.dR = dr * np.asarray(base.dR, float)
            sets.append(p)
            labels.append({"Qslack": p.Qslack.tolist(), "dR": p.dR.tolist()})
    return sets, labels


def leg_closed_loop(batch, laps, warm, dev):
    sets, labels = lmpc_grid()
    idx = np.arange(batch) % len(sets)
    out = rollout_mc.run(batch=batch, laps=laps, mode="independent", local=dev, warm=warm, param_sets=(sets, idx, None))
    for s, lab in zip(out["per_set_rank0"], labels):
        s.update(lab)
    out.pop("benchmark")                              # rollout_mc's own label ("configs[3] ...") would overwrite this leg's
    return {"benchmark": "param_sweep leg 2: closed-loop LMPC tuning grid (4 Qslack x 4 dR), independent mode", **card(dev),
            "sets": len(sets), "controllers_per_set": batch // len(sets), **out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of leg 1")
    ap.add_argument("--steps", type=int, default=20, help="timed launches per arm and round")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch2", type=int, default=8192, help="controllers of leg 2 (16 sets interleaved)")
    ap.add_argument("--laps", type=int, default=3, help="LMPC laps every controller of leg 2 drives")
    ap.add_argument("--warm", action="store_true", help="leg 2 with warm-started interior-point solves")
    ap.add_argument("--legs", default="1,2")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args()
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    lines = []
    if "1" in args.legs.split(","):
        lines.append(leg_qp(args.rounds, args.steps, args.warmup, dev))
    if "2" in args.legs.split(","):
        lines.append(leg_closed_loop(args.batch2, args.laps, args.warm, dev))
    for r in lines:
        print(json.dumps(r), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
