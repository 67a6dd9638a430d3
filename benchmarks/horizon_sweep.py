#!/usr/bin/env python
"""BASELINE.json configs[4]: horizon sweep N in {6,12,24,48}, batch=16384 LTV-MPC QPs on one H100.

Reports, per horizon: solves/s (device-resident inputs, CUDA events on the launching stream), interior-point
iterations to (r_prim, r_dual <= 1e-8, gap <= 1e-11) and, on a 64-instance sample, the iterations the OSQP-algorithm
oracle needs for eps 1e-6 (unpolished ADMM, the reference's algorithm) next to it.  Writes one JSON line per horizon."""
import json
import os
import sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from racinglmpc_b200 import BatchedFTOCP, workloads, reference_params as rp   # noqa: E402


def oracle_iters(N, x0, uold, abc, nsample=64):
    from oracle import ftocp, osqp_port
    par = ftocp.mpc_params(6, 2, N, 0.8)[1]
    par.timeVarying = True
    F, bb = ftocp.build_ineq(par)
    its = []
    for b in range(nsample):
        A = abc[b][:, 0:36].reshape(N, 6, 6); B = abc[b][:, 36:48].reshape(N, 6, 2); C = abc[b][:, 48:54]
        H, q = ftocp.build_cost(par, uold[b]); G, E, L = ftocp.build_eq(par, list(A), list(B), list(C))
        P, q, Am, l, u = ftocp.osqp_form(H, q, F, bb, G, E @ x0[b] + L)
        _, info, _ = osqp_port.solve(P, q, Am, l, u, eps_abs=1e-6, eps_rel=1e-6, polish=0, max_iter=100000)
        its.append(info["iters"])
    return float(np.mean(its)), int(np.max(its))


def main():
    B = int(os.environ.get("SWEEP_BATCH", "16384"))
    dev = torch.device("cuda", 0)
    for N in [int(v) for v in os.environ.get("SWEEP_N", "6,12,24,48").split(",")]:
        x0, uold, abc = workloads.ltv_mpc_batch(B, N=N)
        s = BatchedFTOCP(rp.mpc_params(N), batch=B)
        stream = torch.cuda.ExternalStream(s.stream, device=dev)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        d = [t(x0), t(uold), t(abc)]
        xP = torch.zeros(B, N + 1, 6, dtype=torch.float64, device=dev); uP = torch.zeros(B, N, 2, dtype=torch.float64, device=dev)
        st = torch.zeros(B, dtype=torch.int32, device=dev); it = torch.zeros(B, dtype=torch.int32, device=dev)
        rs = torch.zeros(B, 3, dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        run = lambda: s.solve_dev(d[0], d[1], d[2], N * 54, 54, xP, uP, st, it, rs)
        for _ in range(3):
            run()
        s.sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record(stream)
            for _ in range(5):
                run()
            e1.record(stream)
        s.sync()
        ms = e0.elapsed_time(e1) / 5
        iters = it.cpu().numpy(); status = st.cpu().numpy(); resid = rs.cpu().numpy()
        om, ox = (0.0, 0) if os.environ.get("SWEEP_NO_ORACLE") else oracle_iters(N, x0, uold, abc)
        print(json.dumps({"N": N, "batch": B, "ms_per_launch": ms, "solves_per_s": B / (ms * 1e-3),
                          "solved_fraction": float(np.mean(status == 1)), "ipm_iters_mean": float(iters.mean()),
                          "ipm_iters_max": int(iters.max()), "max_resid": float(resid.max()),
                          "oracle_admm_iters_to_1e-6_mean": om, "oracle_admm_iters_to_1e-6_max": ox}))
        s.close()


if __name__ == "__main__":
    main()
