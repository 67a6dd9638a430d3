"""QP inputs at any instantiated (N, M) for the GPU tests of the QP kernel: LTV-MPC QPs from the workload fixture and LMPC-type
QPs built around them from the PID lap of the reference golden file."""
import numpy as np

from racinglmpc_b200 import workloads


def ltv_inputs(B, N):
    """LTV-MPC inputs at any horizon <= 48: the first N stage models of the N = 48 fixture when N has no fixture of its own."""
    try:
        x0, uold, abc = workloads.ltv_mpc_batch(B, N=N)
        start = np.load(workloads._GOLD + "/workload_ltv.npz")["N%d_start" % N]
    except KeyError:
        x0, uold, abc = workloads.ltv_mpc_batch(B, N=48)
        abc = np.ascontiguousarray(abc[:, :N])
        start = np.load(workloads._GOLD + "/workload_ltv.npz")["N48_start"]
    return x0, uold, abc, start[np.arange(B) % start.shape[0]]


def lmpc_qp_inputs(gold, N, B, duplicate_laps, M=48):
    """LMPC-type QPs at horizon N: stage models from the LTV workload fixture, safe set = 4 x (M / 4) consecutive rows of the PID
    lap around the end of the prediction (4 identical laps when `duplicate_laps`: the reference's own first LMPC laps,
    main.py:109-110, the LP-degenerate case), cost-to-go counting down."""
    x0, uold, abc, start = ltv_inputs(B, N)
    xP, uP = gold["pid_x"], gold["pid_u"]
    P = M // 4
    SS = np.zeros((B, 6, M)); Qf = np.zeros((B, M)); SuS = np.zeros((B, 6, M)); SuU = np.zeros((B, 2, M))
    for b in range(B):
        i0 = int(min(start[b] + N - P // 2, xP.shape[0] - P - 12))
        for j in range(4):
            rows = np.arange(i0, i0 + P + 1) + (0 if duplicate_laps else 2 * j)
            blk = xP[rows].copy()
            if not duplicate_laps:
                blk[:, 0:3] += 1e-3 * (j + 1)
            SS[b, :, P * j:P * j + P] = blk[:P].T
            SuS[b, :, P * j:P * j + P] = blk[1:].T
            SuU[b, :, P * j:P * j + P] = uP[rows[1:]].T
            Qf[b, P * j:P * j + P] = 300.0 - rows[:P] * 0.3 + 5.0 * j
    return x0, uold, abc, SS, Qf, SuS, SuU


def perturbed_ltv_inputs(B, N, seed):
    """LTV-MPC QPs far from the workload's operating point: the fixture's models with the car up to 3 m off the centre line
    (the lane half-width is 2), up to 1 m/s off in speed, and the previous input anywhere inside its bounds.  A few of these take
    the solver's rare branches (recentring passes), which the workload QPs do not."""
    x0, uold, abc, _ = ltv_inputs(B, N)
    rng = np.random.default_rng(seed)
    x0 = x0.copy()
    x0[:, 5] += rng.uniform(-3, 3, B)
    x0[:, 0] += rng.uniform(-1, 1, B)
    uold = np.ascontiguousarray(np.stack([rng.uniform(-0.49, 0.49, B), rng.uniform(-9.9, 9.9, B)], axis=1))
    return x0, uold, abc


def perturbed_lmpc_inputs(gold, N, B, seed, M=48):
    """LMPC-type QPs (lmpc_qp_inputs, distinct laps) with the state and previous input perturbed as in perturbed_ltv_inputs.
    Returns x0, uold, abc, SS, Qf."""
    x0, uold, abc, SS, Qf, _, _ = lmpc_qp_inputs(gold, N, B, False, M)
    rng = np.random.default_rng(seed)
    x0 = x0.copy()
    x0[:, 5] += rng.uniform(-3, 3, B)
    x0[:, 0] += rng.uniform(-1, 1, B)
    uold = np.ascontiguousarray(np.stack([rng.uniform(-0.49, 0.49, B), rng.uniform(-9.9, 9.9, B)], axis=1))
    return x0, uold, abc, SS, Qf
