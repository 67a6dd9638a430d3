#!/usr/bin/env python
"""Generate tests/golden/warm_sequences.npz — sequences of consecutive QPs for the warm-start tests (tests/test_warm_start.py).

A warm-started solve starts from the previous solve of the same controller, so its QPs must come in the order a controller meets
them.  Every prediction a sequence follows is the ORACLE's optimum (oracle/osqp_port.py tight_qp), stored with the QP, so the
sequences do not depend on the kernel under test.

  MPC type, N in {6, 12, 24, 48}: the LTV model of workload_ltv.npz start c (held fixed along chain c), STEPS QPs per chain;
    x0 of QP k+1 is x[1] of QP k's optimum plus noise at the workloads' scale (np.random.default_rng(SEED + N); the LMPC sequence's vehicle noise from default_rng(SEED)), OldInput its u[0].
    Chains with JUMP add a jump in (vx, vy, wz, epsi, ey) every JUMP_EVERY steps: a record of the previous QP is then a poor
    start, and a warm-started solve runs into its restart.
  A hard pair, N = 48: chains that leave the fitted region (x0 following the optimum of a fixed, unstable model, noise from
    np.random.default_rng(0)) reach QPs whose cold solve needs 30+ interior-point iterations.  HARD names one (chain, step),
    found by solving these chains with the kernel's host emulation: the QP before it and the QP itself are stored.  A record
    taken on the first is a poor start for the second, so its warm start restarts cold.
  LMPC type, N = 12, M = 48: the oracle controller of reference_golden.npz's snapshot (lap 4, step 200), driven by the oracle
    vehicle (oracle/vehicle.py dyn_model) for LMPC_STEPS steps through the finish line: s drops by TrackLength there (as the
    reference's next lap starts from xF) and the selected safe set changes wholesale.
"""
import os
import sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests", "support")]
from oracle import ftocp, osqp_port, vehicle      # noqa: E402
from oracle.track import TrackTable              # noqa: E402
import replay                                    # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
SEED = 7
CHAINS, STEPS, JUMP_EVERY = 6, 30, 8
NOISE = 0.01 * np.array([1.0, 0.1, 0.1, 0.01, 1.0, 0.05])
JUMP = np.array([0.5, 0.2, 0.2, 0.1, 0.0, 0.5])
BOUND = 20.0
LMPC_KEY, LMPC_STEPS = (4, 200), 36


def mpc_chain(N, w, i, ltv, jumps, rng):
    """One chain on the model of workload start i, or None when the state leaves the region the model was fitted on."""
    F, bb = ftocp.build_ineq(ltv)
    abc = w["N%d_abc" % N][i]
    A = abc[:, 0:36].reshape(N, 6, 6); B = abc[:, 36:48].reshape(N, 6, 2); C = abc[:, 48:54]
    G, E, L = ftocp.build_eq(ltv, list(A), list(B), list(C))
    x0, uo = w["N%d_x0" % N][i].copy(), w["N%d_uold" % N][i].copy()
    X0, UO, UOP = np.zeros((STEPS, 6)), np.zeros((STEPS, 2)), np.zeros((STEPS, N, 2))
    for k in range(STEPS):
        if np.abs(x0[[0, 1, 2, 3, 5]]).max() > BOUND:
            return None
        H, q = ftocp.build_cost(ltv, uo)
        P, q, Am, l, u = ftocp.osqp_form(H, q, F, bb, G, E @ x0 + L)
        z, info = osqp_port.tight_qp(P, q, Am, l, u)
        assert info["status"] == 1, (N, i, k)
        X0[k], UO[k], UOP[k] = x0, uo, z[6 * (N + 1):6 * (N + 1) + 2 * N].reshape(N, 2)
        x0 = z[6:12] + NOISE * rng.standard_normal(6)
        if jumps and k % JUMP_EVERY == JUMP_EVERY - 1:
            x0 = x0 + JUMP * rng.choice([-1.0, 1.0])
        uo = UOP[k, 0].copy()
    return X0, UO, UOP


def mpc_chains(N, rng, out):
    """CHAINS chains on the first workload starts whose chains stay bounded; odd chains jump."""
    w = np.load(os.path.join(OUT, "workload_ltv.npz"))
    _, ltv = ftocp.mpc_params(6, 2, N, 0.8)
    ltv.timeVarying = True
    rows, starts = [], []
    for i in range(w["N%d_x0" % N].shape[0]):
        r = mpc_chain(N, w, i, ltv, len(rows) % 2 == 1, rng)
        if r is not None:
            rows.append(r); starts.append(i)
        if len(rows) == CHAINS:
            break
    out.update({"N%d_start" % N: np.array(starts), "N%d_x0" % N: np.stack([r[0] for r in rows]),
                "N%d_uold" % N: np.stack([r[1] for r in rows]), "N%d_uopt" % N: np.stack([r[2] for r in rows])})


HARD = {48: (7, 22)}


def hard_pairs(out):
    w = np.load(os.path.join(OUT, "workload_ltv.npz"))
    rng = np.random.default_rng(0)
    for N in HARD:
        _, ltv = ftocp.mpc_params(6, 2, N, 0.8)
        ltv.timeVarying = True
        F, bb = ftocp.build_ineq(ltv)
        for b in range(HARD[N][0] + 1):
            abc = w["N%d_abc" % N][b]
            A = abc[:, 0:36].reshape(N, 6, 6); B = abc[:, 36:48].reshape(N, 6, 2); C = abc[:, 48:54]
            G, E, L = ftocp.build_eq(ltv, list(A), list(B), list(C))
            x0, uo = w["N%d_x0" % N][b].copy(), w["N%d_uold" % N][b].copy()
            rows = []
            for k in range(HARD[N][1] + 1):
                H, q = ftocp.build_cost(ltv, uo)
                P, q, Am, l, u = ftocp.osqp_form(H, q, F, bb, G, E @ x0 + L)
                z, info = osqp_port.tight_qp(P, q, Am, l, u)
                rows.append((x0, uo, z[6 * (N + 1):6 * (N + 1) + 2 * N].reshape(N, 2)))
                x0 = z[6:12] + 0.01 * rng.standard_normal(6) * np.array([1, .1, .1, .01, 1, .05])
                uo = rows[-1][2][0].copy()
            if b == HARD[N][0]:
                assert info["status"] == 1
                out.update({"hard%d_start" % N: np.int64(b), "hard%d_x0" % N: np.stack([r[0] for r in rows[-2:]]),
                            "hard%d_uold" % N: np.stack([r[1] for r in rows[-2:]]), "hard%d_uopt" % N: rows[-1][2]})


def lmpc_sequence(rng, out):
    g = np.load(os.path.join(OUT, "reference_golden.npz"))
    trk = TrackTable(0.4)
    c, x = replay.lmpc_from_snapshot(g, LMPC_KEY, trk)
    xg = np.zeros(6)
    rows = {k: [] for k in ("abc", "x0", "uold", "SS", "Qfun", "uopt")}
    for k in range(LMPC_STEPS):
        uold = np.asarray(c.OldInput, float).ravel().copy()
        c.solve(x)
        assert c.last_info is None or c.last_info.get("status", 1) == 1, k
        abc = np.concatenate([np.asarray(c.A).reshape(12, 36), np.asarray(c.B).reshape(12, 12), np.asarray(c.C).reshape(12, 6)], axis=1)
        for key, v in (("abc", abc), ("x0", x), ("uold", uold), ("SS", c.SS_PointSelectedTot), ("Qfun", c.Qfun_SelectedTot),
                       ("uopt", c.uPred)):
            rows[key].append(np.array(v, float))
        u = c.uPred[0].copy()
        c.addPoint(x, u)
        x, xg = vehicle.dyn_model(trk, x, xg, u, rng=rng)
        if x[4] > trk.TrackLength:                 # the next lap starts from xF (SysModel.py:51, main.py)
            x = x - np.array([0, 0, 0, 0, trk.TrackLength, 0])
    out.update({"lmpc_" + k: np.stack(v) for k, v in rows.items()})
    out["lmpc_track_length"] = np.float64(trk.TrackLength)


def main():
    out = {}
    for N in (6, 12, 24, 48):
        mpc_chains(N, np.random.default_rng(SEED + N), out)
    hard_pairs(out)
    lmpc_sequence(np.random.default_rng(SEED), out)
    np.savez_compressed(os.path.join(OUT, "warm_sequences.npz"), **out)
    print("wrote", os.path.join(OUT, "warm_sequences.npz"), sorted(out))


if __name__ == "__main__":
    main()
