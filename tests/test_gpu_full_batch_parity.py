"""GPU tier: EVERY instance of the BASELINE.json workloads against the oracle (not a sample), and the solver
instantiations the sampled tests did not reach (the reference's own horizon N = 14, LMPC-type QPs at N = 24 / 48).

Oracle side (tests/support/oracle_batch.py): the reference's assembly / regression / selection restated in oracle/, run for
all instances in a process pool, and the OSQP-algorithm C port driven to 1e-9 (OpenMP over the batch).  On the degenerate
LMPC QPs the first-order oracle itself does not always reach 1e-9 (SURVEY App. A: thousands of ADMM iterations, failed
polish); parity of the primal solution is asserted wherever the ORACLE certifies its own answer (residuals <= 1e-8 and
polished), and every instance -- converged oracle or not -- must satisfy the solver-independent KKT conditions of the
reference-assembled QP (oracle/kkt.py) to 1e-6 and must not have a worse objective than the oracle's point.
Tolerances: |dz| <= 1e-6 (north_star), K1 model rows <= 1e-9, K2 selection bit-exact."""
import multiprocessing as mp

import numpy as np
import pytest
import torch

# the worker pools fork on purpose (the workload is shared copy-on-write; the children never touch CUDA or threads)
pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:This process .* is multi-threaded:DeprecationWarning")]

from racinglmpc_b200 import BatchedFTOCP, pack_abc, workloads, reference_params as rp   # noqa: E402
from racinglmpc_b200.controller import BatchedController                                 # noqa: E402
from oracle import ftocp, kkt                                                            # noqa: E402
import oracle_batch as ob                                                                # noqa: E402
from qp_inputs import ltv_inputs, lmpc_qp_inputs                                         # noqa: E402


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _certified(infos, tol=1e-8):
    return np.array([i["status"] == 1 and i["polished"] == 1 and max(i["pri_res"], i["dua_res"]) <= tol for i in infos])


_KKT_CTX = {}


def _kkt_one(b):
    prob, z = _KKT_CTX["prob"], _KKT_CTX["z"]
    patP, patA, Px, q, Ax, l, u = prob
    n, m = q.shape[1], l.shape[1]
    P = np.zeros((n, n)); A = np.zeros((m, n))
    (Pp, Pi), (Ap, Ai) = patP, patA
    cols = np.repeat(np.arange(n), np.diff(Pp)); P[Pi, cols] = Px[b]; P = np.triu(P) + np.triu(P, 1).T
    cols = np.repeat(np.arange(n), np.diff(Ap)); A[Ai, cols] = Ax[b]
    y = kkt.dual_from_primal(P, q[b], A, l[b], u[b], z[b], tol=1e-6)
    r = kkt.residuals(P, q[b], A, l[b], u[b], z[b], y)
    return r["r_prim"], r["r_dual"], kkt.objective(P, q[b], z[b]), kkt.objective(P, q[b], _KKT_CTX["zo"][b])


def _kkt_all(prob, z, zo):
    """Solver-independent KKT residuals of every GPU solution against the reference-assembled QP, in a process pool."""
    _KKT_CTX.update(prob=prob, z=z, zo=zo)
    B = z.shape[0]
    nproc = min(ob.host_threads(), 64)
    if nproc > 1 and B >= 4 * nproc:
        with mp.get_context("fork").Pool(nproc) as pool:
            res = pool.map(_kkt_one, range(B), chunksize=max(1, B // (8 * nproc)))
    else:
        res = [_kkt_one(b) for b in range(B)]
    _KKT_CTX.clear()
    return np.array(res)


def test_config1_all_4096_instances_vs_oracle():
    """BASELINE configs[1]: all 4096 LTV-MPC QPs (126 vars / 174 rows) against the oracle optimum."""
    _need_gpu()
    B, N = 4096, 12
    x0, uold, abc = workloads.ltv_mpc_batch(B, N=N)
    prob = ob.ltv_problem_set(x0, uold, abc, N)
    zo, infos = ob.tight_batch(prob)
    ok = _certified(infos)
    assert ok.all(), "oracle failed on %d of %d MPC-type QPs" % ((~ok).sum(), B)
    s = BatchedFTOCP(rp.mpc_params(N), batch=B)
    o = s.solve(x0, uold, abc)
    assert np.all(o["status"] == 1), np.unique(o["status"], return_counts=True)
    assert o["resid"].max() <= 1.000001e-9
    assert s.late_accepts == 0                      # nobody came in through the 1e-6 safety net
    n = 6 * (N + 1)
    ex = np.abs(o["xPred"].reshape(B, -1) - zo[:, :n]).max(axis=1)
    eu = np.abs(o["uPred"].reshape(B, -1) - zo[:, n:n + 2 * N]).max(axis=1)
    es = np.abs(o["slack"] - zo[:, n + 2 * N:n + 4 * N]).max(axis=1)
    assert ex.max() < 1e-6 and eu.max() < 1e-6 and es.max() < 1e-6, (ex.max(), eu.max(), es.max(), int(ex.argmax()))
    s.close()


def test_config2_all_4096_instances_vs_oracle(track):
    """BASELINE configs[2]: all 4096 full LMPC steps: K1 model, K2 selection and the QP solution of every instance."""
    _need_gpu()
    B, N = 4096, 12
    data = workloads.lmpc_batch(B)
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, B, track.seg_table(), track.TrackLength, trToUse=5, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1280, ss_cap=5, model_cap=5)
    workloads.restore_lmpc_batch(c, data)
    o = c.step(data["x0"])
    assert np.all(o["status"] == 1) and np.all(o["flags"] == 0), (np.unique(o["status"], return_counts=True), np.unique(o["flags"]))
    assert o["resid"].max() <= 1.000001e-9
    assert c.late_accepts == 0
    M = numSS_Points
    abc = c.read_buffer("abc", 0, (B, N, 54))
    sel = {k: c.read_buffer(k, 0, shp) for k, shp in (("SS_sel", (B, 6, M)), ("Qfun_sel", (B, M)), ("Succ_SS", (B, 6, M)),
                                                       ("Succ_uSS", (B, 2, M)))}
    slack = c.read_buffer("slack", 0, (B, 2 * N))
    xi = c.read_buffer("slackT", 0, (B, 6))
    c.close()

    orc = ob.lmpc_oracle_steps(data, track, N=N, trToUse=5)
    # ---- K1: regression rows to 1e-9, closed-form rows to 1e-13 (sin/cos last ulp)
    d = np.abs(abc - orc["abc"])
    assert d.max() < 1e-9, (d.max(), np.unravel_index(d.argmax(), d.shape))
    A_gpu, A_or = abc[:, :, 0:36].reshape(B, N, 6, 6), orc["abc"][:, :, 0:36].reshape(B, N, 6, 6)
    assert np.abs(A_gpu[:, :, 3:, :] - A_or[:, :, 3:, :]).max() < 1e-13
    # ---- K2: bit-exact
    for k in ("SS_sel", "Qfun_sel", "Succ_SS", "Succ_uSS"):
        assert np.array_equal(sel[k], orc[k]), k
    # ---- QP: optimum where the oracle certifies its own answer; KKT + objective everywhere
    zo, infos = ob.tight_batch(orc["prob"])
    ok = _certified(infos)
    assert ok.mean() > 0.5, "the oracle certifies only %.1f %% of the LMPC QPs" % (100 * ok.mean())
    z = np.concatenate([o["xPred"].reshape(B, -1), o["uPred"].reshape(B, -1), slack, o["lambd"], xi], axis=1)
    n = 6 * (N + 1)
    err = np.abs(z[:, :n + 2 * N] - zo[:, :n + 2 * N]).max(axis=1)
    assert err[ok].max() < 1e-6, (err[ok].max(), int(np.where(ok)[0][err[ok].argmax()]))
    r = _kkt_all(orc["prob"], z, zo)
    assert r[:, 0].max() < 1e-6 and r[:, 1].max() < 1e-6, (r[:, 0].max(), r[:, 1].max(), int(r[:, 1].argmax()))
    # same objective as the oracle's certified optimum (both points are feasible only to their residuals, and the multipliers
    # are O(1e3): 1e-9 of the objective + 1e-6).  Uncertified oracle points are infeasible by up to 1e-4 and say nothing.
    gap = np.abs(r[:, 2] - r[:, 3])
    assert np.all(gap[ok] <= 1e-9 * np.abs(r[ok, 3]) + 1e-6), (gap[ok].max(), np.abs(r[ok, 3]).max())
    print("configs[2]: oracle certified %d / %d; max |dz| on those %.2e; KKT max %.2e / %.2e over all" %
          (ok.sum(), B, err[ok].max(), r[:, 0].max(), r[:, 1].max()))


@pytest.mark.parametrize("N,dup,M", [(14, False, 48), (14, True, 48), (24, False, 48), (48, False, 48), (6, True, 48), (4, False, 48),
                                     (16, False, 48), (32, False, 48), (12, False, 24), (12, True, 96), (14, False, 64), (14, False, 32)])
def test_lmpc_qp_instantiations_vs_oracle(gold, track, N, dup, M):
    """ftocp_kernel<N,48> for the reference's own horizon (main.py:43: N = 14) and the sweep horizons, LMPC-type QPs
    (180 + 9 (N - 12) variables) against the oracle on the reference-assembled matrices."""
    _need_gpu()
    B = 16
    numSS_it, _, _, _, Qts, par = rp.lmpc_params(N)
    numSS_Points = M
    x0, uold, abc, SS, Qf, SuS, SuU = lmpc_qp_inputs(gold, N, B, dup, M)
    s = BatchedFTOCP(par, batch=B, numSS_Points=numSS_Points, numSS_it=numSS_it, QterminalSlack=Qts)
    o = s.solve(x0, uold, abc, SS, Qf, SuS, SuU)
    counts = dict(zip(*np.unique(o["status"], return_counts=True)))
    assert counts.get(1, 0) == B, counts
    assert s.late_accepts == 0
    _, _, _, _, oQts, opar = ftocp.lmpc_params(track, N)
    opar.timeVarying = True
    F, bb = ftocp.build_ineq(opar)
    Ps, qs, As, ls, us = [], [], [], [], []
    for b in range(B):
        A = abc[b][:, 0:36].reshape(N, 6, 6); Bm = abc[b][:, 36:48].reshape(N, 6, 2); C = abc[b][:, 48:54]
        H, q = ftocp.build_cost(opar, uold[b])
        G, E, L = ftocp.build_eq(opar, list(A), list(Bm), list(C))
        F2, b2, G2, E2, L2, H2, q2 = ftocp.add_safe_set(F, bb, G, E, L, H, q, 6, N, SS[b], Qf[b], oQts)
        P, q, Am, l, u = ftocp.osqp_form(H2, q2, F2, b2, G2, E2 @ x0[b] + L2)
        Ps.append(P); qs.append(q); As.append(Am); ls.append(l); us.append(u)
    prob = ob._stack_problems(Ps, qs, As, ls, us)
    zo, infos = ob.tight_batch(prob)
    ok = _certified(infos)
    z = np.concatenate([o["xPred"].reshape(B, -1), o["uPred"].reshape(B, -1), o["slack"], o["lambd"], o["slackTerminal"]], axis=1)
    n = 6 * (N + 1) + 2 * N
    if ok.any():
        assert np.abs(z[ok, :n] - zo[ok, :n]).max() < 1e-6, np.abs(z[ok, :n] - zo[ok, :n]).max()
    r = _kkt_all(prob, z, zo)
    assert r[:, 0].max() < 1e-6 and r[:, 1].max() < 1e-6, r[:, :2].max(axis=0)
    assert np.all(np.abs(r[:, 2] - r[:, 3])[ok] <= 1e-9 * np.abs(r[ok, 3]) + 1e-6)
    # zt = Succ_SS lam, zt_u = Succ_uSS lam (PC.py:382-384)
    assert np.abs(o["zt"] - np.einsum("bij,bj->bi", SuS, o["lambd"])).max() < 1e-12
    assert np.abs(o["zt_u"] - np.einsum("bij,bj->bi", SuU, o["lambd"])).max() < 1e-12
    s.close()


@pytest.mark.parametrize("N", [14, 4, 8, 10, 16, 20, 32])
def test_mpc_qp_horizon_grid_vs_oracle(N):
    """ftocp_kernel<N,0> over the instantiated horizon grid (14 = the reference's own, main.py:43): LTV-MPC QPs, all instances
    against the oracle."""
    _need_gpu()
    B = 64
    x0, uold, abc, _ = ltv_inputs(B, N)
    prob = ob.ltv_problem_set(x0, uold, abc, N)
    zo, infos = ob.tight_batch(prob)
    assert _certified(infos).all()
    s = BatchedFTOCP(rp.mpc_params(N), batch=B)
    o = s.solve(x0, uold, abc)
    assert np.all(o["status"] == 1) and s.late_accepts == 0
    n = 6 * (N + 1)
    assert np.abs(o["xPred"].reshape(B, -1) - zo[:, :n]).max() < 1e-6
    assert np.abs(o["uPred"].reshape(B, -1) - zo[:, n:n + 2 * N]).max() < 1e-6
    s.close()
