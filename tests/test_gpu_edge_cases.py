"""GPU tier: edge cases of the hot path against the oracle's restatement of the reference
(PredictiveModel.computeIndices PM.py:180-197, LMPC.selectPoints PC.py:478-514) and the error behaviour of the C ABI.

The reference has no tests of its own (SURVEY §4); these are the cases its code branches on:
few / one neighbour (exact distance ties inside one lap are implementation-defined in the reference: np.argsort's default
sort is not stable; the kernel takes the lowest rows), laps of assorted lengths, the two selection-window rules, the window
running off a lap (the reference: IndexError), a full lap pool, unsupported sizes and null arguments."""
import ctypes as C
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import BatchedFTOCP, _native as nat, reference_params as rp   # noqa: E402
from racinglmpc_b200.controller import BatchedController                             # noqa: E402
from oracle import ftocp, ltv_model                                                   # noqa: E402


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _abc_split(abc_b, N):
    return abc_b[:, 0:36].reshape(N, 6, 6), abc_b[:, 36:48].reshape(N, 6, 2), abc_b[:, 48:54]


def _model_controller(track, laps, xLin, uLin, N=12, trToUse=1):
    """B = 1 LTV-MPC controller whose regression model holds `laps`; linearisation points xLin[N+1,6], uLin[N,2]."""
    par = rp.mpc_params(N)
    c = BatchedController(par, 1, track.seg_table(), track.TrackLength, trToUse=trToUse, Tmax=1536, model_cap=trToUse + 1)
    for x, u in laps:
        c.model_add_trajectory(0, x, u)
    c.set_state(xLin=xLin[None], uLin=uLin[None], OldInput=np.zeros((1, 2)), timeStep=[0])
    return c


def _random_lap(rng, T):
    x = np.zeros((T, 6))
    x[:, 0] = 0.8 + 0.3 * rng.standard_normal(T)
    x[:, 1] = 0.05 * rng.standard_normal(T)
    x[:, 2] = 0.3 * rng.standard_normal(T)
    x[:, 3] = 0.05 * rng.standard_normal(T)
    x[:, 4] = np.linspace(0.0, 18.0, T)
    x[:, 5] = 0.05 * rng.standard_normal(T)
    u = np.stack([0.2 * rng.standard_normal(T), 0.5 * rng.standard_normal(T)], axis=1)
    return x, u


def _oracle_abc(track, laps, xLin, uLin, N, trToUse):
    m = ltv_model.LocalLTVModel(6, 2, track, trToUse)
    for x, u in laps:
        m.addTrajectory(x, u)
    out = [m.regressionAndLinearization(xLin[i], uLin[i]) for i in range(N)]
    return np.array([o[0] for o in out]), np.array([o[1] for o in out]), np.array([o[2] for o in out])


@pytest.mark.parametrize("T", [40, 256, 257, 258, 513, 1000])
def test_k1_lap_lengths_across_tile_boundaries(track, T):
    """Rows 0..T-2 are candidates (PM.py:183) on random laps; the tile-edge lengths of the scan (LMPC_K1_TILE) are the
    parametrisation of test_gpu_knn_regression.py."""
    _need_gpu()
    rng = np.random.default_rng(T)
    N = 12
    lap = _random_lap(rng, T)
    idx = rng.integers(0, T - 1, N + 1)
    xLin = lap[0][idx] + 0.01 * rng.standard_normal((N + 1, 6))
    uLin = lap[1][idx[:N]] + 0.01 * rng.standard_normal((N, 2))
    c = _model_controller(track, [lap], xLin, uLin)
    abc, flags = c.identify()
    c.close()
    assert flags[0] == 0
    A, B, Cc = _abc_split(abc[0], N)
    oA, oB, oC = _oracle_abc(track, [lap], xLin, uLin, N, 1)
    assert np.max(np.abs(A - oA)) < 1e-8 and np.max(np.abs(B - oB)) < 1e-8 and np.max(np.abs(Cc - oC)) < 1e-8


def test_k1_fewer_neighbours_than_maxnumpoint_and_the_raising_cases(track):
    """PM.py:187-191: with fewer than MaxNumPoint rows inside the bandwidth h all of them are used.  One neighbour makes the
    reference raise (np.squeeze) -> flag 4."""
    _need_gpu()
    rng = np.random.default_rng(11)
    N, T = 12, 300
    x, u = _random_lap(rng, T)
    x[:, 1] += 100.0                              # everything far away in vy (scaling 1, h = 5) ...
    near = [20, 90, 150, 151, 220, 260]           # ... except six rows
    x[near, 1] -= 100.0
    q = x[150].copy()
    xLin = np.tile(q, (N + 1, 1)); uLin = np.tile(u[150], (N, 1))
    c = _model_controller(track, [(x, u)], xLin, uLin)
    abc, flags = c.identify()
    c.close()
    assert flags[0] == 0
    A, B, Cc = _abc_split(abc[0], N)
    oA, oB, oC = _oracle_abc(track, [(x, u)], xLin, uLin, N, 1)
    assert np.max(np.abs(A - oA)) < 1e-7 and np.max(np.abs(B - oB)) < 1e-7 and np.max(np.abs(Cc - oC)) < 1e-7
    # one neighbour
    x1 = x.copy(); x1[[20, 90, 151, 220, 260], 1] += 100.0
    c = _model_controller(track, [(x1, u)], xLin, uLin)
    _, flags = c.identify()
    c.close()
    assert flags[0] & 4


def _lmpc_controller(track, laps, N=12, ss_cap=6):
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, 1, track.seg_table(), track.TrackLength, trToUse=1, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=1536, ss_cap=ss_cap, model_cap=2)
    for x, u in laps:
        c.add_trajectory(0, x, u)
    return c, numSS_it, numSS_Points


def _oracle_lmpc(track, laps, zt, N=12):
    numSS_it, numSS_Points, _, _, Qts, par = ftocp.lmpc_params(track, N)
    par.timeVarying = False
    par.A, par.B = np.eye(6), np.zeros((6, 2))
    m = ltv_model.LocalLTVModel(6, 2, track, 1)
    o = ftocp.OracleLMPC(numSS_Points, numSS_it, Qts, par, m, qp=None)
    for x, u in laps:
        o.addTrajectory(x, u, x)
    o.zt = zt.copy()
    o.xLin = np.zeros((N + 1, 6))
    return o


def test_k2_window_rules_and_first_minimum(track):
    """PC.py:486-495: the window is [Min-6, Min+6] when Min - 6.5 >= 0, else [Min, Min+12]; np.argmin returns the FIRST
    minimum (two identical rows in the lap)."""
    _need_gpu()
    rng = np.random.default_rng(3)
    laps = []
    for j in range(4):
        x, u = _random_lap(rng, 120 + 10 * j)
        x[:, 4] = np.linspace(0.0, 19.5, x.shape[0])      # crosses the finish line: computeCost has something to count
        laps.append((x, u))
    laps[2][0][70] = laps[2][0][40]                        # duplicate row: the first one must win
    for zt_row, lapno in ((3, 0), (6, 1), (7, 3), (40, 2), (100, 0)):
        zt = laps[lapno][0][zt_row].copy()
        c, numSS_it, numSS_Points = _lmpc_controller(track, laps)
        c.set_state(xLin=np.zeros((1, 13, 6)), uLin=np.zeros((1, 12, 2)), zt=zt[None], OldInput=np.zeros((1, 2)), timeStep=[0],
                    has_pred=[0])
        x0 = np.array([0.8, 0, 0, 0, zt[4], 0.0])
        sel = c.select(x0[None])
        c.close()
        o = _oracle_lmpc(track, laps, zt)
        o.terminal_components(x0)
        assert sel["flags"][0] == 0
        assert np.array_equal(sel["SS_sel"][0], o.SS_PointSelectedTot), (zt_row, lapno)
        assert np.array_equal(sel["Qfun_sel"][0], o.Qfun_SelectedTot)
        assert np.array_equal(sel["Succ_SS"][0], o.Succ_SS_PointSelectedTot)
        assert np.array_equal(sel["Succ_uSS"][0], o.Succ_uSS_PointSelectedTot)
        order = np.argsort(np.array(o.LapTime), kind="stable")[:numSS_it]
        assert [int(m) for m in sel["min_index"][0]] == [i_min for (_, i_min, _) in o.last_sel_index]
        assert list(order) == [lap for (lap, _, _) in o.last_sel_index]


def test_k2_window_past_the_lap_end_is_flagged(track):
    """The reference indexes past the array (IndexError, PC.py:497) when the nearest point is within 6 rows of a lap's end
    and addPoint has not grown it; the kernel reports bit 8 and leaves the selection of that lap untouched."""
    _need_gpu()
    rng = np.random.default_rng(4)
    laps = [_random_lap(rng, 100) for _ in range(4)]
    zt = laps[1][0][97].copy()
    c, _, _ = _lmpc_controller(track, laps)
    c.set_state(xLin=np.zeros((1, 13, 6)), uLin=np.zeros((1, 12, 2)), zt=zt[None], OldInput=np.zeros((1, 2)), timeStep=[0], has_pred=[0])
    sel = c.select(np.array([[0.8, 0, 0, 0, zt[4], 0.0]]))
    c.close()
    assert sel["flags"][0] & 8
    with pytest.raises(IndexError):
        o = _oracle_lmpc(track, laps, zt)
        o.terminal_components(np.array([0.8, 0, 0, 0, zt[4], 0.0]))


def test_add_point_on_a_full_lap_is_flagged(track):
    _need_gpu()
    rng = np.random.default_rng(6)
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(12)
    c = BatchedController(par, 1, track.seg_table(), track.TrackLength, trToUse=1, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=64, ss_cap=5, model_cap=2)
    for _ in range(4):
        c.add_trajectory(0, *_random_lap(rng, 63))
    c.add_point(np.zeros(6), np.zeros(2))              # row 64 of 64: fits
    assert c.get_lap(0, 3)[0].shape[0] == 64
    # no room: LMPC.addPoint would np.append (PC.py:466-476); the fixed pool must not drop the point silently: the host
    # entry reports it (the device-resident rollout accumulates flag bit 16 in its health record instead)
    with pytest.raises(nat.NativeError, match="Tmax"):
        c.add_point(np.zeros(6), np.zeros(2))
    assert c.get_lap(0, 3)[0].shape[0] == 64
    assert c.step_results()["flags"][0] & 16
    c.close()


def test_c_abi_rejects_bad_arguments_without_raising_through_the_boundary():
    _need_gpu()
    L = nat.lib()
    par = rp.mpc_params(12)
    p = nat.make_params(par, 0, 0, None, 0.0, 0.0, 0)
    h = C.c_void_p()
    assert L.lmpc_create(C.byref(p), 0, 0, C.byref(h)) != 0                     # empty batch
    assert b"batch" in L.lmpc_last_error() or L.lmpc_last_error()
    p_bad = nat.make_params(rp.mpc_params(13), 0, 0, None, 0.0, 0.0, 0)          # horizon without an instantiation
    rc = L.lmpc_create(C.byref(p_bad), 4, 0, C.byref(h))
    if rc == 0:                                                                   # accepted at create: must fail at solve
        x0 = np.zeros((4, 6)); u0 = np.zeros((4, 2)); abc = np.zeros((4, 13, 54))
        out = [np.zeros((4, 14, 6)), np.zeros((4, 13, 2)), np.zeros((4, 26)), np.zeros(4, np.int32), np.zeros(4, np.int32), np.zeros((4, 3))]
        assert L.lmpc_solve_mpc_host(h, nat.ptr(x0), nat.ptr(u0), nat.ptr(abc), 13 * 54, 54, *[nat.ptr(a) for a in out]) != 0
        L.lmpc_destroy(h)
    assert L.lmpc_create(C.byref(p), 4, 0, C.byref(h)) == 0
    x0 = np.zeros((4, 6)); u0 = np.zeros((4, 2)); abc = np.zeros((4, 12, 54))
    out = [np.zeros((4, 13, 6)), np.zeros((4, 12, 2)), np.zeros((4, 24)), np.zeros(4, np.int32), np.zeros(4, np.int32), np.zeros((4, 3))]
    assert L.lmpc_solve_mpc_host(h, None, nat.ptr(u0), nat.ptr(abc), 12 * 54, 54, *[nat.ptr(a) for a in out]) != 0      # null x0
    assert L.lmpc_solve_mpc_host(h, nat.ptr(x0), nat.ptr(u0), nat.ptr(abc), 7, 54, *[nat.ptr(a) for a in out]) != 0      # bad strides
    assert L.lmpc_step_host(h, 0, nat.ptr(x0), *([None] * 10)) != 0                                                        # no lap store yet
    assert L.lmpc_ss_add_point(h, nat.ptr(x0), nat.ptr(u0)) != 0
    assert L.lmpc_rollout_step(h, 0, None, 0) != 0
    # an all-zero model is a legal (if useless) QP: the call itself must succeed and report per-instance status
    assert L.lmpc_solve_mpc_host(h, nat.ptr(x0), nat.ptr(u0), nat.ptr(abc), 12 * 54, 54, *[nat.ptr(a) for a in out]) == 0
    L.lmpc_destroy(h)


def test_lmpc_qp_with_short_horizon_matches_oracle(gold, track):
    """LMPC-type QP at N = 6 (BASELINE configs[4] lists LMPC at N in {6, 12}): the first six stages of a golden LMPC step."""
    _need_gpu()
    from oracle import osqp_port
    from racinglmpc_b200.batched import pack_abc
    N = 6
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    _, _, _, _, oQts, opar = ftocp.lmpc_params(track, N)
    opar.timeVarying = True
    keys = [(4, 60), (5, 90), (6, 40)]
    B = len(keys)
    x0 = np.stack([gold["lmpc_%d_%d_x0" % k] for k in keys])
    uold = np.stack([gold["lmpc_%d_%d_OldInput" % k].ravel() for k in keys])
    A = [gold["lmpc_%d_%d_A" % k][:N] for k in keys]; Bm = [gold["lmpc_%d_%d_B" % k][:N] for k in keys]
    Cm = [gold["lmpc_%d_%d_C" % k][:N] for k in keys]
    abc = np.stack([pack_abc(a, b, c) for a, b, c in zip(A, Bm, Cm)])
    SS = np.stack([gold["lmpc_%d_%d_SS_sel" % k] for k in keys]); Qf = np.stack([gold["lmpc_%d_%d_Qfun_sel" % k] for k in keys])
    s = BatchedFTOCP(par, batch=B, numSS_Points=numSS_Points, numSS_it=numSS_it, QterminalSlack=Qts)
    o = s.solve(x0, uold, abc, SS, Qf)
    s.close()
    assert np.all(o["status"] == 1), (o["status"], o["iters"])
    for b in range(B):
        opar.A, opar.B = list(A[b]), list(Bm[b])
        F, bb = ftocp.build_ineq(opar)
        G, E, Lv = ftocp.build_eq(opar, list(A[b]), list(Bm[b]), list(Cm[b]))
        H, q = ftocp.build_cost(opar, uold[b][None, :])
        F2, b2, G2, E2, L2, H2, q2 = ftocp.add_safe_set(F, bb, G, E, Lv, H, q, 6, N, SS[b], Qf[b], oQts)
        P, qq, Am, l, u = ftocp.osqp_form(H2, q2, F2, b2, G2, E2 @ x0[b] + L2)
        z, info = osqp_port.tight_qp(P, qq, Am, l, u)
        assert info["status"] == 1
        assert np.max(np.abs(o["xPred"][b].ravel() - z[:6 * (N + 1)])) < 1e-6
        assert np.max(np.abs(o["uPred"][b].ravel() - z[6 * (N + 1):6 * (N + 1) + 2 * N])) < 1e-6
