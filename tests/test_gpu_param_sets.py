"""GPU tier: per-controller QP parameters (lmpc_set_param_sets).

A heterogeneous batch is K uniform batches in one launch: every instance's outputs are bit-identical to those of a handle created
with that instance's set solving the same batch (the variant runs the same solver code; only the address space of the parameters
differs).  Checked for MPC-type QPs through the chunked host path and the device path, for LMPC-type QPs, and for the device-resident
closed loop with and without warm start, and at every (horizon, safe-set size) the library is built for (the streamed horizons
N >= 32 as expected failures, an open finding); sampled instances are checked against the oracle on the QP assembled from their own set."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import BatchedFTOCP, workloads, reference_params as rp   # noqa: E402
from racinglmpc_b200 import _native as nat                                   # noqa: E402
from racinglmpc_b200.controller import BatchedController                      # noqa: E402
from oracle import ftocp, kkt                                                 # noqa: E402
import oracle_batch as ob                                                     # noqa: E402

N = 12
LMPC_E_INVALID = -1


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def mpc_sets(K=8):
    """configs[1] tunings (oracle parameter objects, usable by both the library and the oracle's assembly)."""
    _, base = ftocp.mpc_params(6, 2, N, 0.8)
    base.timeVarying = True
    out = []
    for k in range(K):
        p = copy.deepcopy(base)
        p.Q = np.diag([1.0 + 0.25 * k, 1.0, 1, 1, 0.0, 100.0])
        p.R = np.diag([1.0, 10.0 + k])
        p.dR = 0.2 * k * np.array([1.0, 10.0])
        p.Qslack = np.array([0.25 * k, 50.0 + 10.0 * k])
        p.xRef = np.array([0.7 + 0.05 * k, 0, 0, 0, 0, 0])
        p.bx = np.full((2, 1), 1.8 + 0.05 * k)
        out.append(p)
    return out


def lmpc_sets(track, K=8):
    """LMPC tunings varying Qslack, dR and QterminalSlack around the reference's."""
    _, _, _, _, Qts, base = ftocp.lmpc_params(track, N)
    base.timeVarying = True
    ps, qs = [], []
    for k in range(K):
        p = copy.deepcopy(base)
        p.Qslack = (0.5 + 0.25 * k) * np.asarray(base.Qslack, float)
        p.dR = (0.5 + 0.5 * (k % 4)) * np.asarray(base.dR, float)
        ps.append(p)
        qs.append((0.5 + 0.5 * ((k * 3) % 4)) * np.asarray(Qts, float))
    return ps, qs


def lmpc_inputs(gold, B, M=48):
    """configs[2]-shaped LMPC QPs: stage models of the LTV fixture, safe set = 4 x 12 consecutive rows of the PID lap around the
    end of the prediction, cost-to-go counting down (as test_gpu_full_batch_parity builds them)."""
    x0, uold, abc = workloads.ltv_mpc_batch(B, N=N)
    start = np.load(workloads._GOLD + "/workload_ltv.npz")["N%d_start" % N]
    start = start[np.arange(B) % start.shape[0]]
    xP, uP = gold["pid_x"], gold["pid_u"]
    P = M // 4
    SS = np.zeros((B, 6, M)); Qf = np.zeros((B, M)); SuS = np.zeros((B, 6, M)); SuU = np.zeros((B, 2, M))
    for b in range(B):
        i0 = int(min(start[b] + N - P // 2, xP.shape[0] - P - 12))
        for j in range(4):
            rows = np.arange(i0, i0 + P + 1) + 2 * j
            blk = xP[rows].copy()
            blk[:, 0:3] += 1e-3 * (j + 1)
            SS[b, :, P * j:P * j + P] = blk[:P].T
            SuS[b, :, P * j:P * j + P] = blk[1:].T
            SuU[b, :, P * j:P * j + P] = uP[rows[1:]].T
            Qf[b, P * j:P * j + P] = 300.0 - rows[:P] * 0.3 + 5.0 * j
    return x0, uold, abc, SS, Qf, SuS, SuU


def _same(a, b, keys, sel):
    for k in keys:
        assert np.array_equal(a[k][sel], b[k][sel]), k


MPC_KEYS = ("xPred", "uPred", "slack", "status", "iters", "resid")
LMPC_KEYS = MPC_KEYS + ("lambd", "slackTerminal", "zt", "zt_u")


def _solve_dev(s, x0, uold, abc, lm=None):
    """The device entry point with torch tensors; returns host copies of the outputs."""
    B = s.B
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    z = lambda *shape, dt=torch.float64: torch.zeros(*shape, dtype=dt, device="cuda")
    o = dict(xPred=z(B, N + 1, 6), uPred=z(B, N, 2), slack=z(B, 2 * N), status=z(B, dt=torch.int32), iters=z(B, dt=torch.int32),
             resid=z(B, 3))
    args = [t(x0), t(uold), t(abc), N * 54, 54, o["xPred"], o["uPred"], o["status"], o["iters"], o["resid"]]
    if lm is None:
        s.solve_dev(*args, slack=o["slack"])
    else:
        M = s.M
        o.update(lambd=z(B, M), slackTerminal=z(B, 6), zt=z(B, 6), zt_u=z(B, 2))
        SS, Qf, SuS, SuU = (t(a) for a in lm)
        s.solve_dev(*args, slack=o["slack"], SS_sel=SS, Qfun_sel=Qf, Succ_SS=SuS, Succ_uSS=SuU, lambd=o["lambd"],
                    slackTerminal=o["slackTerminal"], zt=o["zt"], zt_u=o["zt_u"])
    s.sync()
    return {k: v.cpu().numpy() for k, v in o.items()}


def _oracle_check(sets, idx, x0, uold, abc, out, lm=None, Qts=None, n_sample=64):
    """Primal solution against the oracle optimum on each sampled instance's own QP (1e-6 where the oracle certifies its answer,
    all of them for MPC-type QPs) and the KKT conditions of that QP (1e-6) everywhere."""
    B = x0.shape[0]
    pick = np.linspace(0, B - 1, n_sample).astype(int)
    Ps, qs, As, ls, us = [], [], [], [], []
    for b in pick:
        p = sets[idx[b]]
        A = abc[b][:, 0:36].reshape(N, 6, 6); Bm = abc[b][:, 36:48].reshape(N, 6, 2); Cc = abc[b][:, 48:54]
        F, bb = ftocp.build_ineq(p)
        H, q = ftocp.build_cost(p, uold[b])
        G, E, L = ftocp.build_eq(p, list(A), list(Bm), list(Cc))
        if lm is not None:
            F, bb, G, E, L, H, q = ftocp.add_safe_set(F, bb, G, E, L, H, q, 6, N, lm[0][b], lm[1][b], Qts[idx[b]])
        P, q, Am, l, u = ftocp.osqp_form(H, q, F, bb, G, E @ x0[b] + L)
        Ps.append(P); qs.append(q); As.append(Am); ls.append(l); us.append(u)
    prob = ob._stack_problems(Ps, qs, As, ls, us)
    zo, infos = ob.tight_batch(prob)
    ok = np.array([i["status"] == 1 and i["polished"] == 1 and max(i["pri_res"], i["dua_res"]) <= 1e-8 for i in infos])
    parts = [out["xPred"][pick].reshape(n_sample, -1), out["uPred"][pick].reshape(n_sample, -1), out["slack"][pick]]
    if lm is not None:
        parts += [out["lambd"][pick], out["slackTerminal"][pick]]
    z = np.concatenate(parts, axis=1)
    n = 6 * (N + 1) + 2 * N
    if lm is None:
        assert ok.all()
    assert ok.mean() > 0.5
    assert np.abs(z[ok, :n] - zo[ok, :n]).max() < 1e-6
    for i in range(n_sample):
        P, q, Am, l, u = Ps[i], qs[i], As[i], ls[i], us[i]
        y = kkt.dual_from_primal(P, q, Am, l, u, z[i], tol=1e-6)
        r = kkt.residuals(P, q, Am, l, u, z[i], y)
        assert r["r_prim"] <= 1e-6 and r["r_dual"] <= 1e-6, (i, r)


def test_mpc_sets_bit_identical_to_uniform_handles_host_and_device_paths():
    _need_gpu()
    B = 4096
    sets = mpc_sets()
    idx = (7 * np.arange(B)) % len(sets)            # neighbouring warps solve different sets
    x0, uold, abc = workloads.ltv_mpc_batch(B, N=N)
    het = BatchedFTOCP(sets[0], batch=B)
    het.set_param_sets(sets, idx)
    o_host = het.solve(x0, uold, abc)               # chunked synchronous host path (4 instance ranges at this size)
    assert nat.lib().lmpc_host_chunks(het._h, 0) == 4
    o_dev = _solve_dev(het, x0, uold, abc)
    assert np.all(o_host["status"] == 1) and het.late_accepts == 0
    for k, p in enumerate(sets):
        uni = BatchedFTOCP(p, batch=B)
        ref = uni.solve(x0, uold, abc)
        sel = idx == k
        _same(o_host, ref, MPC_KEYS, sel)
        _same(o_dev, ref, MPC_KEYS, sel)
        uni.close()
    _oracle_check(sets, idx, x0, uold, abc, o_host)
    het.close()


def test_lmpc_sets_bit_identical_to_uniform_handles(gold, track):
    _need_gpu()
    B = 1024
    sets, qts = lmpc_sets(track)
    idx = (7 * np.arange(B)) % len(sets)
    x0, uold, abc, SS, Qf, SuS, SuU = lmpc_inputs(gold, B)
    het = BatchedFTOCP(sets[0], batch=B, numSS_Points=48, numSS_it=4, QterminalSlack=qts[0])
    het.set_param_sets(sets, idx, qts)
    o = het.solve(x0, uold, abc, SS, Qf, SuS, SuU)
    o_dev = _solve_dev(het, x0, uold, abc, (SS, Qf, SuS, SuU))
    assert np.all(o["status"] == 1) and het.late_accepts == 0
    for k in range(len(sets)):
        uni = BatchedFTOCP(sets[k], batch=B, numSS_Points=48, numSS_it=4, QterminalSlack=qts[k])
        ref = uni.solve(x0, uold, abc, SS, Qf, SuS, SuU)
        _same(o, ref, LMPC_KEYS, idx == k)
        _same(o_dev, ref, LMPC_KEYS, idx == k)
        uni.close()
    _oracle_check(sets, idx, x0, uold, abc, o, lm=(SS, Qf), Qts=qts)
    het.close()


def _closed_loop(par, qts, B, sets=None, idx=None, warm=False, steps=None):
    """Device PID lap, seeding, then LMPC rollout steps until every controller has finished one LMPC lap (or `steps` steps)."""
    numSS_it, numSS_Points = 4, 48
    c = BatchedController(par, B, workloads.track_seg_table(), rp.TRACK_LENGTH, trToUse=4, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=qts, Tmax=1280, ss_cap=7, model_cap=5, warm_start=warm)
    if sets is not None:
        c.set_param_sets(sets[0], idx, sets[1])
    x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (B, 1))
    c.enable_rollout(Tcl=1024)
    c.rollout_set_state(x0, x0)
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(x0, x0)
    n = 0
    while (steps is None and n < 1200) or (steps is not None and n < steps):
        c.rollout_step(seed=1234)
        c.rollout_commit_laps_dev()
        n += 1
        if steps is None and n % 8 == 0 and c.rollout_stats()[0] >= 1:
            break
    bk = c.books()
    flags, unsolved = c.rollout_health()
    st = c.rollout_state()
    laps = {}
    for b in range(0, B, 5):                        # stored safe-set laps of every fifth controller
        for slot in range(7):
            T = C.c_int(0)
            x, u, q = np.zeros((1280, 6)), np.zeros((1280, 2)), np.zeros(1280)
            nat.check(nat.lib().lmpc_ss_get_lap(c._h, b, slot, C.byref(T), nat.ptr(x), nat.ptr(u), nat.ptr(q)))
            laps[(b, slot)] = (x[:T.value].copy(), u[:T.value].copy(), q[:T.value].copy())
    c.close()
    return n, dict(bk, flags=flags, unsolved=unsolved, **st), laps


@pytest.mark.parametrize("warm", [False, True])
def test_closed_loop_sets_bit_identical_to_uniform_runs(warm):
    _need_gpu()
    B = 256
    _, _, _, _, Qts, base = rp.lmpc_params(N)
    ps, qs = [], []
    for k in range(4):
        p = copy.deepcopy(base)
        p.Qslack = (0.5, 1.0, 2.0, 4.0)[k] * np.asarray(base.Qslack, float)
        p.dR = (2.0, 1.0, 0.5, 1.5)[k] * np.asarray(base.dR, float)
        ps.append(p)
        qs.append((1.0, 0.5, 2.0, 1.0)[k] * Qts)
    idx = np.arange(B) % 4
    n, het, het_laps = _closed_loop(base, Qts, B, (ps, qs), idx, warm)
    assert het["lap_n"].min() >= 1, "not every controller finished an LMPC lap in %d steps" % n
    for k in range(4):
        _, ref, ref_laps = _closed_loop(ps[k], qs[k], B, warm=warm, steps=n)
        sel = idx == k
        for key in ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt",
                    "flags", "unsolved"):
            assert np.array_equal(het[key][sel], ref[key][sel]), (k, key)
        for (b, slot), v in het_laps.items():
            if idx[b] == k:
                assert all(np.array_equal(a, r) for a, r in zip(v, ref_laps[(b, slot)])), (k, b, slot)


# Horizons from 32 on read the stage model from global memory inside the sweeps (ftocp_pdip.cuh, stream_model); there the variant
# and the uniform kernel round differently in a few instances (7e-15 on MPC QPs, up to 3e-8 on LMPC QPs, same iterations and
# status; DESIGN.md, "Per-controller parameters").  An open finding, kept visible here instead of loosening the comparison.
_STREAMED = pytest.mark.xfail(reason="streamed stage model: the variant is not yet bit-identical at N >= 32 (DESIGN.md)", strict=False)
GRID = [(4, 0), (6, 0), (8, 0), (10, 0), (12, 0), (14, 0), (16, 0), (20, 0), (24, 0),
        (4, 48), (6, 48), (8, 48), (10, 48), (12, 48), (14, 48), (16, 48), (20, 48), (24, 48),
        (12, 24), (12, 32), (12, 64), (12, 96), (14, 24), (14, 32), (14, 64), (14, 96)] + \
       [pytest.param(n, m, marks=_STREAMED) for n, m in ((32, 0), (48, 0), (32, 48), (48, 48))]


@pytest.mark.parametrize("Nh,M", GRID)
def test_every_instantiation_bit_identical_to_uniform_handles(gold, track, Nh, M):
    """The variant against the uniform kernel at every (horizon, safe-set size) the library is built for, MPC- and LMPC-type
    (64 QPs, 4 sets interleaved): the stage-model streaming of long horizons and every safe-set size included."""
    _need_gpu()
    B = 64
    x0, uold, abc = workloads.ltv_mpc_batch(B, N=48)
    abc = np.ascontiguousarray(abc[:, :Nh])
    idx = (7 * np.arange(B)) % 4
    if M == 0:
        _, base = ftocp.mpc_params(6, 2, Nh, 0.8)
        ps, qs, kw, lm, keys = [], [None] * 4, {}, (), MPC_KEYS
    else:
        _, _, _, _, Qts, base = ftocp.lmpc_params(track, Nh)
        ps, qs, kw, keys = [], [], dict(numSS_Points=M, numSS_it=4), LMPC_KEYS
        xP = gold["pid_x"]
        SS = np.zeros((B, 6, M)); Qf = np.zeros((B, M))
        P = M // 4
        for b in range(B):
            i0 = 40 + 3 * b
            for j in range(4):
                blk = xP[i0 + 2 * j:i0 + 2 * j + P].copy()
                blk[:, 0:3] += 1e-3 * (j + 1)
                SS[b, :, P * j:P * j + P] = blk.T
                Qf[b, P * j:P * j + P] = 300.0 - (i0 + np.arange(P)) * 0.3 + 5.0 * j
        lm = (SS, Qf)
    for k in range(4):
        p = copy.deepcopy(base)
        p.Qslack = (0.5 + 0.5 * k) * np.asarray(base.Qslack, float)
        p.dR = np.asarray(base.dR, float) * (1.0 + 0.5 * k) + 0.1 * k
        ps.append(p)
        if M:
            qs.append((0.5 + 0.5 * ((3 * k) % 4)) * np.asarray(Qts, float))
    mk = lambda p, q: BatchedFTOCP(p, batch=B, QterminalSlack=q, **kw)
    het = mk(base, qs[0])
    het.set_param_sets(ps, idx, qs if M else None)
    o = het.solve(x0, uold, abc, *lm)
    for k in range(4):
        uni = mk(ps[k], qs[k])
        _same(o, uni.solve(x0, uold, abc, *lm), keys, idx == k)
        uni.close()
    het.close()


def test_revert_gives_the_uniform_kernel_results():
    _need_gpu()
    B = 512
    sets = mpc_sets()
    x0, uold, abc = workloads.ltv_mpc_batch(B, N=N)
    fresh = BatchedFTOCP(sets[0], batch=B)
    ref = _solve_dev(fresh, x0, uold, abc)
    s = BatchedFTOCP(sets[0], batch=B)
    s.set_param_sets(sets, np.arange(B) % len(sets))
    het = _solve_dev(s, x0, uold, abc)
    assert not np.array_equal(het["uPred"], ref["uPred"])
    s.set_param_sets(None)
    l0 = s.kernel_launches
    o = _solve_dev(s, x0, uold, abc)
    assert s.kernel_launches - l0 == 1
    _same(o, ref, MPC_KEYS, slice(None))
    fresh.close(); s.close()


def test_rejected_calls_leave_the_handle_as_it_was(gold, track):
    _need_gpu()
    B = 16
    sets, qts = lmpc_sets(track, 4)
    idx = np.arange(B) % 4
    x0, uold, abc, SS, Qf, SuS, SuU = lmpc_inputs(gold, B)
    s = BatchedFTOCP(sets[0], batch=B, numSS_Points=48, numSS_it=4, QterminalSlack=qts[0])
    s.set_param_sets(sets, idx, qts)
    before = s.solve(x0, uold, abc, SS, Qf, SuS, SuU)
    good, gidx = nat.make_param_sets(s._p, sets, idx, B, 48, 4, qts)
    L = nat.lib()

    def call(tab, n, ix):
        return L.lmpc_set_param_sets(s._h, tab, n, nat.ptr(ix) if ix is not None else None)

    def edited(k, **kw):
        tab = (nat.Params * 4)()
        C.memmove(tab, good, C.sizeof(tab))
        for f, v in kw.items():
            if f in ("bu", "QterminalSlack"):
                getattr(tab[k], f)[:] = v
            else:
                setattr(tab[k], f, v)
        return tab

    cases = [edited(1, N=14), edited(2, ncx=1), edited(3, numSS_Points=24), edited(0, numSS_it=2), edited(1, warm_start=1),
             edited(2, bu=[0.5, 0.0, 10.0, 10.0, 0, 0, 0, 0]), edited(3, QterminalSlack=np.zeros(36))]
    for tab in cases:
        assert call(tab, 4, gidx) == LMPC_E_INVALID
    assert call(good, 0, gidx) == LMPC_E_INVALID                         # nsets == 0 with a table
    big = (nat.Params * (B + 1))(*([good[0]] * (B + 1)))
    assert call(big, B + 1, np.zeros(B, np.int32)) == LMPC_E_INVALID      # nsets > batch
    assert call(good, 4, np.full(B, 4, np.int32)) == LMPC_E_INVALID      # index out of range
    assert call(good, 4, np.full(B, -1, np.int32)) == LMPC_E_INVALID
    after = s.solve(x0, uold, abc, SS, Qf, SuS, SuU)
    _same(after, before, LMPC_KEYS, slice(None))
    s.close()
