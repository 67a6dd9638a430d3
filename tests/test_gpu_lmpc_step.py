"""GPU tier: K1 (k-NN regression), K2 (safe-set selection), K6 (addPoint / computeCost) and the fused
LMPC step against golden vectors produced by the REAL reference (tests/golden/make_golden.py)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                  # noqa: E402
from racinglmpc_b200.controller import BatchedController            # noqa: E402
import replay                                                       # noqa: E402


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _restore(gold, track, keys, N=12):
    """One controller instance per snapshot key, restored to the state just before LMPC.solve(x0)."""
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    B = len(keys)
    c = BatchedController(par, B, track.seg_table(), track.TrackLength, trToUse=4, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1536, ss_cap=8, model_cap=5)
    st = dict(xLin=[], uLin=[], zt=[], OldInput=[], timeStep=[], has_pred=[], xPred=[])
    x0 = []
    for b, key in enumerate(keys):
        k = "lmpc_%d_%d_" % key
        for j in range(int(gold[k + "pm_nlap"])):
            c.model_add_trajectory(b, gold[k + "pmx%d" % j], gold[k + "pmu%d" % j])
        for j in range(int(gold[k + "nlap"])):
            c.add_trajectory(b, gold[k + "SS%d" % j], gold[k + "uSS%d" % j], qfun=gold[k + "Qfun%d" % j],
                             lap_time=int(gold[k + "LapTime"][j]))
        assert c.it[b] == int(gold[k + "it"])
        if not int(gold[k + "has_pred"]):
            # very first LMPC solve: reproduce the aliased write of PC.py:394 (row 1+4, column ey of the shared PID lap)
            for j in range(int(gold[k + "nlap"])):
                row = gold[k + "SS%d" % j][5].copy()
                row[5] -= track.TrackLength
                c.patch_row(b, j, 5, row)
        st["xLin"].append(gold[k + "xLin"]); st["uLin"].append(gold[k + "uLin"]); st["zt"].append(gold[k + "zt"])
        st["OldInput"].append(gold[k + "OldInput"].ravel()); st["timeStep"].append(int(gold[k + "timeStep"]))
        st["has_pred"].append(int(gold[k + "has_pred"])); st["xPred"].append(gold[k + "xPred_prev"])
        x0.append(gold[k + "x0"])
    c.set_state(**{k: np.array(v) for k, v in st.items()})
    return c, np.array(x0)


def test_k1_regression_matches_reference(gold, track):
    _need_gpu()
    keys = replay.LMPC_KEYS
    c, x0 = _restore(gold, track, keys)
    abc, flags = c.identify()
    assert np.all(flags == 0), flags
    for b, key in enumerate(keys):
        k = "lmpc_%d_%d_" % key
        A = abc[b][:, 0:36].reshape(12, 6, 6); B = abc[b][:, 36:48].reshape(12, 6, 2); C = abc[b][:, 48:54]
        # rows 3..5 are closed-form (sin/cos may differ in the last ulp); rows 0..2 come from 5x5 solves
        assert np.max(np.abs(A - gold[k + "A"])) < 1e-9, key
        assert np.max(np.abs(B - gold[k + "B"])) < 1e-9, key
        assert np.max(np.abs(C - gold[k + "C"])) < 1e-9, key
        assert np.max(np.abs(A[:, 3:, :] - gold[k + "A"][:, 3:, :])) < 1e-14
    c.close()


def test_k2_selection_is_bit_exact(gold, track):
    _need_gpu()
    keys = replay.LMPC_KEYS
    c, x0 = _restore(gold, track, keys)
    o = c.select(x0)
    assert np.all(o["flags"] == 0), o["flags"]
    for b, key in enumerate(keys):
        k = "lmpc_%d_%d_" % key
        assert np.array_equal(o["SS_sel"][b], gold[k + "SS_sel"]), key
        assert np.array_equal(o["Qfun_sel"][b], gold[k + "Qfun_sel"]), key
        assert np.array_equal(o["Succ_SS"][b], gold[k + "Succ_SS"]), key
        assert np.array_equal(o["Succ_uSS"][b], gold[k + "Succ_uSS"]), key
    c.close()


def test_fused_lmpc_step_matches_reference(gold, track):
    _need_gpu()
    keys = replay.LMPC_KEYS
    c, x0 = _restore(gold, track, keys)
    l0 = c.kernel_launches
    o = c.step(x0)
    assert c.kernel_launches - l0 == 4                       # K1 (writes transposed records itself), K2, QP, shift
    assert np.all(o["status"] == 1) and np.all(o["flags"] == 0), (o["status"], o["flags"])
    st = c.get_state()
    for b, key in enumerate(keys):
        k = "lmpc_%d_%d_" % key
        assert np.max(np.abs(o["xPred"][b] - gold[k + "xPred"])) < 1e-6, key
        assert np.max(np.abs(o["uPred"][b] - gold[k + "uPred"])) < 1e-6, key
        assert np.max(np.abs(o["zt"][b] - gold[k + "zt_out"])) < 1e-5, key
        assert np.array_equal(o["SS_sel"][b], gold[k + "SS_sel"])
        # state shift (PC.py:129-137)
        assert np.array_equal(st["xLin"][b][:-1], o["xPred"][b][1:]) and np.array_equal(st["xLin"][b][-1], o["zt"][b])
        assert np.array_equal(st["uLin"][b][:-1], o["uPred"][b][1:]) and np.array_equal(st["uLin"][b][-1], o["zt_u"][b])
        assert np.array_equal(st["OldInput"][b], o["uPred"][b][0])
        assert st["timeStep"][b] == int(gold[k + "timeStep"]) + 1
    c.close()


def test_add_point_and_rollout_cost(gold, track):
    _need_gpu()
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(12)
    c = BatchedController(par, 2, track.seg_table(), track.TrackLength, trToUse=4, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1536)
    xP, uP = gold["pid_x"], gold["pid_u"]
    for b in range(2):
        for _ in range(4):
            c.add_trajectory(b, xP, uP)
    x, u, q = c.get_lap(0, 3)
    assert np.array_equal(x, xP) and np.array_equal(u, uP)
    assert np.array_equal(q, gold["pid_Qfun"])               # computeCost on the device (PC.py:447-464)
    pts = np.array([[0.6, 0.01, 0.02, 0.03, 0.5, -0.1], [0.7, 0.0, 0.0, 0.0, 1.5, 0.2]])
    us = np.array([[0.1, 0.2], [-0.1, 0.3]])
    c.add_point(pts, us)
    c.add_point(pts + 0.1, us)
    for b in range(2):
        x, u, q = c.get_lap(b, 3)
        assert x.shape[0] == xP.shape[0] + 2
        assert np.array_equal(x[-2], pts[b] + np.array([0, 0, 0, 0, track.TrackLength, 0]))
        assert np.array_equal(u[-1], us[b])
        assert q[-2] == gold["pid_Qfun"][-1] - 1 and q[-1] == gold["pid_Qfun"][-1] - 2
        x2, _, _ = c.get_lap(b, 2)
        assert x2.shape[0] == xP.shape[0]                    # only lap it-1 grows (PC.py:472)
    c.close()


def test_closed_loop_lap_matches_reference_lap(gold, track):
    """Drive LMPC lap 4 (main.py:113-117) with the GPU controller and the oracle's vehicle simulator, same seed
    as the golden run with the real reference: same lap length, same states at the snapshot steps."""
    _need_gpu()
    from oracle import vehicle
    N = 12
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    xP, uP = gold["pid_x"].copy(), gold["pid_u"].copy()
    c = BatchedController(par, 1, track.seg_table(), track.TrackLength, trToUse=4, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1536)
    for _ in range(4):
        c.model_add_trajectory(0, xP, uP)
    for _ in range(4):
        c.add_trajectory(0, xP, uP)
    c.set_state(xLin=xP[1:N + 2], uLin=uP[1:N + 1], zt=np.array([0.0, 0, 0, 0, 10.0, 0]), OldInput=np.zeros(2),
                timeStep=[0], has_pred=[0])
    # aliased write of the first solve (PC.py:394)
    row = xP[5].copy(); row[5] -= track.TrackLength
    for j in range(4):
        c.patch_row(0, j, 5, row)
    np.random.seed(0)
    x0 = np.array([0.5, 0, 0, 0, 0, 0.0])
    vehicle.closed_loop(track, [x0, x0], vehicle.PIDFollower(0.8))      # consume the PID lap's random draws
    xs, gs = [x0], [x0]
    t = 0
    out = c.alloc_step_outputs()
    while True:
        if t in (1, 60, 200):
            assert np.max(np.abs(xs[-1] - gold["lmpc_4_%d_x0" % t])) < 1e-6, t
        o = c.step(xs[-1], out=out)
        assert o["status"][0] == 1 and o["flags"][0] == 0, (t, o["status"], o["flags"])
        u = o["uPred"][0, 0].copy()
        c.add_point(xs[-1], u)
        xt, gt = vehicle.dyn_model(track, xs[-1], gs[-1], u)
        xs.append(xt); gs.append(gt)
        t += 1
        if xs[-1][4] > track.TrackLength or t >= 400:
            break
    assert t == int(gold["lmpc_lap_lengths"][0])
    c.close()


def test_config3_workload_step_vs_oracle(track):
    """BASELINE configs[2] shapes (trToUse = 5, 4-lap safe set, grown lap it-1): a sample of instances is replayed
    through the oracle controller (reference arithmetic) and compared with the fused GPU step."""
    _need_gpu()
    from racinglmpc_b200 import workloads
    from oracle import ftocp, ltv_model, osqp_port
    B, N = 96, 12
    data = workloads.lmpc_batch(B)
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, B, track.seg_table(), track.TrackLength, trToUse=5, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1536, ss_cap=6, model_cap=6)
    workloads.restore_lmpc_batch(c, data)
    o = c.step(data["x0"])
    assert np.all(o["status"] == 1) and np.all(o["flags"] == 0), (np.unique(o["status"]), np.unique(o["flags"]))
    assert o["resid"].max() <= 1.000001e-9
    _, _, _, _, oQts, opar = ftocp.lmpc_params(track, N)
    opar.timeVarying = True
    for b in (0, 1, 37, 60, 95):
        pm = ltv_model.LocalLTVModel(6, 2, track, 5)
        pm.xStored = [lx for lx, _ in data["model_laps"][b]]
        pm.uStored = [lu for _, lu in data["model_laps"][b]]
        pm.lapTime = [lx.shape[0] for lx in pm.xStored]
        lm = ftocp.OracleLMPC(numSS_Points, numSS_it, oQts, opar, pm, qp=osqp_port.tight_qp)
        lm.SS = [s[0] for s in data["ss_laps"][b]]
        lm.uSS = [s[1] for s in data["ss_laps"][b]]
        lm.Qfun = [s[2] for s in data["ss_laps"][b]]
        lm.LapTime = list(data["lap_times"])
        lm.it, lm.timeStep = 4, int(data["t"][b])
        lm.zt, lm.xLin, lm.uLin = data["zt"][b].copy(), data["xLin"][b].copy(), data["uLin"][b].copy()
        lm.OldInput, lm.xPred = data["OldInput"][b].copy(), data["xPred"][b].copy()
        lm.solve(data["x0"][b])
        assert np.max(np.abs(o["uPred"][b] - lm.uPred)) < 1e-6, b
        assert np.max(np.abs(o["xPred"][b] - lm.xPred)) < 1e-6, b
        assert np.max(np.abs(o["zt"][b] - lm.zt)) < 1e-5, b
    c.close()


def test_device_resident_closed_loop_matches_host_driven_loop(gold, track):
    """§8f rank 1: the on-GPU Simulator.dynModel + device addPoint + device lap hand-over.  Two LMPC laps driven entirely
    on the device (noise draws supplied from the host RNG in the reference's order) against the same laps driven step by
    step through the oracle's restated simulator."""
    _need_gpu()
    from oracle import vehicle
    N = 12
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    xP, uP = gold["pid_x"].copy(), gold["pid_u"].copy()

    def fresh():
        c = BatchedController(par, 1, track.seg_table(), track.TrackLength, trToUse=4, numSS_Points=numSS_Points,
                              numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1536, ss_cap=6, model_cap=5)
        for _ in range(4):
            c.model_add_trajectory(0, xP, uP)
        for _ in range(4):
            c.add_trajectory(0, xP, uP)
        c.set_state(xLin=xP[1:N + 2], uLin=uP[1:N + 1], zt=np.array([0.0, 0, 0, 0, 10.0, 0]), OldInput=np.zeros(2), timeStep=[0], has_pred=[0])
        return c
    x0 = np.array([0.5, 0, 0, 0, 0, 0.0])
    # (a) host-driven reference loop: GPU controller + oracle simulator
    ca = fresh()
    rng = np.random.default_rng(42)
    zs = rng.standard_normal((600, 3))
    xa, ga = x0.copy(), x0.copy()
    lapsA, cur = [], []
    k = 0
    out = ca.alloc_step_outputs()
    for lap in range(2):
        xs, us = [], []
        while True:
            o = ca.step(xa, out=out)
            u = o["uPred"][0, 0].copy()
            ca.add_point(xa, u)
            xs.append(xa.copy()); us.append(u)
            zi = iter(zs[k]); k += 1
            fake = type("R", (), {"standard_normal": lambda self, it=zi: next(it)})()
            xa, ga = vehicle.dyn_model(track, xa, ga, u, rng=fake)
            if xa[4] > track.TrackLength:
                break
        xl, ul = np.array(xs), np.array(us)
        lapsA.append((xl, ul))
        ca.add_trajectory(0, xl, ul)
        ca.model_add_trajectory(0, xl, ul)
        ca.set_state(timeStep=[0])                     # LMPC.addTrajectory resets the step counter (PC.py:445)
        xa = xa - np.array([0, 0, 0, 0, track.TrackLength, 0])
    ca.close()
    # (b) device-resident loop
    cb = fresh()
    cb.enable_rollout(Tcl=512)
    cb.rollout_set_state(x0, x0)
    lapsB = []
    k = 0
    while len(lapsB) < 2:
        cb.rollout_step(z=zs[k]); k += 1
        done, n = cb.rollout_done()
        if done[0]:
            lapsB.append(cb.rollout_get_lap(0))
            cb.rollout_finish_laps(done, n)
    for (xa_, ua_), (xb_, ub_) in zip(lapsA, lapsB):
        assert xa_.shape == xb_.shape
        dx_, du_ = np.max(np.abs(xa_ - xb_), axis=1), np.max(np.abs(ua_ - ub_), axis=1)
        # both arms run the same GPU controller; the simulators differ by rounding (~1e-16), which a step near an
        # LP-degenerate terminal simplex amplifies up to the solver's primal accuracy (measured 5.5e-7 transient,
        # back to 4e-10 afterwards) -> the north-star tolerance 1e-6 is the bound, not bit equality.
        assert dx_.max() < 1e-6 and du_.max() < 1e-6, (dx_.max(), du_.max(), dx_[::40], du_[::40])
    # the lap handed over on the device equals the recorded one; Q-function computed on the device
    xs_, us_, q_ = cb.get_lap(0, 5)
    assert np.array_equal(xs_, lapsB[1][0]) and q_[0] == lapsB[1][0].shape[0] - 1
    cb.close()


def test_pooled_lap_exchange_export_import(track):
    """SURVEY §8e pooled-safe-set mode: a stored lap packed on the device (send buffer of the all-gather) and handed to another
    instance arrives bit-exact, sits BEFORE that instance's own latest lap (which stays the lap LMPC.addPoint extends), is ranked
    by its lap time like any other lap (PC.py:395) and is skipped where it would never be selected."""
    _need_gpu()
    from racinglmpc_b200 import workloads
    N, B, Tpad = 12, 4, 512
    data = workloads.lmpc_batch(B)
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, B, track.seg_table(), track.TrackLength, trToUse=5, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1536, ss_cap=7, model_cap=7)
    workloads.restore_lmpc_batch(c, data)
    assert c.it == [4] * B
    rows = torch.zeros(B, Tpad, 9, dtype=torch.float64, device="cuda")
    lens = torch.zeros(B, dtype=torch.int32, device="cuda")
    c.export_laps([1, 1, 1, -1], Tpad, rows, lens)
    rows_h, lens_h = rows.cpu().numpy(), lens.cpu().numpy()
    x1, u1, q1 = c.get_lap(0, 1)
    T = x1.shape[0]
    assert lens_h[0] == T and lens_h[3] == 0 and not rows_h[3].any()
    assert np.array_equal(rows_h[0, :T, 0:6], x1) and np.array_equal(rows_h[0, :T, 6:8], u1) and np.array_equal(rows_h[0, :T, 8], q1)
    assert not rows_h[0, T:].any()
    own_latest = c.get_lap(2, 3)
    # instance 2 gets instance 0's lap with a winning lap time, instance 3 with a hopeless one, 0 and 1 nothing
    took = c.import_laps(np.array([-1, -1, 0, 0]), np.array([0, 0, 100, 100000]), Tpad, rows, lens)
    assert list(took) == [2] and c.it == [4, 4, 5, 4]
    xf, uf, qf = c.get_lap(2, 3)                     # the foreign lap took lap number it-1 (old) ...
    assert np.array_equal(xf, x1) and np.array_equal(uf, u1) and np.array_equal(qf, q1)
    xo, uo, qo = c.get_lap(2, 4)                     # ... and the own latest lap moved up
    assert np.array_equal(xo, own_latest[0]) and np.array_equal(qo, own_latest[2])
    assert c.own_lap_number(2, 3) == 4 and c.LapTime[2][3] == 100
    # selection: the imported lap is the fastest -> its points fill the first numSS_Points/numSS_it columns (PC.py:402-407)
    sel = c.select(data["x0"])
    P = numSS_Points // numSS_it
    for j in range(P):
        col = sel["SS_sel"][2][:, j]
        assert np.any(np.all(x1 == col[None, :], axis=1)), j
    assert np.array_equal(sel["SS_sel"][0], c.select(data["x0"])["SS_sel"][0])
    o = c.step(data["x0"])
    assert np.all(o["status"] == 1) and np.all(o["flags"] == 0), (o["status"], o["flags"])
    # addPoint still extends the instance's OWN latest lap
    c.add_point(data["x0"], o["uPred"][:, 0])
    assert c.get_lap(2, 4)[0].shape[0] == own_latest[0].shape[0] + 1 and c.get_lap(2, 3)[0].shape[0] == T
    c.close()


def test_device_pid_lap_sysid_lti_mpc_and_seeding(gold, track):
    """SURVEY §8f rank 3: main.py's seeding pipeline on the device against the oracle's restatement of Simulator.sim + PID
    (SysModel.py:22-54, Utilities.py:42-68), Regression (Utilities.py:5-28), the LTI MPC lap (main.py:72-80) and the seeding of
    LMPC + PredictiveModel with four copies of the PID lap (main.py:99-110) — same standard-normal draws on both sides."""
    _need_gpu()
    from oracle import vehicle, osqp_port, ftocp
    N, K = 12, 300
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, 2, track.seg_table(), track.TrackLength, trToUse=4, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=1536, ss_cap=6, model_cap=5)
    c.enable_rollout(Tcl=1024)
    x0 = np.array([0.5, 0, 0, 0, 0, 0.0])
    c.rollout_set_state(np.tile(x0, (2, 1)), np.tile(x0, (2, 1)))
    rng = np.random.default_rng(99)
    zs = rng.standard_normal((2, K, 5))
    for k in range(K):
        c.rollout_pid_step(0.8, z_pid=zs[:, k, 0:2], z_sim=zs[:, k, 2:5])
    done, n = c.rollout_done()
    assert list(n) == [K, K]
    laps, recs = [], []
    for b in range(2):
        it = iter(zs[b].ravel())
        fake = type("R", (), {"standard_normal": lambda self, it=it: next(it)})()
        xo, uo, _, _ = vehicle.closed_loop(track, [x0, x0], vehicle.PIDFollower(0.8, rng=fake), multi_lap=True, rng=fake, max_steps=K)
        xg, ug = c.rollout_get_lap(b)
        assert xg.shape == (K, 6) and np.max(np.abs(xg - xo)) < 1e-9 and np.max(np.abs(ug - uo)) < 1e-9, b
        laps.append((xo, uo))
        recs.append((xg, ug))
    # ---- ridge system identification of each record
    A, Bm, flags = c.rollout_sysid(1e-7)
    assert np.all(flags == 0)
    for b in range(2):
        oA, oB, _ = vehicle.ridge_sysid(laps[b][0], laps[b][1], 1e-7)
        assert np.max(np.abs(A[b] - oA)) < 1e-6 and np.max(np.abs(Bm[b] - oB)) < 1e-6, (np.max(np.abs(A[b] - oA)), np.max(np.abs(Bm[b] - oB)))
    # ---- a few LTI-MPC closed-loop steps with the identified model (mode 2, main.py:72-80 with initMPCParams) against the
    #      oracle controller holding the SAME model: a second controller with the MPC cost drives the same PID lap first
    cm = BatchedController(rp.mpc_params(N), 2, track.seg_table(), track.TrackLength, trToUse=1, Tmax=1536, model_cap=2)
    cm.enable_rollout(Tcl=1024)
    cm.rollout_set_state(np.tile(x0, (2, 1)), np.tile(x0, (2, 1)))
    for k in range(K):
        cm.rollout_pid_step(0.8, z_pid=zs[:, k, 0:2], z_sim=zs[:, k, 2:5])
    A2, B2, _ = cm.rollout_sysid(1e-7)
    assert np.array_equal(A2, A) and np.array_equal(B2, Bm)
    cm.rollout_set_state(np.tile(x0, (2, 1)), np.tile(x0, (2, 1)))
    z2 = rng.standard_normal((2, 30, 3))
    for k in range(30):
        cm.rollout_step(z=z2[:, k], mode=2)
    assert np.all(cm.step_results()["status"] == 1)
    for b in range(2):
        omp, _ = ftocp.mpc_params(6, 2, N, 0.8)
        omp.A, omp.B = A[b], Bm[b]
        it = iter(z2[b].ravel())
        fake = type("R", (), {"standard_normal": lambda self, it=it: next(it)})()
        xo, uo, _, _ = vehicle.closed_loop(track, [x0, x0], ftocp.OracleMPC(omp, qp=osqp_port.tight_qp), multi_lap=True, rng=fake, max_steps=30)
        xg, ug = cm.rollout_get_lap(b)
        assert xg.shape[0] == K + 30
        assert np.max(np.abs(xg[K:] - xo)) < 1e-6 and np.max(np.abs(ug[K:] - uo)) < 1e-6, b
    cm.close()
    # ---- seeding: four copies of the PID record in both stores, controller state as LMPC.__init__/addTrajectory leave it
    c.rollout_seed_from_record(n, copies=4)
    assert c.it == [4, 4] and c.LapTime[0] == [K] * 4
    for b in range(2):
        for lapno in range(4):
            xs_, us_, q_ = c.get_lap(b, lapno)
            assert np.array_equal(xs_, recs[b][0]) and np.array_equal(us_, recs[b][1])      # the device record, bit for bit
            assert np.array_equal(q_, ftocp.rollout_cost(recs[b][0], track.TrackLength))
    st = c.get_state()
    for b in range(2):
        assert np.array_equal(st["xLin"][b], recs[b][0][1:N + 2]) and np.array_equal(st["uLin"][b], recs[b][1][1:N + 1])
        assert np.array_equal(st["zt"][b], [0, 0, 0, 0, 10.0, 0]) and st["timeStep"][b] == 0
    assert list(c.rollout_done()[1]) == [0, 0]
    # and the first LMPC step from the start line solves with these stores
    c.rollout_set_state(np.tile(x0, (2, 1)), np.tile(x0, (2, 1)))
    c.rollout_step(z=np.zeros((2, 3)))
    r = c.step_results()
    assert np.all(r["status"] == 1) and np.all(r["flags"] == 0), (r["status"], r["flags"])
    c.close()


def test_device_lap_books_and_pooled_exchange_match_the_host_books(gold, track):
    """SURVEY §8f rank 3 / §8e: the once-per-lap bookkeeping on the device (csrc/lapbooks.cuh: which laps are the numSS_it
    fastest, lap it-1, usedIt, eviction) and the device-side pooled exchange, against the host-side books that restate the
    reference's lists (controller.py): two batches driven with the same noise must visit bit-identical states, hand over the
    same laps and -- after exchanging laps -- keep doing so."""
    _need_gpu()
    from racinglmpc_b200 import sharding
    N, B, Tpad, share = 12, 6, 320, 2
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    xP, uP = gold["pid_x"].copy(), gold["pid_u"].copy()

    def fresh():
        c = BatchedController(par, B, track.seg_table(), track.TrackLength, trToUse=4, numSS_Points=numSS_Points,
                              numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1536, ss_cap=7, model_cap=5)
        for b in range(B):
            for _ in range(4):
                c.model_add_trajectory(b, xP, uP)
            for _ in range(4):
                c.add_trajectory(b, xP, uP)
        c.set_state(xLin=np.tile(xP[1:N + 2], (B, 1, 1)), uLin=np.tile(uP[1:N + 1], (B, 1, 1)), zt=np.tile(np.array([0.0, 0, 0, 0, 10.0, 0]), (B, 1)),
                    OldInput=np.zeros((B, 2)), timeStep=np.zeros(B, np.int32), has_pred=np.zeros(B, np.int32))
        c.enable_rollout(Tcl=512)
        x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (B, 1))
        c.rollout_set_state(x0, x0)
        return c
    ca, cb = fresh(), fresh()
    cb.enable_device_books()
    rng = np.random.default_rng(7)
    zs = rng.standard_normal((700, B, 3)) * np.linspace(0.5, 3.0, B)[None, :, None]      # different noise levels -> different lap lengths
    laps_a = [[] for _ in range(B)]

    def step(k):
        ca.rollout_step(z=zs[k]); cb.rollout_step(z=zs[k])
        done, n = ca.rollout_done()
        if done.any():
            for b in np.nonzero(done)[0]:
                laps_a[b].append(int(n[b]))
            ca.rollout_finish_laps(done, n)
        cb.rollout_commit_laps_dev()
        sa, sb = ca.rollout_state(), cb.rollout_state()
        assert np.array_equal(sa["x"], sb["x"]) and np.array_equal(sa["cl_len"], sb["cl_len"]), k

    k = 0
    while min(len(l) for l in laps_a) < 2:
        step(k); k += 1
        assert k < 560
    for _ in range(40):                                     # well into the next lap: lap it-1 has grown by addPoint rows
        step(k); k += 1

    def check_books():
        bk = cb.books()
        for b in range(B):
            host = sorted((ca.LapTime[b][ln], ln) for ln in ca.ss_book[b].slot_of)
            devb = sorted((int(t), int(l)) for t, l in zip(bk["ss_time"][b], bk["ss_lap"][b]) if l >= 0)
            assert host == devb, (b, host, devb)
            assert int(bk["it"][b]) == ca.it[b]
            order = [int(bk["ss_lap"][b][s]) for s in bk["sel"][b]]
            assert order == [int(j) for j in np.argsort(np.array(ca.LapTime[b]), kind="stable")[:numSS_it]], b
            hostm = sorted((T, ln) for T, ln in ca.model_laps[b] if ln in ca.model_book[b].slot_of)
            devm = sorted((int(t), int(q)) for t, q in zip(bk["md_time"][b], bk["md_seq"][b]) if q >= 0)
            assert hostm == devm, (b, hostm, devm)
            assert [int(bk["md_seq"][b][s]) for s in bk["used"][b]] == [ln for _, ln in ca.model_laps[b][:4]], b
            assert list(bk["lap_hist"][b][:len(laps_a[b])]) == laps_a[b]
    check_books()

    # ---- pooled exchange: host books (all laps gathered, Python hand-out) vs device books (fastest few, one kernel)
    rows = torch.zeros(B, Tpad, 9, dtype=torch.float64, device="cuda"); lens = torch.zeros(B, dtype=torch.int32, device="cuda")
    own = [ca.it[b] - 1 for b in range(B)]
    ca.export_laps(own, Tpad, rows, lens)
    times = np.array([ca.LapTime[b][own[b]] for b in range(B)])
    best = [int(i) for i in sharding.pooled_fastest(times, share + 1)]
    for j in range(share):
        src = np.full(B, -1, np.int32); lt = np.zeros(B, np.int64)
        for b in range(B):
            cand = [g for g in best if g != b]
            src[b], lt[b] = cand[j], times[cand[j]]
        ca.import_laps(src, lt, Tpad, rows, lens)
    rows_k = torch.zeros(share + 1, Tpad, 9, dtype=torch.float64, device="cuda"); meta = torch.zeros(share + 1, 4, dtype=torch.int32, device="cuda")
    cb.pool_export(share + 1, Tpad, 0, rows_k, meta)
    took = cb.pool_import(share + 1, share, Tpad, 0, rows_k, meta, count=True)
    m = meta.cpu().numpy()
    assert [int(g) for g in m[:, 2]] == best and [int(t) for t in m[:, 1]] == [int(times[g]) for g in best]
    assert took >= 1
    check_books()
    for _ in range(60):
        step(k); k += 1
    ca.close(); cb.close()


def test_warm_started_closed_loop_matches_cold_start(gold, track):
    """SURVEY §8f rank 2: controllers that start every solve from the shifted mid-path iterate of their previous solve
    (lmpc_params.warm_start) must drive the same closed loop as cold-started ones -- the optimum of each QP is the same, only the
    iteration count changes -- and need fewer interior-point iterations."""
    _need_gpu()
    N, B = 12, 8
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    xP, uP = gold["pid_x"].copy(), gold["pid_u"].copy()

    def fresh(warm):
        c = BatchedController(par, B, track.seg_table(), track.TrackLength, trToUse=4, numSS_Points=numSS_Points,
                              numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1536, ss_cap=7, model_cap=5, warm_start=warm)
        for b in range(B):
            for _ in range(4):
                c.model_add_trajectory(b, xP, uP)
            for _ in range(4):
                c.add_trajectory(b, xP, uP)
        c.set_state(xLin=np.tile(xP[1:N + 2], (B, 1, 1)), uLin=np.tile(uP[1:N + 1], (B, 1, 1)), zt=np.tile(np.array([0.0, 0, 0, 0, 10.0, 0]), (B, 1)),
                    OldInput=np.zeros((B, 2)), timeStep=np.zeros(B, np.int32), has_pred=np.zeros(B, np.int32))
        c.enable_rollout(Tcl=512)
        c.enable_device_books()
        x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (B, 1))
        c.rollout_set_state(x0, x0)
        return c
    cc, cw = fresh(False), fresh(True)
    zs = np.random.default_rng(5).standard_normal((300, B, 3))
    it_c, it_w, worst = [], [], 0.0
    for k in range(300):
        for c, acc in ((cc, it_c), (cw, it_w)):
            c.rollout_step(z=zs[k])
            r = c.step_results()
            assert np.all(r["status"] == 1) and np.all(r["flags"] == 0), (k, r["status"], r["flags"])
            acc.append(r["iters"].mean())
            c.rollout_commit_laps_dev()
        worst = max(worst, np.abs(cc.rollout_state()["x"] - cw.rollout_state()["x"]).max())
    assert worst < 1e-5, worst                                # same optimum every step; the closed loop amplifies 1e-9 a little
    assert list(cc.books()["lap_hist"][:, 0]) == list(cw.books()["lap_hist"][:, 0])
    mc, mw = float(np.mean(it_c[1:])), float(np.mean(it_w[1:]))
    print("interior-point iterations per solve: cold %.2f, warm %.2f" % (mc, mw))
    assert mw < mc - 0.3, (mc, mw)
    cc.close(); cw.close()
