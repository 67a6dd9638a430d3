"""GPU tier: the device's warm-started solves (lmpc_params.warm_start) QP by QP against the host emulation of the same kernel
(tests/support/host_core.cpp), in the device-resident closed loop.

Before every step the controller's warm-start record and its valid flag are read from the buffer table by name ("warm",
"warm_valid"; one record of warm_stride = 2N + 4N ncx + N ncu + 2M + 2 doubles per controller, laid out as Pdip::WS_*:
u [N*2] | s, w1, nu1, nu3 [N*ncx each] | nu2 [N*ncu] | lam, nu4 [M each] | y1, pad), with the QP's x0 (the plant state) and
OldInput; after it, the QP's stage model ("abc") and selected safe set ("SS_sel", "Qfun_sel") and the answer.  Each QP is
re-solved by the host emulation from the device's pre-step record, and warm against cold:
  - status and the valid flag after the step are equal;
  - iteration counts are equal but for a small fraction of QPs (never more than one apart): the host runs the scalar Riccati
    sweeps, the device the tensor-core ones, so rounding differs;
  - the answers agree to 1e-8, and the device's warm answer is within 1e-6 of the host's cold one, wherever no solve is a late
    accept; the device's late accepts (lmpc_late_accepts) are printed.
Events that must drop every record (each write of d_warm_valid in csrc/lmpc_b200.cu apart from the kernel's own): a new
controller state (lmpc_state_set) and new parameter sets (lmpc_set_param_sets) leave every valid flag at 0, and after a change of
problem type between steps every flag is at most 1 (each solve of that step started cold) (a solve without a usable record is bit for bit a cold solve:
tests/test_warm_start.py).  The seeding calls (lmpc_rollout_seed_from_record / _dev) clear the flags the same way; they are
not exercised here."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp          # noqa: E402
from racinglmpc_b200.controller import BatchedController     # noqa: E402
import hostcore as hc                                        # noqa: E402

B, N, STEPS = 16, 12, 40
# measured on an H100 80GB HBM3 (700 W): 1 of 1280 QPs (0.08 %) one iteration apart, profiles/h100_warm_start_host_vs_device.txt
MAX_ITER_MISMATCH = 0.01


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _controller(gold, track, warm=True):
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    xP, uP = gold["pid_x"].copy(), gold["pid_u"].copy()
    c = BatchedController(par, B, track.seg_table(), track.TrackLength, trToUse=4, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1536, ss_cap=7, model_cap=5, warm_start=warm)
    for b in range(B):
        for _ in range(4):
            c.model_add_trajectory(b, xP, uP)
        for _ in range(4):
            c.add_trajectory(b, xP, uP)
    c.set_state(xLin=np.tile(xP[1:N + 2], (B, 1, 1)), uLin=np.tile(uP[1:N + 1], (B, 1, 1)),
                zt=np.tile(np.array([0.0, 0, 0, 0, 10.0, 0]), (B, 1)), OldInput=np.zeros((B, 2)),
                timeStep=np.zeros(B, np.int32), has_pred=np.zeros(B, np.int32))
    c.enable_rollout(Tcl=512)
    c.enable_device_books()
    x0 = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (B, 1))
    c.rollout_set_state(x0, x0)
    return c, par, Qts, numSS_Points


def _stride(c, M):
    return N * 2 + 4 * N * 2 + N * 4 + 2 * M + 2


def _valid(c):
    return np.array([c.read_buffer("warm_valid", b, (1,), np.int32)[0] for b in range(B)])


def _late(status, resid):
    return status == 1 and (max(resid[0], resid[1]) > 1.000001e-9 or resid[2] > 1.000001e-11)


def test_device_record_equals_host_record(gold, track):
    """LMPC steps at (N, M) = (12, 48), then LTV-MPC steps (mode 0, the <12, 0> kernel) on the same controllers: every QP
    re-solved by the host emulation from the device's pre-step record."""
    _need_gpu()
    c, par, Qts, M = _controller(gold, track)
    stride = _stride(c, M)
    zs = np.random.default_rng(11).standard_normal((2 * STEPS, B, 3))
    stats = dict(qps=0, iter_mismatch=0, late_dev=0, restarts=0, warm_started=0)
    worst = 0.0
    for k in range(2 * STEPS):
        mode = 1 if k < STEPS else 0
        const = hc.make_const(par, Qts)
        x0 = c.rollout_state()["x"].copy()
        old = np.stack([c.read_buffer("OldInput", b, (2,)) for b in range(B)])
        rec = np.stack([c.read_buffer("warm", b, (stride,)) for b in range(B)])
        v_in = _valid(c)
        if k == STEPS:
            v_in[:] = 0                     # the change of problem type drops the records before the QP (checked below)
        c.rollout_step(z=zs[k], mode=mode)
        r = c.step_results()
        v_out = _valid(c)
        if k == STEPS:
            assert np.all(v_out <= 1), v_out
        abc = c.read_buffer("abc", 0, (B, N, 54))
        xp, up = c.read_buffer("xPred", 0, (B, N + 1, 6)), c.read_buffer("uPred", 0, (B, N, 2))
        SS = c.read_buffer("SS_sel", 0, (B, 6, M)) if mode == 1 else None
        Qf = c.read_buffer("Qfun_sel", 0, (B, M)) if mode == 1 else None
        for b in range(B):
            buf = np.zeros(4096); buf[:stride] = rec[b]
            w = {"buf": buf, "valid": np.array([v_in[b]], np.int32)}
            args = (const, N, abc[b], x0[b], old[b]) + ((SS[b], Qf[b]) if mode == 1 else ())
            hw = hc.solve(*args, warm=w)
            hcold = hc.solve(*args)
            assert hw["status"] == r["status"][b], (k, b, hw["status"], r["status"][b])
            assert int(w["valid"][0]) == v_out[b], (k, b, v_in[b], int(w["valid"][0]), v_out[b])
            d_it = abs(hw["iters"] - int(r["iters"][b]))
            assert d_it <= 1, (k, b, hw["iters"], r["iters"][b])
            stats["qps"] += 1
            stats["iter_mismatch"] += int(d_it != 0)
            stats["warm_started"] += int(1 <= v_in[b] <= 8)
            stats["restarts"] += int(1 <= v_in[b] <= 8 and r["iters"][b] >= 16)
            dev_late = _late(int(r["status"][b]), r["resid"][b])
            stats["late_dev"] += int(dev_late)
            if not (dev_late or _late(hw["status"], (hw["r_prim"], hw["r_dual"], hw["gap"]))):
                err = max(np.abs(xp[b] - hw["x"]).max(), np.abs(up[b] - hw["u"]).max())
                assert err < 1e-8, (k, b, err)
                worst = max(worst, err)
                if not _late(hcold["status"], (hcold["r_prim"], hcold["r_dual"], hcold["gap"])):
                    assert max(np.abs(xp[b] - hcold["x"]).max(), np.abs(up[b] - hcold["u"]).max()) < 1e-6, (k, b)
    frac = stats["iter_mismatch"] / stats["qps"]
    print("host vs device: %d QPs (%d warm-started, %d restarted), iteration mismatches %d (%.4f), device late accepts %d "
          "(lmpc_late_accepts %d), max |dz| %.2e" % (stats["qps"], stats["warm_started"], stats["restarts"], stats["iter_mismatch"],
                                                   frac, stats["late_dev"], c.late_accepts, worst))
    assert stats["warm_started"] > stats["qps"] // 2
    assert frac <= MAX_ITER_MISMATCH, frac
    c.close()


def test_events_drop_every_record(gold, track):
    """A new controller state, new parameter sets and a change of problem type each leave every valid flag at 0 (the next solve
    of every controller starts cold)."""
    _need_gpu()
    c, par, Qts, M = _controller(gold, track)
    zs = np.random.default_rng(12).standard_normal((12, B, 3))

    def warm_up(k0, mode=1):
        for k in range(3):
            c.rollout_step(z=zs[k0 + k], mode=mode)
        assert np.any(_valid(c) > 0)

    warm_up(0)
    numSS_it, numSS_Points, _, _, Qts2, par2 = rp.lmpc_params(N)
    c.set_param_sets([par2], np.zeros(B, int), QterminalSlack=[Qts2])
    assert np.all(_valid(c) == 0), "lmpc_set_param_sets"
    warm_up(3)
    xLin = np.stack([c.read_buffer("xLin", b, (N + 1, 6)) for b in range(B)])
    uLin = np.stack([c.read_buffer("uLin", b, (N, 2)) for b in range(B)])
    c.set_state(xLin=xLin, uLin=uLin, zt=np.tile(np.array([0.0, 0, 0, 0, 10.0, 0]), (B, 1)), OldInput=np.zeros((B, 2)),
                timeStep=np.zeros(B, np.int32), has_pred=np.zeros(B, np.int32))
    assert np.all(_valid(c) == 0), "lmpc_state_set"
    warm_up(6)
    c.rollout_step(z=zs[9], mode=0)            # the records of LMPC-type QPs are dropped before the first LTV-MPC QP
    assert np.all(_valid(c) <= 1), "change of problem type"
    c.close()
