"""GPU tier: per-controller vehicles of the device simulator (lmpc_rollout_set_vehicles).

A batch of several cars is several one-car batches in one launch: every controller's closed loop (PID lap, seeding, LMPC laps) is
bit-identical to that of a same-size handle on which every controller drives its car.  Checked for a plain batch, for a traced
batch (the trace kernel runs between the solve and the simulator) and for a crossed design of QP tunings x vehicles.  The
heterogeneous PID lap is checked against dynModel on each car (tests/support/vehicle_model.py), and the reference car installed
as one set against a handle without sets."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import workloads, reference_params as rp    # noqa: E402
from racinglmpc_b200 import _native as nat                       # noqa: E402
from racinglmpc_b200.controller import BatchedController         # noqa: E402
from racinglmpc_b200.reference_params import VehicleParams       # noqa: E402
from oracle import vehicle as ov                                 # noqa: E402
import closed_loop as cl                                         # noqa: E402
import vehicle_model as vm                                       # noqa: E402
from closed_loop import N, X0                                    # noqa: E402

LMPC_E_INVALID = -1


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def golden_vehicles():
    """The eight cars of tests/golden/vehicle_golden.npz (the reference, other friction, mass, axle split and tyres)."""
    vg = np.load(workloads._GOLD + "/vehicle_golden.npz")
    return [VehicleParams(*row) for row in vg["vehicles"]]


FOUR = [VehicleParams.reference(), VehicleParams.from_friction(0.6), VehicleParams.from_friction(1.0, m=2.4, Iz=0.029),
        VehicleParams.from_friction(0.8, lf=0.10, lr=0.15)]


def test_heterogeneous_pid_lap_matches_dyn_model_on_every_car(track):
    """Eight cars interleaved, host-given draws: one PID step to 1e-12 in both frames, a 300-step PID lap to 1e-9."""
    _need_gpu()
    vs = golden_vehicles()
    B, K = 2 * len(vs), 300
    idx = np.arange(B) % len(vs)
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, B, track.seg_table(), track.TrackLength, trToUse=4, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=1536, ss_cap=6, model_cap=5)
    c.set_vehicles(vs, idx)
    c.enable_rollout(Tcl=1024)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    zs = np.random.default_rng(7).standard_normal((B, K, 5))
    for k in range(K):
        c.rollout_pid_step(0.8, z_pid=zs[:, k, 0:2], z_sim=zs[:, k, 2:5])
        if k == 0:
            st = c.rollout_state()
            for b in range(B):
                it = iter(zs[b, 0])
                fake = type("R", (), {"standard_normal": lambda self, it=it: next(it)})()
                pid = ov.PIDFollower(0.8, rng=fake)
                pid.solve(X0)
                xo, go = vm.dyn_model(track, X0, X0, pid.uPred[0], vs[idx[b]], rng=fake)
                assert np.max(np.abs(st["x"][b] - xo)) < 1e-12 and np.max(np.abs(st["xglob"][b] - go)) < 1e-12, b
    st = c.rollout_state()
    assert np.all(st["cl_len"] == K)
    for b in range(B):
        it = iter(zs[b].ravel())
        fake = type("R", (), {"standard_normal": lambda self, it=it: next(it)})()
        xo, uo, go, last = vm.closed_loop(track, [X0, X0], ov.PIDFollower(0.8, rng=fake), vs[idx[b]], max_steps=K, rng=fake)
        xg, ug = c.rollout_get_lap(b)
        assert np.max(np.abs(xg - xo)) < 1e-9 and np.max(np.abs(ug - uo)) < 1e-9, b
        # the state after the last step, both frames
        assert np.max(np.abs(st["x"][b] - last[0])) < 1e-9 and np.max(np.abs(st["xglob"][b] - last[1])) < 1e-9, b
    # the cars drive differently
    assert np.abs(st["x"][idx == 1, 4] - st["x"][idx == 0, 4]).max() > 1e-3
    c.close()


@pytest.fixture(scope="module")
def uniform_runs():
    """Reference closed loops: B = 256, every controller on one of FOUR, steps set by the heterogeneous run."""
    _need_gpu()
    B = 256
    vidx = np.arange(B) % 4

    def reject(c):                                  # rejected calls leave the handle as it was
        L, good = nat.lib(), nat.make_vehicle_sets(FOUR, vidx, B)
        bad = (nat.VehicleParams * 4)()
        C.memmove(bad, good[0], C.sizeof(bad))
        bad[2].Iz = 0.0
        nan = (nat.VehicleParams * 4)()
        C.memmove(nan, good[0], C.sizeof(nan))
        nan[1].Br = float("nan")
        cases = [(bad, 4, good[1]), (nan, 4, good[1]), (good[0], 4, np.full(B, 4, np.int32)), (good[0], 4, np.full(B, -1, np.int32)),
                 (good[0], 0, good[1]), (None, 4, good[1]), (good[0], 4, None)]
        for tab, n, ix in cases:
            assert L.lmpc_rollout_set_vehicles(c._h, tab, n, nat.ptr(ix) if ix is not None else None) == LMPC_E_INVALID
        big = (nat.VehicleParams * (B + 1))(*([good[0][0]] * (B + 1)))
        assert L.lmpc_rollout_set_vehicles(c._h, big, B + 1, nat.ptr(np.zeros(B, np.int32))) == LMPC_E_INVALID

    n, het, het_laps = cl.run(B, vehicles=FOUR, vidx=vidx, hook=reject)
    assert het["lap_n"].min() >= 1, "not every controller finished an LMPC lap in %d steps" % n
    refs = [cl.run(B, vehicles=[v], vidx=np.zeros(B, np.int32), steps=n)[1:] for v in FOUR]
    return dict(B=B, n=n, vidx=vidx, het=(het, het_laps), refs=refs)


def test_closed_loop_vehicles_bit_identical_to_one_car_handles(uniform_runs):
    """A batch of four cars equals four one-car handles; invalid calls before the run changed nothing."""
    u = uniform_runs
    for k in range(4):
        cl.same(u["het"], u["refs"][k], u["vidx"] == k, "vehicle %d" % k)
    # the cars drove different laps
    h = u["het"][0]
    assert len({float(h["lap_hist"][u["vidx"] == k, 0].mean()) for k in range(4)}) == 4


def test_traced_batch_gives_the_same_results(uniform_runs):
    """The trace kernel between the solve and the simulator changes nothing the controllers compute."""
    u = uniform_runs
    _, het, laps = cl.run(u["B"], vehicles=FOUR, vidx=u["vidx"], steps=u["n"], trace=True)
    for k in range(4):
        cl.same((het, laps), u["refs"][k], u["vidx"] == k, "traced, vehicle %d" % k)


def test_reference_car_as_one_set_equals_no_sets_and_revert(uniform_runs):
    u = uniform_runs
    B, n = u["B"], u["n"]
    none = cl.run(B, steps=n)[1:]
    everything = np.ones(B, bool)
    cl.same(none, u["refs"][0], everything, "reference as one set vs no sets")

    def install_then_revert(c):
        c.set_vehicles(FOUR, u["vidx"])
        with pytest.raises(ValueError):
            c.set_vehicles(None, u["vidx"])        # reverting takes no index
        with pytest.raises(ValueError):
            c.set_vehicles(FOUR)                   # vehicles need one
        c.set_vehicles(None)

    reverted = cl.run(B, hook=install_then_revert, steps=n)[1:]
    cl.same(reverted, none, everything, "nsets == 0 reverts")


def test_crossed_tunings_and_vehicles():
    """Two QP tunings x two cars, indices independent of each other, against the four single-tuning, single-car handles."""
    _need_gpu()
    B = 256
    _, _, _, _, Qts, base = rp.lmpc_params(N)
    ps, qs = [], []
    for k in range(2):
        p = copy.deepcopy(base)
        p.Qslack = (0.5, 2.0)[k] * np.asarray(base.Qslack, float)
        p.dR = (2.0, 0.5)[k] * np.asarray(base.dR, float)
        ps.append(p)
        qs.append((1.0, 0.5)[k] * Qts)
    cars = [FOUR[0], FOUR[1]]
    pidx = np.arange(B) % 2
    vidx = (np.arange(B) // 2) % 2
    n, het, het_laps = cl.run(B, vehicles=cars, vidx=vidx, psets=(ps, pidx, qs))
    assert het["lap_n"].min() >= 1
    for i in range(2):
        for j in range(2):
            ref = cl.run(B, vehicles=[cars[j]], vidx=np.zeros(B, np.int32), par=ps[i], qts=qs[i], steps=n)[1:]
            cl.same((het, het_laps), ref, (pidx == i) & (vidx == j), "tuning %d, vehicle %d" % (i, j))
