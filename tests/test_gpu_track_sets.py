"""GPU tier: per-controller tracks (lmpc_set_tracks).

A batch on several circuits is several one-circuit batches in one launch: every controller's closed loop (PID lap, seeding, LMPC
laps) is bit-identical to that of a same-size handle created with its circuit.  Checked through all three places the simulator
runs from (the fused step tail, the unfused step of a traced batch, the step cut into instance ranges), for the host-driven
regression (K1) and safe-set selection (K2), and for a crossed design of circuits x cars x QP tunings.  The heterogeneous PID lap
is checked against dynModel on each circuit (tests/support/track_model.py, vehicle_model.py), the reference track installed as
one set against a handle without sets, and the refusals (malformed tables, laps already stored, pooled exchange on several
circuits) against the handle's state."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import workloads, reference_params as rp    # noqa: E402
from racinglmpc_b200 import _native as nat                       # noqa: E402
from racinglmpc_b200.controller import BatchedController         # noqa: E402
from racinglmpc_b200.reference_params import TrackParams, VehicleParams   # noqa: E402
from oracle import vehicle as ov, ltv_model                      # noqa: E402
import track_model                                               # noqa: E402
import vehicle_model as vm                                       # noqa: E402

N = 12
LMPC_E_INVALID, LMPC_E_STATE = -1, -4
X0 = np.array([0.5, 0, 0, 0, 0, 0.0])
THREE = [TrackParams.l_shaped(), TrackParams.goggle(), TrackParams.oval()]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _ctrl(B, track=None, par=None, qts=None, trToUse=4, ss_cap=7, model_cap=5, Tmax=1280):
    """A controller created with `track` (default: the reference's L track) through lmpc_store_create."""
    numSS_it, numSS_Points, _, _, Qts, base = rp.lmpc_params(N)
    track = THREE[0] if track is None else track
    return BatchedController(base if par is None else par, B, track.seg_table, track.TrackLength, trToUse=trToUse,
                             numSS_Points=numSS_Points, numSS_it=numSS_it, QterminalSlack=Qts if qts is None else qts,
                             Tmax=Tmax, ss_cap=ss_cap, model_cap=model_cap)


class _Fake:
    def __init__(self, z):
        self._it = iter(np.asarray(z, float).ravel())

    def standard_normal(self):
        return next(self._it)


def test_heterogeneous_pid_lap_matches_dyn_model_on_every_track():
    """Three circuits interleaved, the same host-given draws for the controllers b, b + 3, b + 6 ...: one PID step to 1e-12 in
    both frames, a 300-step PID lap to 1e-9; controllers with the same draws on different circuits end at different s."""
    _need_gpu()
    B, K = 12, 300
    idx = np.arange(B) % 3
    c = _ctrl(B, Tmax=1536, ss_cap=6)
    c.set_tracks(THREE, idx)
    c.enable_rollout(Tcl=1024)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    zs = np.random.default_rng(7).standard_normal((B // 3, K, 5))[np.arange(B) // 3]
    maps = [track_model.from_table(t.table6) for t in THREE]
    for k in range(K):
        c.rollout_pid_step(0.8, z_pid=zs[:, k, 0:2], z_sim=zs[:, k, 2:5])
        if k == 0:
            st = c.rollout_state()
            for b in range(B):
                fake = _Fake(zs[b, 0])
                pid = ov.PIDFollower(0.8, rng=fake)
                pid.solve(X0)
                xo, go = vm.dyn_model(maps[idx[b]], X0, X0, pid.uPred[0], VehicleParams.reference(), rng=fake)
                assert np.max(np.abs(st["x"][b] - xo)) < 1e-12 and np.max(np.abs(st["xglob"][b] - go)) < 1e-12, b
    st = c.rollout_state()
    assert np.all(st["cl_len"] == K)
    for b in range(B):
        fake = _Fake(zs[b])
        xo, uo, go, last = vm.closed_loop(maps[idx[b]], [X0, X0], ov.PIDFollower(0.8, rng=fake), VehicleParams.reference(),
                                          max_steps=K, rng=fake)
        xg, ug = c.rollout_get_lap(b)
        assert np.max(np.abs(xg - xo)) < 1e-9 and np.max(np.abs(ug - uo)) < 1e-9, b
        assert np.max(np.abs(st["x"][b] - last[0])) < 1e-9 and np.max(np.abs(st["xglob"][b] - last[1])) < 1e-9, b
    for g in range(B // 3):
        s = st["x"][3 * g:3 * g + 3, 4]
        assert len(set(s.tolist())) == 3, s
    c.close()


def test_host_driven_regression_and_selection_per_track():
    """lmpc_identify_host / lmpc_select_host of a three-circuit batch equal those of one-circuit handles bit for bit (lap-wrap
    fix and Q-function shift included), and the regression matches the oracle's LocalLTVModel on each circuit."""
    _need_gpu()
    B = 48
    data = workloads.lmpc_batch(B)
    idx = np.arange(B) % 3
    het = _ctrl(B, trToUse=5, ss_cap=6, model_cap=6, Tmax=1536)
    het.set_tracks(THREE, idx)
    workloads.restore_lmpc_batch(het, data)
    abc, flags = het.identify()
    sel = het.select(data["x0"])
    het.close()
    outs = []
    for k, t in enumerate(THREE):
        c = _ctrl(B, track=t, trToUse=5, ss_cap=6, model_cap=6, Tmax=1536)
        workloads.restore_lmpc_batch(c, data)
        ra, rf = c.identify()
        rs = c.select(data["x0"])
        c.close()
        m = idx == k
        assert np.array_equal(abc[m], ra[m]) and np.array_equal(flags[m], rf[m]), k
        for key, v in sel.items():
            assert np.array_equal(v[m], rs[key][m]), (k, key)
        outs.append((ra, rs))
    # the circuit matters: the oval's curvature changes the model
    m2 = idx == 2
    assert not np.array_equal(outs[2][0][m2], outs[0][0][m2])
    for b in (0, 1, 2, 4, 5):
        pm = ltv_model.LocalLTVModel(6, 2, track_model.from_table(THREE[idx[b]].table6), 5)
        pm.xStored = [lx for lx, _ in data["model_laps"][b]]
        pm.uStored = [lu for _, lu in data["model_laps"][b]]
        pm.lapTime = [lx.shape[0] for lx in pm.xStored]
        for i in range(N):
            A, Bm, Cc = pm.regressionAndLinearization(data["xLin"][b][i], data["uLin"][b][i])
            assert np.max(np.abs(abc[b, i, 0:36] - A.ravel())) < 1e-8, (b, i)
            assert np.max(np.abs(abc[b, i, 36:48] - Bm.ravel())) < 1e-8, (b, i)
            assert np.max(np.abs(abc[b, i, 48:54] - Cc)) < 1e-8, (b, i)


def test_ss_put_lap_cost_uses_each_tracks_length():
    """LMPC.computeCost on the device (lmpc_ss_put_lap with qfun NULL) counts down to the controller's own finish line."""
    _need_gpu()
    B = 3
    c = _ctrl(B, ss_cap=6)
    c.set_tracks(THREE, np.arange(B))
    x, u, _ = workloads.lmpc_batch(1)["ss_laps"][0][0]          # a lap grown past the L track's finish line
    x, u = np.ascontiguousarray(x), np.ascontiguousarray(u)
    L = nat.lib()
    for b in range(B):
        nat.check(L.lmpc_ss_put_lap(c._h, b, 0, x.shape[0], nat.ptr(x), nat.ptr(u), None))
        T = C.c_int(0)
        q = np.zeros(1536)
        nat.check(L.lmpc_ss_get_lap(c._h, b, 0, C.byref(T), None, None, nat.ptr(q)))
        ref = np.zeros(x.shape[0])                               # PC.py:447-464
        for j in range(x.shape[0] - 2, -1, -1):
            ref[j] = ref[j + 1] + 1 if x[j, 4] < THREE[b].TrackLength else 0
        assert np.array_equal(q[:T.value], ref), b
    c.close()


def _closed_loop(B, track=None, tracks=None, tidx=None, vehicles=None, vidx=None, par=None, qts=None, psets=None, steps=None,
                 trace=False, hook=None):
    """Device PID lap (Philox), seeding, then LMPC rollout steps until every controller has finished one LMPC lap (or `steps`
    steps).  `hook(c)` runs once the tables are installed."""
    c = _ctrl(B, track=track, par=par, qts=qts)
    if psets is not None:
        c.set_param_sets(*psets)
    if vehicles is not None:
        c.set_vehicles(vehicles, vidx)
    if tracks is not None:
        c.set_tracks(tracks, tidx)
    if hook is not None:
        hook(c)
    c.enable_rollout(Tcl=1024)
    if trace:
        inst = np.array([0, 1, 2, 3], np.int32)
        nat.check(nat.lib().lmpc_rollout_trace_create(c._h, len(inst), nat.ptr(inst), 16))
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
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


KEYS = ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt", "flags", "unsolved")


def _same(a, b, sel, what):
    a_run, a_laps = a
    b_run, b_laps = b
    for key in KEYS:
        assert np.array_equal(a_run[key][sel], b_run[key][sel]), (what, key)
    for (i, slot), v in a_laps.items():
        if sel[i] and (i, slot) in b_laps:
            assert all(np.array_equal(p, q) for p, q in zip(v, b_laps[(i, slot)])), (what, i, slot)


def _bad_sets(good, B):
    """Malformed tables and indices that lmpc_set_tracks must refuse with LMPC_E_INVALID."""
    def edited(k, f):
        t = (nat.TrackParams * 3)()
        C.memmove(t, good[0], C.sizeof(t))
        f(t[k])
        return t
    tabs = [edited(0, lambda r: setattr(r, "nseg", 0)), edited(1, lambda r: setattr(r, "nseg", 17)),
            edited(2, lambda r: r.seg.__setitem__(5, float("nan"))), edited(1, lambda r: setattr(r, "TrackLength", float("inf"))),
            edited(2, lambda r: r.seg.__setitem__(4, -r.seg[4])), edited(0, lambda r: r.seg.__setitem__(0, 1e-12)),
            edited(1, lambda r: r.seg.__setitem__(9, np.nextafter(r.seg[9], 0))),
            edited(2, lambda r: setattr(r, "TrackLength", np.nextafter(r.TrackLength, 0)))]
    cases = [(t, 3, good[1]) for t in tabs]
    cases += [(good[0], 3, np.full(B, 3, np.int32)), (good[0], 3, np.full(B, -1, np.int32)), (good[0], 0, good[1]),
              (None, 3, good[1]), (good[0], 3, None)]
    return cases


@pytest.fixture(scope="module")
def uniform_runs():
    """Reference closed loops: B = 256, controller b on circuit b mod 3, steps set by the heterogeneous fused run."""
    _need_gpu()
    B = 256
    tidx = np.arange(B) % 3

    def reject(c):                                  # rejected calls leave the handle as it was
        L, good = nat.lib(), nat.make_track_sets(THREE, tidx, B)
        for tab, n, ix in _bad_sets(good, B):
            assert L.lmpc_set_tracks(c._h, tab, n, nat.ptr(ix) if ix is not None else None) == LMPC_E_INVALID

    n, het, het_laps = _closed_loop(B, tracks=THREE, tidx=tidx, hook=reject)
    assert het["lap_n"].min() >= 1, "not every controller finished an LMPC lap in %d steps" % n
    refs = [_closed_loop(B, track=t, steps=n)[1:] for t in THREE]
    return dict(B=B, n=n, tidx=tidx, het=(het, het_laps), refs=refs)


def test_closed_loop_tracks_bit_identical_to_one_track_handles(uniform_runs):
    """Default path: the simulator runs in the fused step tail; invalid calls before the run changed nothing."""
    u = uniform_runs
    for k in range(3):
        _same(u["het"], u["refs"][k], u["tidx"] == k, "fused, track %d" % k)
    h = u["het"][0]
    assert len({float(h["lap_hist"][u["tidx"] == k, 0].mean()) for k in range(3)}) == 3


def test_traced_batch_runs_the_unfused_simulator_with_the_same_results(uniform_runs):
    u = uniform_runs
    _, het, laps = _closed_loop(u["B"], tracks=THREE, tidx=u["tidx"], steps=u["n"], trace=True)
    for k in range(3):
        _same((het, laps), u["refs"][k], u["tidx"] == k, "traced, track %d" % k)


def test_step_cut_into_instance_ranges_gives_the_same_results(uniform_runs, monkeypatch):
    """LMPC_B200_STEP_SPLIT=2 on 512 controllers: the first 256 must match the 256-controller references."""
    u = uniform_runs
    monkeypatch.setenv("LMPC_B200_STEP_SPLIT", "2")
    B2 = 2 * u["B"]
    _, het, laps = _closed_loop(B2, tracks=THREE, tidx=np.arange(B2) % 3, steps=u["n"])
    first = {k: (v[:u["B"]] if np.ndim(v) and len(v) == B2 else v) for k, v in het.items()}
    first_laps = {key: v for key, v in laps.items() if key[0] < u["B"]}
    for k in range(3):
        _same((first, first_laps), u["refs"][k], u["tidx"] == k, "split, track %d" % k)


def test_reference_track_as_one_set_equals_no_sets_and_revert(uniform_runs):
    u = uniform_runs
    B, n = u["B"], u["n"]
    everything = np.ones(B, bool)
    one = _closed_loop(B, tracks=[THREE[0]], tidx=np.zeros(B, np.int32), steps=n)[1:]
    _same(one, u["refs"][0], everything, "reference track as one set vs no sets")

    def install_then_revert(c):
        c.set_tracks(THREE, u["tidx"])
        with pytest.raises(ValueError):
            c.set_tracks(None, u["tidx"])          # reverting takes no index
        with pytest.raises(ValueError):
            c.set_tracks(THREE)                    # tracks need one
        c.set_tracks(None)

    reverted = _closed_loop(B, track=THREE[2], hook=install_then_revert, steps=n)[1:]
    _same(reverted, u["refs"][2], everything, "nsets == 0 reverts to the handle's own track")


def test_crossed_tracks_vehicles_and_tunings():
    """Two circuits x two cars x two lane widths (bx through lmpc_set_param_sets), three independent indices, against the eight
    one-circuit, one-car, one-tuning handles."""
    _need_gpu()
    B = 256
    _, _, _, _, Qts, base = rp.lmpc_params(N)
    ps = []
    for w in (0.4, 0.3):
        p = copy.deepcopy(base)
        p.bx = np.array([w, w])
        ps.append(p)
    cars = [VehicleParams.reference(), VehicleParams.from_friction(0.6)]
    tracks = [THREE[0], THREE[2]]
    b = np.arange(B)
    tidx, vidx, pidx = b % 2, (b // 2) % 2, (b // 4) % 2
    n, het, het_laps = _closed_loop(B, tracks=tracks, tidx=tidx, vehicles=cars, vidx=vidx, psets=(ps, pidx, [Qts, Qts]))
    assert het["lap_n"].min() >= 1
    for i in range(2):
        for j in range(2):
            for k in range(2):
                ref = _closed_loop(B, track=tracks[k], vehicles=[cars[j]], vidx=np.zeros(B, np.int32), par=ps[i], steps=n)[1:]
                _same((het, het_laps), ref, (pidx == i) & (vidx == j) & (tidx == k), "tuning %d, car %d, track %d" % (i, j, k))


def test_refusals():
    """Before lmpc_store_create and once a lap is stored: LMPC_E_STATE.  The pooled exchange with two circuits: LMPC_E_STATE on
    both sides; with one circuit installed it runs."""
    _need_gpu()
    L = nat.lib()
    B = 8
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    p = nat.make_params(par, numSS_Points, numSS_it, Qts)
    h = C.c_void_p()
    nat.check(L.lmpc_create(C.byref(p), B, 0, C.byref(h)))
    sets, idx = nat.make_track_sets(THREE, np.arange(B) % 3, B)
    assert L.lmpc_set_tracks(h, sets, 3, nat.ptr(idx)) == LMPC_E_STATE
    L.lmpc_destroy(h)

    # a stored lap fixes the tracks: put_lap and device seeding
    x, u, _ = workloads.lmpc_batch(1)["ss_laps"][0][0]
    x, u = np.ascontiguousarray(x), np.ascontiguousarray(u)
    c = _ctrl(B)
    nat.check(L.lmpc_model_put_lap(c._h, 0, 0, x.shape[0], nat.ptr(x), nat.ptr(u)))
    assert L.lmpc_set_tracks(c._h, sets, 3, nat.ptr(idx)) == LMPC_E_STATE
    assert L.lmpc_set_tracks(c._h, None, 0, None) == LMPC_E_STATE
    c.close()

    def seeded(tracks):
        c = _ctrl(B)
        c.set_tracks(tracks, np.arange(B) % len(tracks))
        c.enable_rollout(Tcl=1024)
        c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
        for _ in range(300):
            c.rollout_pid_step(0.8, seed=11)
        c.rollout_seed_from_record_dev(copies=4)
        c.sync()
        return c

    dev = torch.device("cuda", 0)
    rows = torch.zeros(3, 288, 9, dtype=torch.float64, device=dev)
    meta = torch.zeros(3, 4, dtype=torch.int32, device=dev)
    two = seeded(THREE[:2])
    assert L.lmpc_set_tracks(two._h, sets, 3, nat.ptr(idx)) == LMPC_E_STATE
    assert L.lmpc_pool_export_dev(two._h, 3, 288, 0, nat.ptr(rows), nat.ptr(meta)) == LMPC_E_STATE
    assert L.lmpc_pool_import_dev(two._h, 3, 2, 288, 0, nat.ptr(rows), nat.ptr(meta), None) == LMPC_E_STATE
    zeros = np.zeros(B, np.int32)
    assert L.lmpc_ss_import_laps_dev(two._h, nat.ptr(zeros), None, nat.ptr(zeros), 1, 288, nat.ptr(rows), nat.ptr(meta)) == LMPC_E_STATE
    two.close()
    one = seeded([THREE[2]])
    one.pool_export(3, 288, 0, rows, meta)
    assert one.pool_import(3, 2, 288, 0, rows, meta, count=True) >= 0
    one.close()


def test_malformed_table_leaves_the_handle_as_it_was():
    """A refused call between two steps changes nothing: the next step equals that of a handle that never saw it."""
    _need_gpu()
    B = 6
    tidx = np.arange(B) % 3

    def run(refuse):
        c = _ctrl(B)
        c.set_tracks(THREE, tidx)
        if refuse:
            good = nat.make_track_sets(list(reversed(THREE)), tidx, B)
            for tab, n, ix in _bad_sets(good, B):
                assert nat.lib().lmpc_set_tracks(c._h, tab, n, nat.ptr(ix) if ix is not None else None) == LMPC_E_INVALID
        c.enable_rollout(Tcl=64)
        c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
        for _ in range(40):
            c.rollout_pid_step(0.8, seed=3)
        st = c.rollout_state()
        c.close()
        return st

    a, b = run(False), run(True)
    for key in ("x", "xglob", "cl_len", "done"):
        assert np.array_equal(a[key], b[key]), key
