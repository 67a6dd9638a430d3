"""GPU tier: a controller whose plant state stops being finite stays contained.

One controller of a batch gets a NaN or inf (or 1e300) in its state after the PID lap, the seeding and a few closed-loop steps.
Every call keeps returning OK; in independent mode every other controller's state, record, lap books, health and prediction are
bit for bit those of the same batch without the injection, in modes 1, 0 and 2 and with per-controller shapes and measurement noise;
the diverged controller reports it (health bit 512 when addPoint refuses its point, 128 when the plant's curvature lookup fails, and
unsolved steps).  Pooled: a diverged controller that holds the fastest latest lap of its pool group hands no non-finite row to any
importer, and a second group is untouched."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                 # noqa: E402
from racinglmpc_b200 import _native as nat                         # noqa: E402
from racinglmpc_b200.controller import BatchedController           # noqa: E402
from racinglmpc_b200.reference_params import MeasurementParams, TrackParams   # noqa: E402

X0 = np.array([0.5, 0, 0, 0, 0, 0.0])
TRACK = TrackParams.l_shaped()
B = 16
K = 5                                                   # the controller that diverges
INJECT = {"nan vx": (0, np.nan), "nan ey": (5, np.nan), "inf s": (4, np.inf), "1e300 vx": (0, 1e300)}
SHAPES = [(12, 48), (14, 96), (12, 24)]
SENSOR = MeasurementParams((0.01, 0.01, 0.01, 0.005, 0.01, 0.01), (0.05, 0.05, 0.05, 0.025, 0.05, 0.05))


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _seeded(shaped=False, groups=None):
    """A batch after the device PID lap and the seeding, back at the start line"""
    N, M = (14, 96) if shaped else (12, 48)
    numSS_it, _, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, B, TRACK.seg_table, TRACK.TrackLength, trToUse=4, numSS_Points=M, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=1280, ss_cap=7, model_cap=5)
    c.enable_rollout(Tcl=1024)
    if shaped:
        c.set_shapes(SHAPES, np.arange(B) % len(SHAPES))
        c.set_measurement_noise([SENSOR], np.zeros(B, int))
    c.set_noise_streams(np.arange(B))
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    if groups is not None:
        c.set_pool_groups(groups)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    return c


def _inject(c, inst, what):
    ch, v = INJECT[what]
    st = c.rollout_state()
    x = st["x"].copy()
    x[inst, ch] = v
    c.rollout_set_state(x, st["xglob"])


def _step(c, mode):
    c.rollout_step(seed=77, mode=mode)
    c.rollout_commit_laps_dev()


def _stored_laps(c, inst):
    """Every safe-set lap the device books hold for controller `inst`: (x, u, Qfun) per occupied slot"""
    out = []
    for slot, lap in enumerate(c.books()["ss_lap"][inst]):
        if lap < 0:
            continue
        T = C.c_int(0)
        x, u, q = np.zeros((c.Tmax, 6)), np.zeros((c.Tmax, 2)), np.zeros(c.Tmax)
        nat.check(c._lib.lmpc_ss_get_lap(c._h, int(inst), slot, C.byref(T), nat.ptr(x), nat.ptr(u), nat.ptr(q)))
        out.append((x[:T.value], u[:T.value], q[:T.value]))
    return out


def _result(c):
    flags, unsolved = c.rollout_health()
    out = dict(c.books(), flags=flags, unsolved=unsolved, **c.rollout_state())
    out["record"] = [c.rollout_get_lap(b) for b in range(B)]
    out["xPred"] = [c.read_buffer("xPred", b, (c.N + 1, 6)) for b in range(B)]
    out["laps"] = [_stored_laps(c, b) for b in range(B)]
    return out


def _same(a, b):
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return np.array_equal(np.asarray(a), np.asarray(b))


@functools.lru_cache(maxsize=None)
def _independent(mode, what, shaped):
    """12 closed-loop steps, the injection into controller K (none for what=None), 6 more steps"""
    c = _seeded(shaped)
    try:
        if mode == 2:
            c.rollout_sysid()
        for _ in range(12):
            _step(c, mode)
        before = c.rollout_health()
        if what is not None:
            _inject(c, K, what)
        for _ in range(6):
            _step(c, mode)
        return before, _result(c)
    finally:
        c.close()


@pytest.mark.parametrize("what", list(INJECT))
@pytest.mark.parametrize("mode,shaped", [(1, False), (0, False), (2, False), (1, True)])
def test_a_diverged_controller_leaves_the_others_bit_for_bit(mode, shaped, what):
    _need_gpu()
    _, clean = _independent(mode, None, shaped)
    (flags0, unsolved0), res = _independent(mode, what, shaped)
    for key, v in res.items():
        for b in range(B):
            if b != K:
                assert _same(v[b], clean[key][b]), (key, b)
    flags, unsolved = res["flags"][K], res["unsolved"][K]
    assert unsolved > unsolved0[K], (unsolved, unsolved0[K])
    if mode == 1:
        assert flags & (512 if what != "1e300 vx" else 512 | 128), flags
    if what == "inf s":
        assert flags & 128, flags


def _pooled(what, steps):
    """Two pool groups (even / odd controllers).  After every controller has driven one LMPC lap, the controller of group 0 with
    the fastest latest lap gets the injection (none for what=None), the batch takes `steps` steps and one exchange runs."""
    groups = np.arange(B) % 2
    c = _seeded(groups=groups)
    try:
        for n in range(1, 800):
            _step(c, 1)
            if n % 4 == 0 and c.books()["lap_n"].min() >= 1:
                break
        bk = c.books()
        assert bk["lap_n"].min() >= 1
        latest = np.array([bk["ss_time"][b, bk["prev_slot"][b]] for b in range(B)])
        k = int(np.argmin(np.where(groups == 0, latest, np.iinfo(np.int32).max)))
        if what is not None:
            _inject(c, k, what)
        for _ in range(steps):
            _step(c, 1)
        G, kbest, Tpad = 2, 3, c.Tmax
        rows = torch.zeros(G * kbest, Tpad, 9, dtype=torch.float64, device="cuda")
        meta = torch.zeros(G * kbest, 4, dtype=torch.int32, device="cuda")
        c.pool_export(kbest, Tpad, 0, rows, meta)
        c.pool_import(G * kbest, 2, Tpad, 0, rows, meta)
        c.sync()                                        # the exchange runs on the controller's stream
        exported = meta.cpu().numpy()
        res = _result(c)
        res["exported"] = exported
        res["k"] = k
        if steps > 1:                                   # the importers run on with what they took
            for _ in range(4):
                _step(c, 1)
            res["after"] = _result(c)
            M = c.M
            res["sel"] = [dict((name, c.read_buffer(name, b, shp)) for name, shp in
                               (("SS_sel", (6, M)), ("Qfun_sel", (M,)), ("Succ_SS", (6, M)), ("x0", (6,)), ("abc", (c.N, 54))))
                          for b in range(B)]
        return res
    finally:
        c.close()


@pytest.mark.parametrize("steps", [1, 5])
def test_a_diverged_controller_exports_no_non_finite_row(steps):
    """The one-step form takes exactly one step after the injection before the exchange: addPoint's refusal alone decides
    whether the exported lap carries the NaN row"""
    _need_gpu()
    clean = _pooled(None, steps)
    res = _pooled("nan vx", steps)
    k = res["k"]
    assert k == clean["k"]
    assert k in res["exported"][:3, 2], res["exported"]          # the diverged controller's lap is among group 0's exports
    for b in range(B):
        if b == k:
            continue
        for x, u, q in res["laps"][b]:
            assert np.isfinite(x).all() and np.isfinite(u).all() and np.isfinite(q).all(), b
    for b in range(1, B, 2):                                     # group 1 exchanged among itself as without the injection
        for key in ("x", "xglob", "done", "cl_len", "flags", "unsolved", "ss_time", "ss_lap", "it", "lap_n", "record", "xPred", "laps"):
            assert _same(res[key][b], clean[key][b]), (key, b)
    if steps > 1:
        assert res["after"]["flags"][k] & 512
        for b in range(B):
            if b == k:
                continue
            for name, v in res["sel"][b].items():
                assert np.isfinite(v).all(), (name, b)
            for x, u, q in res["after"]["laps"][b]:
                assert np.isfinite(x).all() and np.isfinite(u).all() and np.isfinite(q).all(), b
        for b in range(1, B, 2):
            for key in ("x", "flags", "unsolved", "ss_time", "record", "xPred", "laps"):
                assert _same(res["after"][key][b], clean["after"][key][b]), (key, b)
