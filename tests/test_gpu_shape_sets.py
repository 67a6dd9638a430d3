"""GPU tier: per-controller horizons and safe-set sizes (lmpc_set_shapes).

Every controller of a shaped batch equals, bit for bit on its valid rows, a handle created with its own (N, numSS_Points) and the
same parameters installed as a one-set table (the arithmetic of the parameter-set kernel): lmpc_step_host in modes 0 and 1 after a
device PID lap and seeding, and the device closed loop -- PID lap, seeding and three LMPC laps under lap budgets, in mode 1, and
steps in modes 0 and 2 -- for interleaved shapes on both axes, pooled with one group per shape, and crossed with parameter sets.
One shape equal to the handle's equals no table, nsets == 0 reverts, refusals change nothing, the caller-problem entry points are
refused while shaped, a snapshot resumes bit for bit, and a step launches one QP kernel per distinct shape present."""
import copy

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                # noqa: E402
from racinglmpc_b200 import _native as nat                        # noqa: E402
from racinglmpc_b200.controller import BatchedController          # noqa: E402
from racinglmpc_b200.reference_params import TrackParams          # noqa: E402

LMPC_E_INVALID, LMPC_E_STATE = -1, -4
X0 = np.array([0.5, 0, 0, 0, 0, 0.0])
TRACK = TrackParams.l_shaped()
# interleaved shapes on both axes, and the smallest grid pair that dominates them
SHAPES = [(6, 48), (14, 96), (12, 24), (10, 48), (14, 32), (12, 64)]
HANDLE = (14, 96)
B = 36
IDX = np.arange(B) % len(SHAPES)
KEYS = ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt", "flags", "unsolved")


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _controller(Bc, N, M, warm=False):
    numSS_it, _, _, _, Qts, par = rp.lmpc_params(N)
    return BatchedController(par, Bc, TRACK.seg_table, TRACK.TrackLength, trToUse=4, numSS_Points=M, numSS_it=numSS_it,
                             QterminalSlack=Qts, Tmax=1280, ss_cap=7, model_cap=5, warm_start=warm)


def _with(p, **kw):
    q = copy.copy(p)
    q.__dict__.update(kw)
    return q


def _one_set(c, par=None):
    """The reference's parameters (or `par`) as a one-set table: the parameter-set kernel's arithmetic"""
    c.set_param_sets([rp.lmpc_params(c.N)[5] if par is None else _with(par, N=c.N)], np.zeros(c.B, int))


def _seeded(c, streams, hook=None, Tcl=1024):
    """Tables (hook), the device PID lap on the given noise streams and the seeding; the state is back at the start line"""
    if hook is not None:
        hook(c)
    c.enable_rollout(Tcl=Tcl)
    c.set_noise_streams(streams)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))


def _laps(c, laps=3, mode=1, pooled=False):
    """LMPC laps under a lap budget (every controller ends where it would end alone); with `pooled`, one exchange at a fixed step
    (the same step for every batch, so a group exchanges the same laps whatever else is in the batch)"""
    c.set_lap_budget(laps)
    rows = torch.zeros(c.pool_groups * 3, 288, 9, dtype=torch.float64, device="cuda")
    meta = torch.zeros(c.pool_groups * 3, 4, dtype=torch.int32, device="cuda")
    for n in range(1, 300 * laps + 1):
        c.rollout_step(seed=1234, mode=mode)
        c.rollout_commit_laps_dev()
        if pooled and n == 320:
            c.pool_export(3, 288, 0, rows, meta)
            c.pool_import(c.pool_groups * 3, 2, 288, 0, rows, meta)
        if n % 8 == 0 and n > 320 and c.books()["lap_n"].min() >= laps:
            break
    return _result(c)


def _result(c):
    flags, unsolved = c.rollout_health()
    return dict(c.books(), flags=flags, unsolved=unsolved, **c.rollout_state())


def _per_shape(shapes, idx, body, par_of=None):
    """body(c) on one handle per shape, created with that (N, numSS_Points), holding the controllers of that shape on their noise
    streams; returns the results scattered back to the positions of the shaped batch"""
    out = {}
    for k, (N, M) in enumerate(shapes):
        members = np.nonzero(idx == k)[0]
        if members.size == 0:
            continue
        c = _controller(members.size, N, M)
        try:
            res = body(c, members, k)
        finally:
            c.close()
        for key, v in res.items():
            if key not in out:
                out[key] = [None] * idx.size
            for j, b in enumerate(members):
                out[key][b] = v[j]
    return out


def _same(shaped, own, what):
    for key in KEYS:
        for b in range(len(own[key])):
            if own[key][b] is None:
                continue
            assert np.array_equal(np.asarray(shaped[key][b]), np.asarray(own[key][b])), (what, key, b)


def _step_host(c, mode):
    Bc, N, M = c.B, c.N, max(c.M, 1)
    o = dict(xPred=np.zeros((Bc, N + 1, 6)), uPred=np.zeros((Bc, N, 2)), lambd=np.zeros((Bc, M)), zt=np.zeros((Bc, 6)),
             zt_u=np.zeros((Bc, 2)), SS_sel=np.zeros((Bc, 6, M)), status=np.zeros(Bc, np.int32), iters=np.zeros(Bc, np.int32),
             resid=np.zeros((Bc, 3)), flags=np.zeros(Bc, np.int32))
    x0 = np.ascontiguousarray(np.tile(X0, (Bc, 1)))
    nat.check(nat.lib().lmpc_step_host(c._h, mode, nat.ptr(x0), nat.ptr(o["xPred"]), nat.ptr(o["uPred"]), nat.ptr(o["lambd"]),
                                       nat.ptr(o["zt"]), nat.ptr(o["zt_u"]), nat.ptr(o["SS_sel"]), nat.ptr(o["status"]),
                                       nat.ptr(o["iters"]), nat.ptr(o["resid"]), nat.ptr(o["flags"])))
    return o


def _cut(o, b, Nb, Mb, mode):
    """Controller b's valid part of a step's outputs: N_b + 1 / N_b rows, the [6, M_b] block and M_b multipliers"""
    r = dict(xPred=o["xPred"][b, :Nb + 1], uPred=o["uPred"][b, :Nb], status=o["status"][b], iters=o["iters"][b], resid=o["resid"][b],
             flags=o["flags"][b])
    if mode == 1:
        r.update(lambd=o["lambd"][b, :Mb], zt=o["zt"][b], zt_u=o["zt_u"][b], SS_sel=o["SS_sel"][b].reshape(-1)[:6 * Mb].reshape(6, Mb))
    return r


@pytest.mark.parametrize("mode", [0, 1])
def test_step_host_equals_one_handle_per_shape(mode):
    _need_gpu()
    c = _controller(B, *HANDLE)
    try:
        _seeded(c, np.arange(B), hook=lambda c: c.set_shapes(SHAPES, IDX))
        for _ in range(3):                       # a few steps: the shifted state and the previous prediction come into play
            o = _step_host(c, mode)
        shaped = [_cut(o, b, *SHAPES[IDX[b]], mode) for b in range(B)]
    finally:
        c.close()

    def body(h, members, k):
        _seeded(h, members, hook=_one_set)
        for _ in range(3):
            oo = _step_host(h, mode)
        return {"r": [_cut(oo, j, h.N, h.M, mode) for j in range(h.B)]}
    own = _per_shape(SHAPES, IDX, body)["r"]
    for b in range(B):
        for key, v in own[b].items():
            assert np.array_equal(shaped[b][key], v), (mode, SHAPES[IDX[b]], b, key)


def test_closed_loop_equals_one_handle_per_shape():
    _need_gpu()
    c = _controller(B, *HANDLE)
    try:
        _seeded(c, np.arange(B), hook=lambda c: c.set_shapes(SHAPES, IDX))
        assert [c.shape_of(b) for b in range(B)] == [SHAPES[k] for k in IDX]
        res = _laps(c)
    finally:
        c.close()
    shaped = {k: list(v) for k, v in res.items()}
    assert (res["lap_n"] == 3).all()
    own = _per_shape(SHAPES, IDX, lambda h, m, k: (_seeded(h, m, hook=_one_set), _laps(h))[1])
    _same(shaped, own, "closed loop")
    # the horizons differ in what they learn: not every shape drove the same third lap
    assert len({int(res["lap_hist"][b, 2]) for b in range(B)}) > 1


@pytest.mark.parametrize("mode", [0, 2])
def test_mpc_modes_equal_one_handle_per_shape(mode):
    _need_gpu()

    def drive(h, streams, hook):
        _seeded(h, streams, hook=hook)
        if mode == 2:
            h.rollout_sysid()
        for _ in range(40):
            h.rollout_step(seed=99, mode=mode)
        return _result(h)
    c = _controller(B, *HANDLE)
    try:
        res = drive(c, np.arange(B), lambda c: c.set_shapes(SHAPES, IDX))
    finally:
        c.close()
    own = _per_shape(SHAPES, IDX, lambda h, m, k: drive(h, m, _one_set))
    _same({k: list(v) for k, v in res.items()}, own, "mode %d" % mode)


def test_pooled_with_one_group_per_shape_equals_one_handle_per_shape():
    _need_gpu()
    shapes = [(10, 48), (14, 96)]
    idx = np.arange(24) % 2
    c = _controller(24, *HANDLE)
    try:
        _seeded(c, np.arange(24), hook=lambda c: (c.set_shapes(shapes, idx), c.set_pool_groups(idx)))
        res = _laps(c, laps=2, pooled=True)
    finally:
        c.close()
    own = _per_shape(shapes, idx, lambda h, m, k: (_seeded(h, m, hook=_one_set), _laps(h, laps=2, pooled=True))[1])
    _same({k: list(v) for k, v in res.items()}, own, "pooled")


def test_crossed_shapes_and_parameter_sets_equal_one_handle_per_cell():
    _need_gpu()
    shapes = [(8, 48), (12, 64)]
    base = rp.lmpc_params(12)[5]
    pars = [base, _with(base, dR=2.0 * np.asarray(base.dR))]
    Bc = 16
    sidx, pidx = np.arange(Bc) % 2, (np.arange(Bc) // 2) % 2
    cell = 2 * sidx + pidx
    c = _controller(Bc, 14, 64)
    try:
        _seeded(c, np.arange(Bc), hook=lambda c: (c.set_shapes(shapes, sidx),
                                                   c.set_param_sets([_with(p, N=14) for p in pars], pidx)))
        res = _laps(c, laps=2)
    finally:
        c.close()
    cells = [shapes[s] for s in (0, 0, 1, 1)]
    own = _per_shape(cells, cell, lambda h, m, k: (_seeded(h, m, hook=lambda h: _one_set(h, pars[k % 2])), _laps(h, laps=2))[1])
    _same({k: list(v) for k, v in res.items()}, own, "crossed")


def _trivial_run(hook):
    c = _controller(16, 12, 48)
    try:
        _seeded(c, np.arange(16), hook=hook)
        return _laps(c, laps=2)
    finally:
        c.close()


def test_one_shape_equal_to_the_handle_equals_no_table_and_nsets_zero_reverts():
    _need_gpu()
    plain = _trivial_run(None)
    one = _trivial_run(lambda c: c.set_shapes([(12, 48)], np.zeros(16, int)))
    reverted = _trivial_run(lambda c: (c.set_shapes([(6, 48), (12, 48)], np.arange(16) % 2), c.set_shapes(None)))
    for key in KEYS:
        assert np.array_equal(plain[key], one[key]), key
        assert np.array_equal(plain[key], reverted[key]), key


def test_refusals_leave_the_handle_as_it_was():
    _need_gpu()
    L = nat.lib()
    c = _controller(B, *HANDLE)
    try:
        c.set_shapes(SHAPES, IDX)
        bad = (nat.ShapeParams * 1)(nat.ShapeParams(13, 48))
        zero = np.zeros(B, np.int32)
        for rows in ((nat.ShapeParams * 1)(nat.ShapeParams(13, 48)), (nat.ShapeParams * 1)(nat.ShapeParams(16, 48)),
                     (nat.ShapeParams * 1)(nat.ShapeParams(12, 0))):
            assert L.lmpc_set_shapes(c._h, rows, 1, nat.ptr(zero)) == LMPC_E_INVALID
        assert L.lmpc_set_shapes(c._h, bad, 1, nat.ptr(np.full(B, 1, np.int32))) == LMPC_E_INVALID
        # the caller-problem entry points have no per-controller shape
        x = np.zeros((B, 6)); u = np.zeros((B, 2)); abc = np.zeros((B, 14, 54))
        xp, up = np.zeros((B, 15, 6)), np.zeros((B, 14, 2))
        st, it, rs = np.zeros(B, np.int32), np.zeros(B, np.int32), np.zeros((B, 3))
        assert L.lmpc_solve_mpc_host(c._h, nat.ptr(x), nat.ptr(u), nat.ptr(abc), 14 * 54, 54, nat.ptr(xp), nat.ptr(up), None,
                                     nat.ptr(st), nat.ptr(it), nat.ptr(rs)) == LMPC_E_STATE
        xd, ud = torch.zeros(B, 6, dtype=torch.float64, device="cuda"), torch.zeros(B, 2, dtype=torch.float64, device="cuda")
        ad = torch.zeros(B, 14, 54, dtype=torch.float64, device="cuda")
        xpd, upd = torch.zeros(B, 15, 6, dtype=torch.float64, device="cuda"), torch.zeros(B, 14, 2, dtype=torch.float64, device="cuda")
        sd, idd = torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda")
        rd = torch.zeros(B, 3, dtype=torch.float64, device="cuda")
        assert L.lmpc_solve_mpc_dev(c._h, nat.ptr(xd), nat.ptr(ud), nat.ptr(ad), 14 * 54, 54, nat.ptr(xpd), nat.ptr(upd), None,
                                    nat.ptr(sd), nat.ptr(idd), nat.ptr(rd)) == LMPC_E_STATE
        # the shapes are still installed: one QP launch per distinct shape
        _seeded(c, np.arange(B))
        l0 = c.kernel_launches
        x0 = torch.tensor(np.tile(X0, (B, 1)), device="cuda")
        nat.check(L.lmpc_step_dev(c._h, 1, nat.ptr(x0)))
        c.sync()
        assert c.kernel_launches - l0 == 3 + len(SHAPES)
        # after a lap is stored
        assert L.lmpc_set_shapes(c._h, None, 0, None) == LMPC_E_STATE
        assert b"laps are stored" in L.lmpc_last_error()
    finally:
        c.close()
    w = _controller(4, 12, 48, warm=True)
    try:
        assert L.lmpc_set_shapes(w._h, (nat.ShapeParams * 1)(nat.ShapeParams(12, 48)), 1, nat.ptr(np.zeros(4, np.int32))) == LMPC_E_STATE
        assert b"warm_start" in L.lmpc_last_error()
    finally:
        w.close()


def test_kernel_launches_grow_by_one_qp_launch_per_distinct_shape():
    _need_gpu()
    for shapes, idx, n_lmpc, n_mpc in (([(6, 48), (12, 48), (14, 96)], np.arange(12) % 3, 3, 3),
                                       ([(12, 24), (12, 64), (14, 96)], np.arange(12) % 3, 3, 2),
                                       ([(6, 48), (12, 48), (14, 96)], np.zeros(12, int), 1, 1)):    # shapes without a controller
        c = _controller(12, *HANDLE)
        try:
            _seeded(c, np.arange(12), hook=lambda c: c.set_shapes(shapes, idx))
            x0 = torch.tensor(np.tile(X0, (12, 1)), device="cuda")
            for mode, n in ((1, n_lmpc), (0, n_mpc)):
                l0 = c.kernel_launches
                nat.check(nat.lib().lmpc_step_dev(c._h, mode, nat.ptr(x0)))
                c.sync()
                assert c.kernel_launches - l0 == (3 if mode == 1 else 2) + n, (shapes, mode)
        finally:
            c.close()


def test_lap_budgets_retire_shaped_controllers():
    _need_gpu()
    c = _controller(B, *HANDLE)
    try:
        _seeded(c, np.arange(B), hook=lambda c: c.set_shapes(SHAPES, IDX))
        res = _laps(c, laps=1)
        assert (res["lap_n"] == 1).all()
        before = c.rollout_state()["x"].copy()
        for _ in range(16):
            c.rollout_step(seed=1234)
            c.rollout_commit_laps_dev()
        assert np.array_equal(c.rollout_state()["x"], before)
    finally:
        c.close()


def test_snapshot_restores_a_shaped_controller_bit_for_bit():
    _need_gpu()
    shapes, idx = [(8, 48), (14, 96)], np.arange(8) % 2

    def run(split):
        c = _controller(8, *HANDLE)
        try:
            _seeded(c, np.arange(8), hook=lambda c: c.set_shapes(shapes, idx))
            c.set_lap_budget(2)
            for n in range(1, 600):
                c.rollout_step(seed=1234)
                c.rollout_commit_laps_dev()
                if split and n == 150:
                    rec = c.snapshot()
                    clock = c.rollout_clock
                    d = _controller(8, *HANDLE)
                    d.set_shapes(shapes, idx)
                    d.enable_rollout(Tcl=1024)
                    d.set_noise_streams(np.arange(8))
                    d.restore(rec)
                    d.rollout_clock = clock
                    d.set_lap_budget(2)
                    c.close()
                    c = d
                if n % 8 == 0 and c.books()["lap_n"].min() >= 2:
                    break
            return _result(c)
        finally:
            c.close()
    a, b = run(False), run(True)
    for key in KEYS:
        assert np.array_equal(a[key], b[key]), key
