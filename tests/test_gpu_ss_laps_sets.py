"""GPU tier: per-controller safe-set lap counts (lmpc_set_ss_laps).

Every controller of a batch with interleaved numSS_it 1..4 equals, bit for bit, a handle created with its own numSS_it and the
same ss_cap and seeding: the safe-set selection and the QP of lmpc_step_host in mode 1, three LMPC laps of the device closed loop
under lap budgets (books, end states, health), the host-slot hand-over with host books, the pooled exchange with one group per
value, and lap counts crossed with shapes.  One value equal to the handle's equals no table, nsets == 0 reverts, refusals change
nothing, and a snapshot restored into a controller of the same value resumes bit for bit."""
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
VALUES = [1, 2, 3, 4]
B = 16
IDX = np.arange(B) % len(VALUES)
NIT = 4                                                            # the handle's numSS_it
KEYS = ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt", "prev_slot",
        "used", "flags", "unsolved")


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _controller(Bc, nit=NIT, N=12, M=48):
    _, _, _, _, Qts, par = rp.lmpc_params(N)
    return BatchedController(par, Bc, TRACK.seg_table, TRACK.TrackLength, trToUse=4, numSS_Points=M, numSS_it=nit,
                             QterminalSlack=Qts, Tmax=1280, ss_cap=7, model_cap=5)


def _laps_table(values=VALUES, idx=IDX):
    return lambda c: c.set_ss_laps(values, idx)


def _seeded(c, streams, hook=None, Tcl=1024):
    """Tables (hook), the device PID lap on the given noise streams and the device seeding; the state is back at the start line"""
    if hook is not None:
        hook(c)
    c.enable_rollout(Tcl=Tcl)
    c.set_noise_streams(streams)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))


def _laps(c, laps=3, pooled=False):
    """LMPC laps under a lap budget; with `pooled`, one exchange at a fixed step (the same for every batch)"""
    c.set_lap_budget(laps)
    rows = torch.zeros(c.pool_groups * 3, 288, 9, dtype=torch.float64, device="cuda")
    meta = torch.zeros(c.pool_groups * 3, 4, dtype=torch.int32, device="cuda")
    for n in range(1, 300 * laps + 1):
        c.rollout_step(seed=1234)
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


def _per_value(body, values=VALUES, idx=IDX, **kw):
    """body(h, members) on one handle per value, created with that numSS_it, holding the controllers of that value on their
    noise streams; returns the results scattered back to the positions of the batch"""
    out = {}
    for k, v in enumerate(values):
        members = np.nonzero(idx == k)[0]
        if members.size == 0:
            continue
        h = _controller(members.size, nit=v, **kw)
        try:
            res = body(h, members)
        finally:
            h.close()
        for key, val in res.items():
            out.setdefault(key, [None] * idx.size)
            for j, b in enumerate(members):
                out[key][b] = val[j]
    return out


def _same(batch, own, what, values=VALUES, idx=IDX):
    """Controller by controller: every key of KEYS, and the controller's entries of sel / is_prev (the tail repeats the last
    selected slot with is_prev 0)"""
    for key in KEYS:
        for b in range(idx.size):
            assert np.array_equal(np.asarray(batch[key][b]), np.asarray(own[key][b])), (what, key, b)
    for b in range(idx.size):
        v = values[idx[b]]
        assert np.array_equal(batch["sel"][b][:v], own["sel"][b][:v]), (what, "sel", b)
        assert np.array_equal(batch["is_prev"][b][:v], own["is_prev"][b][:v]), (what, "is_prev", b)
        assert (batch["sel"][b][v:] == batch["sel"][b][v - 1]).all() and (batch["is_prev"][b][v:] == 0).all(), (what, "tail", b)


def _step_host(c):
    Bc, N, M = c.B, c.N, c.M
    o = dict(xPred=np.zeros((Bc, N + 1, 6)), uPred=np.zeros((Bc, N, 2)), lambd=np.zeros((Bc, M)), zt=np.zeros((Bc, 6)),
             zt_u=np.zeros((Bc, 2)), SS_sel=np.zeros((Bc, 6, M)), status=np.zeros(Bc, np.int32), iters=np.zeros(Bc, np.int32),
             resid=np.zeros((Bc, 3)), flags=np.zeros(Bc, np.int32))
    x0 = np.ascontiguousarray(np.tile(X0, (Bc, 1)))
    nat.check(nat.lib().lmpc_step_host(c._h, 1, nat.ptr(x0), nat.ptr(o["xPred"]), nat.ptr(o["uPred"]), nat.ptr(o["lambd"]),
                                       nat.ptr(o["zt"]), nat.ptr(o["zt_u"]), nat.ptr(o["SS_sel"]), nat.ptr(o["status"]),
                                       nat.ptr(o["iters"]), nat.ptr(o["resid"]), nat.ptr(o["flags"])))
    return o


def _select_then_steps(c):
    """K2 alone (lmpc_select_host), then three host steps (K1, K2, QP, shift), per controller"""
    x0 = np.tile(X0, (c.B, 1))
    sel = c.select(x0)
    outs = [_step_host(c) for _ in range(3)]
    r = {k: [sel[k][b] for b in range(c.B)] for k in ("SS_sel", "Qfun_sel", "Succ_SS", "Succ_uSS", "min_index", "flags")}
    for i, o in enumerate(outs):
        for k, v in o.items():
            r["step%d_%s" % (i, k)] = [v[b] for b in range(c.B)]
    return r


def test_select_and_step_host_equal_one_handle_per_value():
    _need_gpu()
    c = _controller(B)
    try:
        _seeded(c, np.arange(B), hook=_laps_table())
        got = _select_then_steps(c)
    finally:
        c.close()
    own = _per_value(lambda h, m: (_seeded(h, m), _select_then_steps(h))[1])
    for key in got:
        for b in range(B):
            v = VALUES[IDX[b]]
            mine, ref = np.asarray(got[key][b]), np.asarray(own[key][b])
            if key == "min_index":                 # only the controller's entries: warps c >= numSS_it_b select nothing
                mine = mine[:v]
            assert np.array_equal(mine, ref), (key, b, v)
    # the lap counts change what is selected: 48 points from one lap or 12 from each of four
    assert not np.array_equal(got["SS_sel"][0], got["SS_sel"][3])


def test_closed_loop_equals_one_handle_per_value():
    _need_gpu()
    c = _controller(B)
    try:
        _seeded(c, np.arange(B), hook=_laps_table())
        assert [c.ss_laps_of(b) for b in range(B)] == [VALUES[k] for k in IDX]
        res = _laps(c)
    finally:
        c.close()
    assert (res["lap_n"] == 3).all()
    own = _per_value(lambda h, m: (_seeded(h, m), _laps(h))[1])
    _same({k: list(v) for k, v in res.items()}, own, "closed loop")
    assert len({int(res["lap_hist"][b, 2]) for b in range(B)}) > 1


def _host_books_laps(c, streams, hook=None, laps=2):
    """The host-slot hand-over: device PID lap, seeding with host books, 300 * laps closed-loop steps with host-chosen slots
    (rollout_finish_laps)"""
    if hook is not None:
        hook(c)
    c.enable_rollout(Tcl=1024)
    c.set_noise_streams(streams)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    _, n = c.rollout_done()
    c.rollout_seed_from_record(n, copies=4)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))
    for _ in range(300 * laps):                  # a fixed number of steps: every batch stops at the same step
        c.rollout_step(seed=1234)
        done, n = c.rollout_done()
        if done.any():
            c.rollout_finish_laps(done, n)
    st = c.rollout_state()
    return dict(x=st["x"], cl_len=st["cl_len"], LapTime=[list(t) for t in c.LapTime], it=list(c.it),
                slots=[sorted(c.ss_book[b].slot_of.items()) for b in range(c.B)])


def test_host_slot_hand_over_equals_one_handle_per_value():
    _need_gpu()
    c = _controller(B)
    try:
        got = _host_books_laps(c, np.arange(B), hook=_laps_table())
    finally:
        c.close()
    own = _per_value(lambda h, m: _host_books_laps(h, m))
    for key in got:
        for b in range(B):
            assert np.array_equal(np.asarray(got[key][b], dtype=object), np.asarray(own[key][b], dtype=object)), (key, b)
    assert min(len(t) for t in got["LapTime"]) >= 6         # four seeded copies and at least two own laps


def test_pooled_with_one_group_per_value_equals_one_handle_per_value():
    _need_gpu()
    c = _controller(B)
    try:
        _seeded(c, np.arange(B), hook=lambda c: (c.set_ss_laps(VALUES, IDX), c.set_pool_groups(IDX, len(VALUES))))
        res = _laps(c, laps=2, pooled=True)
    finally:
        c.close()
    own = _per_value(lambda h, m: (_seeded(h, m), _laps(h, laps=2, pooled=True))[1])
    _same({k: list(v) for k, v in res.items()}, own, "pooled")


def test_pooled_mixed_group_takes_imports_against_each_importers_value():
    """One pool for all values: a run completes, and every controller's books stay within its own value's rules (its selection
    holds its numSS_it fastest stored laps)."""
    _need_gpu()
    c = _controller(B)
    try:
        _seeded(c, np.arange(B), hook=_laps_table())
        res = _laps(c, laps=2, pooled=True)
    finally:
        c.close()
    assert (res["lap_n"] == 2).all() and (res["flags"] & 64 == 0).all()
    for b in range(B):
        v = VALUES[IDX[b]]
        stored = sorted((int(t), int(l), s) for s, (t, l) in enumerate(zip(res["ss_time"][b], res["ss_lap"][b])) if l >= 0)
        assert list(res["sel"][b][:v]) == [s for (_, _, s) in stored[:v]], b


def test_lap_counts_crossed_with_shapes_equal_one_handle_per_pair():
    _need_gpu()
    cells = [(v, m) for v in VALUES for m in (24, 48)]
    idx = np.arange(B) % len(cells)
    lv = np.array([cells[k][0] for k in idx])
    shapes, sidx = [(12, 24), (12, 48)], np.array([0 if cells[k][1] == 24 else 1 for k in idx])
    c = _controller(B)
    try:
        _seeded(c, np.arange(B), hook=lambda c: (c.set_shapes(shapes, sidx), c.set_ss_laps(VALUES, lv - 1)))
        res = _laps(c)
    finally:
        c.close()
    batch = {k: list(v) for k, v in res.items()}
    for k, (v, m) in enumerate(cells):
        members = np.nonzero(idx == k)[0]
        h = _controller(members.size, nit=v, M=m)
        try:
            h.set_param_sets([rp.lmpc_params(12)[5]], np.zeros(h.B, int))   # the shaped QP kernel's arithmetic
            _seeded(h, members)
            own = _laps(h)
        finally:
            h.close()
        for key in KEYS:
            for j, b in enumerate(members):
                assert np.array_equal(np.asarray(batch[key][b]), np.asarray(own[key][j])), ((v, m), key, b)


def test_the_handles_value_as_a_table_equals_no_table_and_reverting_restores_it():
    _need_gpu()
    runs = []
    for hook in (None, lambda c: c.set_ss_laps([NIT], np.zeros(B, int)),
                 lambda c: (c.set_ss_laps(VALUES, IDX), c.set_ss_laps(None))):
        c = _controller(B)
        try:
            _seeded(c, np.arange(B), hook=hook)
            runs.append(_laps(c))
        finally:
            c.close()
    for r in runs[1:]:
        for key in KEYS + ("sel", "is_prev"):
            assert np.array_equal(runs[0][key], r[key]), key


def test_refusals_change_nothing():
    _need_gpu()
    L = nat.lib()
    c = _controller(B)
    try:
        def call(values, idx):
            rows = (nat.SsLapsParams * len(values))(*[nat.SsLapsParams(v) for v in values])
            ix = np.ascontiguousarray(idx, np.int32)
            return L.lmpc_set_ss_laps(c._h, rows, len(values), nat.ptr(ix))
        c.set_ss_laps(VALUES, IDX)
        assert call([0], np.zeros(B)) == LMPC_E_INVALID
        assert call([NIT + 1], np.zeros(B)) == LMPC_E_INVALID
        assert call([1, 2], np.full(B, 2)) == LMPC_E_INVALID
        assert L.lmpc_set_ss_laps(c._h, None, 1, None) == LMPC_E_INVALID
        # a shape whose points do not split into the controller's laps, in both orders: 32 points into 3 laps
        sh = (nat.ShapeParams * 1)(nat.ShapeParams(12, 32))
        assert L.lmpc_set_shapes(c._h, sh, 1, nat.ptr(np.zeros(B, np.int32))) == LMPC_E_INVALID
        assert [c.ss_laps_of(b) for b in range(B)] == [VALUES[k] for k in IDX]
        _seeded(c, np.arange(B))
        res = _laps(c)
        # a lap is stored: the table is fixed from now on
        assert call([1], np.zeros(B)) == LMPC_E_STATE
        assert L.lmpc_set_ss_laps(c._h, None, 0, None) == LMPC_E_STATE
    finally:
        c.close()
    own = _per_value(lambda h, m: (_seeded(h, m), _laps(h))[1])
    _same({k: list(v) for k, v in res.items()}, own, "after refusals")
    d = _controller(4)
    try:
        d.set_shapes([(12, 32)], np.zeros(4, int))
        rows = (nat.SsLapsParams * 1)(nat.SsLapsParams(3))
        assert L.lmpc_set_ss_laps(d._h, rows, 1, nat.ptr(np.zeros(4, np.int32))) == LMPC_E_INVALID
    finally:
        d.close()
    m = BatchedController(rp.mpc_params(12), 4, TRACK.seg_table, TRACK.TrackLength, trToUse=4)
    try:
        rows = (nat.SsLapsParams * 1)(nat.SsLapsParams(1))
        assert L.lmpc_set_ss_laps(m._h, rows, 1, nat.ptr(np.zeros(4, np.int32))) == LMPC_E_INVALID
    finally:
        m.close()


def test_snapshot_restored_into_a_controller_of_the_same_value_resumes_bit_for_bit():
    _need_gpu()

    def run(split):
        c = _controller(8)
        idx = np.arange(8) % 4
        try:
            _seeded(c, np.arange(8), hook=_laps_table(idx=idx))
            c.set_lap_budget(2)
            for n in range(1, 600):
                c.rollout_step(seed=1234)
                c.rollout_commit_laps_dev()
                if split and n == 150:
                    rec = c.snapshot()
                    clock = c.rollout_clock
                    d = _controller(8)
                    d.set_ss_laps(VALUES, idx)
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
    for key in KEYS + ("sel", "is_prev"):
        assert np.array_equal(a[key], b[key]), key
