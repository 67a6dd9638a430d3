"""GPU tier: lane-safe safe sets (lmpc_set_lane_rules).

An all-mode-0 table and a mode 1 table whose tolerance no finite row exceeds equal the closed loop without the call bit for bit
(independent and pooled: books, states, health, step results, reports, snapshot records).  On lanes of half-width 0.4 / 0.25 /
0.1 the device books follow tests/support/lapbook_lane.LaneBooks event by event (own laps and imports, with and without lap
windows); an own lap's verdict equals its report's viol_max > lane_tol without measurement noise, and the judgement of the record
rows the controller saw under measurement noise; imports are judged by the importer and the export works on raw lap times; rows
interleaved in one batch equal one handle per row; a snapshot resumes bit for bit and a lane-unsafe key is refused by a
controller whose rule is off; refused calls change nothing."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                # noqa: E402
from racinglmpc_b200 import _native as nat                        # noqa: E402
from racinglmpc_b200.controller import BatchedController          # noqa: E402
from racinglmpc_b200.reference_params import TrackParams, LaneRuleParams as R, LapWindowParams as W   # noqa: E402
from lapbook_lane import LaneBooks, lane_unsafe, lane_key, LANE_UNSAFE_KEY   # noqa: E402
import lapbook_exact as lx                                        # noqa: E402
import test_gpu_lap_books_exact as gx                             # noqa: E402

LMPC_E_INVALID, LMPC_E_STATE = -1, -4
X0 = np.array([0.5, 0, 0, 0, 0, 0.0])
TRACK = TrackParams.l_shaped()
B = 12
WIDTHS = (0.4, 0.25, 0.1, 0.02)        # the last one is crossed within a few LMPC laps
KEYS = ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt", "sel",
        "is_prev", "prev_slot", "used", "flags", "unsolved")


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _par(width, N=12):
    p = rp.lmpc_params(N)[5]
    return SimpleNamespace(**{**vars(p), "bx": np.array([width, width])})


def _controller(Bc, widths=None):
    _, _, _, _, Qts, par = rp.lmpc_params(12)
    c = BatchedController(par, Bc, TRACK.seg_table, TRACK.TrackLength, trToUse=4, numSS_Points=48, numSS_it=4,
                          QterminalSlack=Qts, Tmax=1280, ss_cap=7, model_cap=5)
    if widths is not None:
        c.set_param_sets([_par(w) for w in WIDTHS], np.asarray(widths))
    return c


def _seeded(c, streams, hook=None, reports=0, meas=None):
    if hook is not None:
        hook(c)
    c.enable_rollout(Tcl=1024)
    if reports:
        c.enable_lap_reports(reports)
    if meas is not None:
        c.set_measurement_noise([rp.MeasurementParams(sigma=(meas,) * 6, clip=(5 * meas,) * 6)], np.zeros(c.B, int))
    c.set_noise_streams(streams)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))


def _laps(c, laps=3, pooled=False, records=False, share=2):
    c.set_lap_budget(laps)
    rows = torch.zeros(c.pool_groups * 3, 288, 9, dtype=torch.float64, device="cuda")
    meta = torch.zeros(c.pool_groups * 3, 4, dtype=torch.int32, device="cuda")
    for n in range(1, 400 * laps + 1):
        c.rollout_step(seed=1234)
        c.rollout_commit_laps_dev()
        if pooled and n in (320, 520):
            c.pool_export(3, 288, 0, rows, meta)
            c.pool_import(c.pool_groups * 3, share, 288, 0, rows, meta)
        if n % 8 == 0 and n > 520 and c.books()["lap_n"].min() >= laps:
            break
    flags, unsolved = c.rollout_health()
    out = dict(c.books(), flags=flags, unsolved=unsolved, **c.rollout_state())
    out.update({"step_" + k: v for k, v in c.step_results().items()})
    if getattr(c, "lap_report_cap", 0):
        out.update({"rep_" + k: v for k, v in c.lap_reports().items()})
    if records:
        out["records"] = c.snapshot().cpu().numpy()
    return out


def _run(hook, pooled=False, Bc=B, widths=None, **kw):
    c = _controller(Bc, widths)
    try:
        _seeded(c, np.arange(Bc), hook=hook, reports=4, **kw)
        return _laps(c, pooled=pooled, records=True)
    finally:
        c.close()


@pytest.mark.parametrize("pooled", [False, True], ids=["independent", "pooled"])
def test_reference_rule_and_an_unreachable_tolerance_equal_no_table(pooled):
    _need_gpu()
    ref = _run(None, pooled)
    assert (ref["lap_n"] == 3).all()
    for hook in (lambda c: c.set_lane_rules([R.reference()], np.zeros(B, int)),
                 lambda c: c.set_lane_rules([R(1, 1e300), R(0, 0.0)], np.arange(B) % 2),
                 lambda c: (c.set_lane_rules([R(1, 0.0)], np.zeros(B, int)), c.set_lane_rules(None))):
        got = _run(hook, pooled)
        for key in ref:
            assert np.array_equal(ref[key], got[key]), key


# (numSS_it, ss_cap, trToUse, model_cap) of test_gpu_lap_books_exact.py, with and without lap windows.  gx's rows are standard
# normal, so the lane rows' margin is |ey| - w: tolerances around the maximum of |ey| over a lap give both verdicts.
LANE_ROWS = [R(0, 0.0), R(1, 1.9), R(1, 2.4), R(1, 0.0)]
EXACT = [((4, 6, 4, 5), None), ((4, 6, 4, 5), [(0, 0), (4, 4), (6, 5), (5, 0)]), ((2, 4, 8, 8), None),
         ((1, 2, 1, 1), [(1, 1), (2, 1), (0, 1)])]


@pytest.mark.parametrize("cfg, wins", EXACT, ids=["nit%d_ss%d_tr%d_md%d" % e[0] + ("_win" if e[1] else "") for e in EXACT])
def test_device_books_follow_the_lane_lists_event_by_event(cfg, wins):
    _need_gpu()
    rng = np.random.default_rng(3000 + EXACT.index((cfg, wins)))
    c = gx._controller(cfg, gx.B)
    widx = np.arange(gx.B) % len(WIDTHS)
    lidx = (np.arange(gx.B) // 2) % len(LANE_ROWS)
    pars = [_par(w) for w in WIDTHS]
    c.set_param_sets(pars, widx)
    c.set_lane_rules(LANE_ROWS, lidx)
    win = [(0, 0)] * gx.B
    if wins:
        win = [wins[b % len(wins)] for b in range(gx.B)]
        c.set_lap_windows([W(*w) for w in wins], np.arange(gx.B) % len(wins))
    grp = np.arange(gx.B) % gx.G
    c.set_pool_groups(grp, gx.G)
    models = [LaneBooks(*cfg, Tmax=gx.TMAX, TrackLength=TRACK.TrackLength, ss_window=win[b][0], md_window=win[b][1],
                        lane_mode=LANE_ROWS[lidx[b]].mode, lane_tol=LANE_ROWS[lidx[b]].lane_tol, Fx=pars[widx[b]].Fx,
                        bx=pars[widx[b]].bx) for b in range(gx.B)]
    lengths = [gx._lap_lengths(rng, b % 6, gx.ROUNDS + 1) for b in range(gx.B)]
    lap = [0] * gx.B
    try:
        for r in range(gx.ROUNDS):
            if r % gx.XEVERY == 0:
                fresh = gx._import_round(c, models, rng, grp)
                gx._check_books(c, models, fresh)
            fresh = gx._own_round(c, models, rng, lengths, lap)
            bk = gx._check_books(c, models, fresh)
            if r % 5 == 4:
                gx._check_pools(c, models, bk, cfg)
    finally:
        c.close()
    verdicts = [v for m in models if m.lane_mode == 1 for v in m.unsafe_hist]
    assert any(verdicts) and not all(verdicts)                        # both verdicts occurred
    keys = [t for m in models if not m.dead for t in m.times]
    assert any(t >= LANE_UNSAFE_KEY for t in keys)


def _report_bits(meas):
    widths = np.arange(B) % len(WIDTHS)
    c = _controller(B, widths=widths)
    tol = [0.0, 0.02, 0.05]
    lidx = np.arange(B) % 3
    try:
        _seeded(c, np.arange(B), hook=lambda c: c.set_lane_rules([R(1, t) for t in tol], lidx), reports=8, meas=meas)
        c.set_lap_budget(4)
        seen = [[] for _ in range(B)]                                  # own verdict from the record rows, per lap
        for n in range(1, 2000):
            c.rollout_step(seed=1234)
            done, cl = c.rollout_done()
            for b in np.nonzero(done)[0]:
                x, _ = c.rollout_get_lap(int(b))
                seen[b].append(lane_unsafe(x, rp.lmpc_params(12)[5].Fx, [WIDTHS[widths[b]]] * 2, tol[lidx[b]]))
            c.rollout_commit_laps_dev()
            if n % 8 == 0 and c.books()["lap_n"].min() >= 4:
                break
        return c.lap_reports(), seen, [tol[k] for k in lidx]
    finally:
        c.close()


def test_own_verdict_is_the_reports_violation_without_measurement_noise():
    _need_gpu()
    rep, seen, tol = _report_bits(None)
    bits = 0
    for b in range(B):
        n = min(int(rep["n"][b]), 8)
        assert n >= 4
        for j in range(n):
            bit = bool(rep["flags"][b, j] & nat.REPORT_LANE_UNSAFE)
            assert bit == bool(rep["viol_max"][b, j] > tol[b]), (b, j)
            assert bit == seen[b][j], (b, j)
            bits += bit
    assert 0 < bits < B * 4                                            # the narrowest lane is crossed, the wide ones kept


def test_own_verdict_judges_the_measured_record_under_measurement_noise():
    _need_gpu()
    rep, seen, _ = _report_bits(0.01)
    for b in range(B):
        n = min(int(rep["n"][b]), 8)
        got = [bool(f & nat.REPORT_LANE_UNSAFE) for f in rep["flags"][b, :n]]
        assert got == seen[b][:n], b


def test_imports_are_judged_by_the_importer_and_the_export_ships_raw_lap_times():
    _need_gpu()
    widths = 2 + np.arange(B) % 2                                       # two lane widths (0.1, 0.02) in one pool group
    rules = [R(0, 0.0), R(1, 0.0), R(1, 0.03)]
    lidx = np.arange(B) % 3
    pars = [_par(w) for w in WIDTHS]
    c = _controller(B, widths)
    try:
        _seeded(c, np.arange(B), hook=lambda c: c.set_lane_rules(rules, lidx))
        for _ in range(330):
            c.rollout_step(seed=1234)
            c.rollout_commit_laps_dev()
        kbest, tpad = 4, 288
        rows = torch.zeros(kbest, tpad, 9, dtype=torch.float64, device="cuda")
        meta = torch.zeros(kbest, 4, dtype=torch.int32, device="cuda")
        bk = c.books()
        recs = c.snapshot().cpu().numpy()
        sect = nat.decode_snapshot_header(recs[0])["sections"]
        off, nb = sect["ss_len"]
        ss_len = recs[:, off:off + nb].view(np.int32)
        cands = []
        for b in range(B):
            sl = int(bk["prev_slot"][b])
            if sl >= 0:
                t, _ = nat.split_lane_key(int(bk["ss_time"][b][sl]))
                cands.append((t, b, int(ss_len[b, sl])))
        assert any(t >= LANE_UNSAFE_KEY for t in bk["ss_time"][bk["ss_lap"] >= 0])
        c.pool_export(kbest, tpad, 0, rows, meta)
        m, R_ = meta.cpu().numpy(), rows.cpu().numpy()
        assert list(m[:, 2]) == lx.pool_local_best(cands, kbest, tpad, 0)
        assert (m[:, 1] < LANE_UNSAFE_KEY).all()
        before = c.books()
        c.pool_import(kbest, 1, tpad, 0, rows, meta)
        after = c.books()
        order = lx.pool_rank(m, 1)[0]
        judged = 0
        for b in range(B):
            pick = lx.pool_pick(order, m, b, 1)
            it0 = int(before["it"][b])
            slots = [s for s in range(7) if after["ss_lap"][b][s] == it0 - 1]
            if not pick or int(after["it"][b]) == it0:
                continue                                                # nothing filed
            i = pick[0]
            lt, ln = int(m[i, 1]), int(m[i, 0])
            want = rules[lidx[b]].mode == 1 and lane_unsafe(R_[i, :min(lt, ln, tpad)], pars[widths[b]].Fx, pars[widths[b]].bx,
                                                               rules[lidx[b]].lane_tol)
            assert [int(after["ss_time"][b][s]) for s in slots] == [lane_key(lt, want)], b
            judged += 1
        assert judged > 0
    finally:
        c.close()


ROWS = [R(0, 0.0), R(1, 0.0), R(1, 0.05)]


def test_interleaved_rows_equal_one_handle_per_row():
    _need_gpu()
    idx = np.arange(B) % len(ROWS)
    widths = (np.arange(B) // 3) % len(WIDTHS)
    c = _controller(B, widths)
    try:
        _seeded(c, np.arange(B), hook=lambda c: c.set_lane_rules(ROWS, idx))
        assert [c.lane_rules_of(b) for b in range(B)] == [(ROWS[k].mode, ROWS[k].lane_tol) for k in idx]
        res = _laps(c)
    finally:
        c.close()
    for k, row in enumerate(ROWS):
        members = np.nonzero(idx == k)[0]
        h = _controller(members.size, widths[members])
        try:
            _seeded(h, members, hook=lambda h: h.set_lane_rules([row], np.zeros(h.B, int)))
            own = _laps(h)
        finally:
            h.close()
        for key in KEYS:
            for j, b in enumerate(members):
                assert np.array_equal(res[key][b], own[key][j]), (key, b)
    assert (res["ss_time"][res["ss_lap"] >= 0] >= LANE_UNSAFE_KEY).any()


def test_snapshot_resumes_bit_for_bit_and_a_lane_key_needs_the_rule():
    _need_gpu()
    idx = np.arange(8) % len(ROWS)
    widths = np.arange(8) % len(WIDTHS)
    hook = lambda c: c.set_lane_rules(ROWS, idx)                       # noqa: E731
    saved = {}

    def run(split):
        c = _controller(8, widths)
        try:
            _seeded(c, np.arange(8), hook=hook)
            c.set_lap_budget(5)
            for n in range(1, 3000):
                c.rollout_step(seed=1234)
                c.rollout_commit_laps_dev()
                if split and "rec" not in saved and n % 8 == 0 and c.books()["lap_n"].min() >= 2:
                    rec, clock = c.snapshot(), c.rollout_clock
                    saved["rec"] = rec.clone()
                    d = _controller(8, widths)
                    hook(d)
                    d.enable_rollout(Tcl=1024)
                    d.set_noise_streams(np.arange(8))
                    d.restore(rec)
                    d.rollout_clock = clock
                    d.set_lap_budget(5)
                    c.close()
                    c = d
                if n % 8 == 0 and c.books()["lap_n"].min() >= 5:
                    break
            flags, unsolved = c.rollout_health()
            return dict(c.books(), flags=flags, unsolved=unsolved, **c.rollout_state())
        finally:
            c.close()
    a, b = run(False), run(True)
    for key in KEYS:
        assert np.array_equal(a[key], b[key]), key
    # a record holding a lane-unsafe key, restored into a controller whose rule is off
    rec = saved["rec"]
    sect = nat.decode_snapshot_header(rec[0].cpu().numpy())["sections"]
    off, nb = sect["ss_time"]
    keys = rec[:, off:off + nb].cpu().numpy().view(np.int32)
    off2, nb2 = sect["ss_lap"]
    laps = rec[:, off2:off2 + nb2].cpu().numpy().view(np.int32)
    r = int(np.nonzero(((keys >= LANE_UNSAFE_KEY) & (laps >= 0)).any(axis=1))[0][0])
    d = _controller(8, widths)
    try:
        d.set_lane_rules([R(0, 0.0)], np.zeros(8, int))
        d.enable_rollout(Tcl=1024)
        d.enable_device_books()
        before = d.snapshot().cpu().numpy()
        with pytest.raises(nat.NativeError, match="lane key"):
            d.restore(rec, [3], [r])
        assert np.array_equal(before, d.snapshot().cpu().numpy())
    finally:
        d.close()


def test_refusals_change_nothing():
    _need_gpu()
    L = nat.lib()

    def call(c, rules, idx):
        rows = (nat.LaneRuleParams * len(rules))(*[nat.LaneRuleParams(m, 0, t) for m, t in rules])
        return L.lmpc_set_lane_rules(c._h, rows, len(rules), nat.ptr(np.ascontiguousarray(idx, np.int32)))
    c = _controller(B)
    try:
        zero = np.zeros(B)
        for bad in ([(2, 0.0)], [(-1, 0.0)], [(1, -1e-9)], [(1, float("nan"))], [(0, float("inf"))]):
            assert call(c, bad, zero) == LMPC_E_INVALID, bad
        assert call(c, [(1, 0.0)], np.full(B, 1)) == LMPC_E_INVALID   # bad index
        assert L.lmpc_set_lane_rules(c._h, None, 1, None) == LMPC_E_INVALID
        assert call(c, [(1, 0.0)], zero) == 0
        c.set_lane_rules([R(1, 0.0)], np.zeros(B, int))
        # host-slot paths under a mode 1 row
        c.enable_rollout(Tcl=1024)
        fin = np.zeros(B, np.int32)
        sl = -np.ones(B, np.int32)
        assert L.lmpc_rollout_commit_laps(c._h, nat.ptr(fin), nat.ptr(sl), nat.ptr(sl)) == LMPC_E_STATE
        assert L.lmpc_rollout_seed_from_record(c._h, 4, 0, 0) == LMPC_E_STATE
        with pytest.raises(ValueError):
            c.rollout_finish_laps(np.ones(B, int), np.full(B, 10))
        # lmpc_books_set: a lane-unsafe key for a controller whose rule is off
        c.set_lane_rules([R(0, 0.0), R(1, 0.0)], np.arange(B) % 2)
        bk = c.books()
        st, sl_, it = bk["ss_time"].copy(), bk["ss_lap"].copy(), bk["it"].copy()
        st[:, 0], sl_[:, 0], it[:] = LANE_UNSAFE_KEY + 5, 0, 1
        args = [nat.ptr(np.ascontiguousarray(a, np.int32)) for a in (st, sl_, it, bk["md_time"], bk["md_seq"], bk["md_cnt"])]
        assert L.lmpc_books_set(c._h, *args) == LMPC_E_INVALID
        assert np.array_equal(c.books()["ss_lap"], bk["ss_lap"])
        st[0::2, 0] = 5                                                 # only the rule-on controllers keep the key
        args = [nat.ptr(np.ascontiguousarray(a, np.int32)) for a in (st, sl_, it, bk["md_time"], bk["md_seq"], bk["md_cnt"])]
        assert L.lmpc_books_set(c._h, *args) == 0
        assert (c.books()["ss_time"][1::2, 0] == LANE_UNSAFE_KEY + 5).all()
    finally:
        c.close()
    c = _controller(B)
    try:
        _seeded(c, np.arange(B), hook=lambda c: c.set_lane_rules(ROWS, np.arange(B) % 3))
        ref = _laps(c, laps=1)
    finally:
        c.close()
    c = _controller(B)
    try:
        c.set_lane_rules(ROWS, np.arange(B) % 3)
        for bad in ([(1, -1.0)], [(3, 0.0)]):
            assert call(c, bad, np.zeros(B)) == LMPC_E_INVALID
        _seeded(c, np.arange(B))
        got = _laps(c, laps=1)
        assert call(c, [(0, 0.0)], np.zeros(B)) == LMPC_E_STATE          # laps are stored: installing ...
        assert L.lmpc_set_lane_rules(c._h, None, 0, None) == LMPC_E_STATE  # ... or removing
    finally:
        c.close()
    for key in KEYS:
        assert np.array_equal(ref[key], got[key]), key
    m = BatchedController(rp.mpc_params(12), 4, TRACK.seg_table, TRACK.TrackLength, trToUse=4)
    try:
        assert call(m, [(1, 0.0)], np.zeros(4)) == LMPC_E_STATE        # no safe set
    finally:
        m.close()
