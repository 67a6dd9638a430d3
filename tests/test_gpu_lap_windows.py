"""GPU tier: per-controller lap windows (lmpc_set_lap_windows).

No table, an all-unbounded table and a reverted table equal the closed loop without the call bit for bit (independent and
pooled: books, states, health, reports, snapshot records).  A window that covers every lap filed selects the laps no window
selects and drives the same closed loop.  The device books follow the window-aware exact lists of tests/support/lapbook_window.py
event by event (the method of test_gpu_lap_books_exact.py, whose helpers this file drives), at ss_cap = W and model_cap = Wm, and
a window never sets health bit 64.  Windows of the most recent laps select exactly those laps; windows interleaved in one batch
equal one handle per window (lap budgets, and pooled with one group per window); the host-slot hand-over's host books select
what the device books select; a snapshot resumes bit for bit under the same windows; refused calls change nothing."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                # noqa: E402
from racinglmpc_b200 import _native as nat                        # noqa: E402
from racinglmpc_b200.controller import BatchedController          # noqa: E402
from racinglmpc_b200.reference_params import TrackParams, LapWindowParams as W   # noqa: E402
from lapbook_window import WindowBooks                            # noqa: E402
import test_gpu_lap_books_exact as gx                              # noqa: E402

LMPC_E_INVALID, LMPC_E_STATE = -1, -4
X0 = np.array([0.5, 0, 0, 0, 0, 0.0])
TRACK = TrackParams.l_shaped()
B = 16
WINDOWS = [W(0, 0), W(4, 4), W(7, 5), W(5, 0)]                   # on the rollout_mc handle: numSS_it 4, ss_cap 7, trToUse 4, model_cap 5
IDX = np.arange(B) % len(WINDOWS)
KEYS = ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt", "sel",
        "is_prev", "prev_slot", "used", "flags", "unsolved")


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _controller(Bc, ss_cap=7, model_cap=5):
    _, _, _, _, Qts, par = rp.lmpc_params(12)
    return BatchedController(par, Bc, TRACK.seg_table, TRACK.TrackLength, trToUse=4, numSS_Points=48, numSS_it=4,
                             QterminalSlack=Qts, Tmax=1280, ss_cap=ss_cap, model_cap=model_cap)


def _seeded(c, streams, hook=None, reports=0):
    if hook is not None:
        hook(c)
    c.enable_rollout(Tcl=1024)
    if reports:
        c.enable_lap_reports(reports)
    c.set_noise_streams(streams)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))


def _laps(c, laps=3, pooled=False, records=False):
    c.set_lap_budget(laps)
    rows = torch.zeros(c.pool_groups * 3, 288, 9, dtype=torch.float64, device="cuda")
    meta = torch.zeros(c.pool_groups * 3, 4, dtype=torch.int32, device="cuda")
    for n in range(1, 300 * laps + 1):
        c.rollout_step(seed=1234)
        c.rollout_commit_laps_dev()
        if pooled and n in (320, 520):
            c.pool_export(3, 288, 0, rows, meta)
            c.pool_import(c.pool_groups * 3, 2, 288, 0, rows, meta)
        if n % 8 == 0 and n > 520 and c.books()["lap_n"].min() >= laps:
            break
    flags, unsolved = c.rollout_health()
    out = dict(c.books(), flags=flags, unsolved=unsolved, **c.rollout_state())
    if getattr(c, "lap_report_cap", 0):
        out.update({"rep_" + k: v for k, v in c.lap_reports().items()})
    if records:
        out["records"] = c.snapshot().cpu().numpy()
    return out


def _run(hook, pooled=False, Bc=B, **kw):
    c = _controller(Bc, **kw)
    try:
        _seeded(c, np.arange(Bc), hook=hook, reports=4)
        return _laps(c, pooled=pooled, records=True)
    finally:
        c.close()


@pytest.mark.parametrize("pooled", [False, True], ids=["independent", "pooled"])
def test_unbounded_and_reverted_tables_equal_no_table(pooled):
    _need_gpu()
    ref = _run(None, pooled)
    assert (ref["lap_n"] == 3).all()
    for hook in (lambda c: c.set_lap_windows([W.unbounded()], np.zeros(B, int)),
                 lambda c: c.set_lap_windows([W.unbounded(), W(0, 0)], IDX % 2),
                 lambda c: (c.set_lap_windows(WINDOWS, IDX), c.set_lap_windows(None))):
        got = _run(hook, pooled)
        for key in ref:
            assert np.array_equal(ref[key], got[key]), key


def _lap_numbers(r, b):
    sel = [int(r["ss_lap"][b][s]) for s in r["sel"][b]]
    used = [int(r["md_seq"][b][u]) for u in r["used"][b]]
    return sel, used


def test_a_window_covering_every_lap_selects_and_drives_what_no_window_does():
    """4 seeded copies + 3 own laps = 7 laps and 7 arrivals: windows of 8 cover them all (on pools of 8 slots)."""
    _need_gpu()
    ref = _run(None, ss_cap=8, model_cap=8)
    got = _run(lambda c: c.set_lap_windows([W(8, 8)], np.zeros(B, int)), ss_cap=8, model_cap=8)
    assert (ref["lap_n"] == 3).all() and (ref["it"] == 7).all()
    for key in ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "it", "md_cnt", "is_prev", "flags", "unsolved", "rep_steps",
                "rep_ipm_iters"):
        assert np.array_equal(ref[key], got[key]), key
    for b in range(B):
        assert _lap_numbers(ref, b) == _lap_numbers(got, b), b


def test_windows_of_the_most_recent_laps_select_exactly_those_laps():
    _need_gpu()
    r = _run(lambda c: c.set_lap_windows([W(4, 4)], np.zeros(c.B, int)), Bc=8)
    assert (r["lap_n"] == 3).all() and (r["flags"] & 64 == 0).all()
    for b in range(8):
        sel, used = _lap_numbers(r, b)
        it, cnt = int(r["it"][b]), int(r["md_cnt"][b])
        assert sorted(sel) == list(range(it - 4, it)), (b, sel)
        assert sorted(used) == list(range(cnt - 4, cnt)), (b, used)


def _per_window(body, windows=WINDOWS, idx=IDX):
    """body(h, members) on one handle per window, every controller of it under that window, on their noise streams; the
    results scattered back to the positions of the batch"""
    out = {}
    for k, w in enumerate(windows):
        members = np.nonzero(idx == k)[0]
        h = _controller(members.size)
        try:
            res = body(h, members, w)
        finally:
            h.close()
        for key, val in res.items():
            out.setdefault(key, [None] * idx.size)
            for j, b in enumerate(members):
                out[key][b] = val[j]
    return out


def test_interleaved_windows_equal_one_handle_per_window():
    _need_gpu()
    c = _controller(B)
    try:
        _seeded(c, np.arange(B), hook=lambda c: c.set_lap_windows(WINDOWS, IDX))
        assert [c.lap_windows_of(b) for b in range(B)] == [(WINDOWS[k].ss_window, WINDOWS[k].model_window) for k in IDX]
        res = _laps(c)
    finally:
        c.close()
    own = _per_window(lambda h, m, w: (_seeded(h, m, hook=lambda h: h.set_lap_windows([w], np.zeros(h.B, int))), _laps(h))[1])
    for key in KEYS:
        for b in range(B):
            assert np.array_equal(res[key][b], own[key][b]), (key, b)
    # the windows change what is selected
    assert any(_lap_numbers(res, b) != _lap_numbers(res, b - 1) for b in range(1, 4))


def test_pooled_with_one_group_per_window_equals_one_handle_per_window():
    _need_gpu()
    c = _controller(B)
    try:
        _seeded(c, np.arange(B), hook=lambda c: (c.set_lap_windows(WINDOWS, IDX), c.set_pool_groups(IDX, len(WINDOWS))))
        res = _laps(c, laps=2, pooled=True)
    finally:
        c.close()
    own = _per_window(lambda h, m, w: (_seeded(h, m, hook=lambda h: h.set_lap_windows([w], np.zeros(h.B, int))),
                                       _laps(h, laps=2, pooled=True))[1])
    for key in KEYS:
        for b in range(B):
            assert np.array_equal(res[key][b], own[key][b]), (key, b)
    assert (res["it"] > 4 + 2).any()                                   # imports were filed


# (numSS_it, ss_cap, trToUse, model_cap) of test_gpu_lap_books_exact.py, and the windows interleaved over its batch: ss_cap = W
# and model_cap = Wm in every configuration, numSS_it = 1 (imports dropped on arrival), model_window = trToUse
EXACT = [((4, 6, 4, 5), [(0, 0), (4, 4), (6, 5), (5, 0)]),
         ((4, 4, 4, 4), [(4, 4), (0, 4), (4, 0)]),
         ((1, 2, 1, 1), [(1, 1), (2, 1), (0, 1), (2, 0)]),
         ((2, 4, 8, 8), [(2, 8), (4, 0), (3, 8), (0, 8)])]


@pytest.mark.parametrize("cfg, wins", EXACT, ids=["nit%d_ss%d_tr%d_md%d" % e[0] for e in EXACT])
def test_device_books_follow_the_window_lists_event_by_event(cfg, wins):
    _need_gpu()
    rng = np.random.default_rng(2000 + [e[0] for e in EXACT].index(cfg))
    c = gx._controller(cfg, gx.B)
    widx = np.arange(gx.B) % len(wins)
    c.set_lap_windows([W(*w) for w in wins], widx)
    grp = np.arange(gx.B) % gx.G
    c.set_pool_groups(grp, gx.G)
    models = [WindowBooks(*cfg, Tmax=gx.TMAX, TrackLength=TRACK.TrackLength, ss_window=wins[widx[b]][0], md_window=wins[widx[b]][1])
              for b in range(gx.B)]
    windowed = [wins[widx[b]][0] > 0 for b in range(gx.B)]
    lengths = [gx._lap_lengths(rng, b % 6, gx.ROUNDS + 1) for b in range(gx.B)]
    lap = [0] * gx.B
    dropped = 0
    try:
        for r in range(gx.ROUNDS):
            if r % gx.XEVERY == 0:
                before = [m.seq - m.it for m in models]
                fresh = gx._import_round(c, models, rng, grp)
                bk = gx._check_books(c, models, fresh)
                dropped += sum((m.seq - m.it) > x for m, x, w in zip(models, before, windowed) if w)
                _check_windows(c, models, bk, windowed)
            fresh = gx._own_round(c, models, rng, lengths, lap)
            bk = gx._check_books(c, models, fresh)
            _check_windows(c, models, bk, windowed)
            if r % 5 == 4:
                gx._check_pools(c, models, bk, cfg)
    finally:
        c.close()
    assert max(len(m.lap_hist) for m in models) >= 44
    if cfg[0] == 1:
        assert dropped > 0                                             # imports a window left out of the safe set


def _check_windows(c, models, bk, windowed):
    """What gx._check_books leaves out: the model laps a window must keep are stored, and a window never sets bit 64."""
    flags, _ = c.rollout_health()
    for b, m in enumerate(models):
        if windowed[b]:
            assert not m.dead and not flags[b] & 64, b
        if m.dead:
            continue
        md = {int(s) for s in bk["md_seq"][b] if s >= 0}
        assert m.md_resident() <= md, (b, [(t, s) for t, s, _ in m.md])


def _host_books_laps(c, streams, laps=2):
    c.enable_rollout(Tcl=1024)
    c.set_noise_streams(streams)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    _, n = c.rollout_done()
    c.rollout_seed_from_record(n, copies=4)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))
    for _ in range(300 * laps):
        c.rollout_step(seed=1234)
        done, n = c.rollout_done()
        if done.any():
            c.rollout_finish_laps(done, n)


def test_host_slot_hand_over_selects_what_the_device_books_select():
    """Host books with windows through two LMPC laps of the host-slot hand-over; then the same tables handed to the device books
    (lmpc_books_set), whose refresh must select, flag and use the laps the host books pushed."""
    _need_gpu()
    c = _controller(B)
    try:
        c.set_lap_windows(WINDOWS, IDX)
        _host_books_laps(c, np.arange(B))
        c._flush()
        inv = [{s: ln for ln, s in c.ss_book[b].slot_of.items()} for b in range(B)]
        minv = [{s: ln for ln, s in c.model_book[b].slot_of.items()} for b in range(B)]
        host = [([inv[b][int(s)] for s in c._sel[b]], [int(v) for v in c._isp[b]], inv[b].get(int(c._prev[b]), -1),
                 [minv[b][int(s)] for s in c._used[b]]) for b in range(B)]
        assert min(c.it) >= 6
        c.enable_device_books()
        bk = c.books()
        for b in range(B):
            dev = ([int(bk["ss_lap"][b][s]) for s in bk["sel"][b]], [int(v) for v in bk["is_prev"][b]],
                   int(bk["ss_lap"][b][bk["prev_slot"][b]]), [int(bk["md_seq"][b][u]) for u in bk["used"][b]])
            assert dev == host[b], (b, c.lap_windows_of(b))
    finally:
        c.close()


def test_snapshot_resumes_bit_for_bit_under_the_same_windows():
    _need_gpu()

    def run(split):
        c = _controller(8)
        idx = np.arange(8) % len(WINDOWS)
        try:
            _seeded(c, np.arange(8), hook=lambda c: c.set_lap_windows(WINDOWS, idx))
            c.set_lap_budget(2)
            for n in range(1, 600):
                c.rollout_step(seed=1234)
                c.rollout_commit_laps_dev()
                if split and n == 150:
                    rec, clock = c.snapshot(), c.rollout_clock
                    d = _controller(8)
                    d.set_lap_windows(WINDOWS, idx)
                    d.enable_rollout(Tcl=1024)
                    d.set_noise_streams(np.arange(8))
                    d.restore(rec)
                    d.rollout_clock = clock
                    d.set_lap_budget(2)
                    c.close()
                    c = d
                if n % 8 == 0 and c.books()["lap_n"].min() >= 2:
                    break
            flags, unsolved = c.rollout_health()
            return dict(c.books(), flags=flags, unsolved=unsolved, **c.rollout_state())
        finally:
            c.close()
    a, b = run(False), run(True)
    for key in KEYS:
        assert np.array_equal(a[key], b[key]), key


def test_refusals_change_nothing():
    _need_gpu()
    L = nat.lib()

    def call(c, windows, idx):
        rows = (nat.LapWindowParams * len(windows))(*[nat.LapWindowParams(*w) for w in windows])
        return L.lmpc_set_lap_windows(c._h, rows, len(windows), nat.ptr(np.ascontiguousarray(idx, np.int32)))
    c = _controller(B)
    try:
        c.set_lap_windows(WINDOWS, IDX)
        zero = np.zeros(B)
        assert call(c, [(3, 0)], zero) == LMPC_E_INVALID                # below numSS_it
        assert call(c, [(8, 0)], zero) == LMPC_E_INVALID                # above ss_cap
        assert call(c, [(-1, 0)], zero) == LMPC_E_INVALID
        assert call(c, [(0, 3)], zero) == LMPC_E_INVALID                # below trToUse
        assert call(c, [(0, 6)], zero) == LMPC_E_INVALID                # above model_cap
        assert call(c, [(4, 4)], np.full(B, 1)) == LMPC_E_INVALID        # bad index
        assert L.lmpc_set_lap_windows(c._h, None, 1, None) == LMPC_E_INVALID
        # the other install order: a lap count above a controller's window
        rows = (nat.SsLapsParams * 1)(nat.SsLapsParams(4))
        c2 = _controller(4)
        try:
            c2.set_ss_laps([2], np.zeros(4, int))
            c2.set_lap_windows([W(3, 0)], np.zeros(4, int))
            assert L.lmpc_set_ss_laps(c2._h, rows, 1, nat.ptr(np.zeros(4, np.int32))) == LMPC_E_INVALID
            assert L.lmpc_set_ss_laps(c2._h, None, 0, None) == LMPC_E_INVALID   # the handle's 4 against the window 3
        finally:
            c2.close()
        _seeded(c, np.arange(B))
        res = _laps(c)
        assert call(c, [(4, 4)], zero) == LMPC_E_STATE                  # a lap is stored: the table is fixed from now on
        assert L.lmpc_set_lap_windows(c._h, None, 0, None) == LMPC_E_STATE
    finally:
        c.close()
    c = _controller(B)
    try:
        _seeded(c, np.arange(B), hook=lambda c: c.set_lap_windows(WINDOWS, IDX))
        ref = _laps(c)
    finally:
        c.close()
    for key in KEYS:
        assert np.array_equal(res[key], ref[key]), key
    m = BatchedController(rp.mpc_params(12), 4, TRACK.seg_table, TRACK.TrackLength, trToUse=4)
    try:
        assert call(m, [(4, 0)], np.zeros(4)) == LMPC_E_INVALID        # no safe set
        assert call(m, [(0, 4)], np.zeros(4)) == 0                     # the model window alone is fine
    finally:
        m.close()
