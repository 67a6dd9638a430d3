"""GPU tier: lane margins (lmpc_set_lane_margins).

At every instantiated (N, M), MPC- and LMPC-type, a table of margin0 = 0 rows solves bit for bit what a handle whose parameter
sets equal its own parameters solves (and, at N <= 24, what a handle without a table solves: the N >= 32 rounding of the SETS
kernel is an open finding, DESIGN.md), and a margin m solves what parameter sets carrying bx - m solve.  In the closed loop a fixed
margin equals such parameter sets bit for bit (books, states, step results) while its reports judge the given lane; adaptive
margins follow tests/support/lane_margin.py after every hand-over on a narrow lane with and without measurement noise; rows of all
three modes interleaved equal one handle per row; a hand-over that changes m_b drops that controller's warm-start record only;
a snapshot resumes bit for bit and mismatched records are refused; retired controllers and imports leave m_b alone; refused
calls change nothing."""
import copy
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import BatchedFTOCP, workloads, reference_params as rp   # noqa: E402
from racinglmpc_b200 import _native as nat                                   # noqa: E402
from racinglmpc_b200.controller import BatchedController                      # noqa: E402
from racinglmpc_b200.reference_params import TrackParams, LaneMarginParams as G   # noqa: E402
from oracle import ftocp                                                      # noqa: E402
import lane_margin as lm                                                      # noqa: E402
import hostcore as hc                                                         # noqa: E402
import test_gpu_param_sets as ps                                              # noqa: E402

LMPC_E_INVALID, LMPC_E_STATE = -1, -4
X0 = np.array([0.5, 0, 0, 0, 0, 0.0])
TRACK = TrackParams.l_shaped()
FX = rp.lmpc_params(12)[5].Fx
B = 12
KEYS = ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt", "sel",
        "is_prev", "prev_slot", "used", "flags", "unsolved")
ROWS = [G(0), G(1, 0.05, 0.05), G(2, 0.005, 0.1, 0.01, 0.0025)]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _raw(h, rows, idx):
    """lmpc_set_lane_margins with rows (mode, margin0, margin_max, step_up, step_down), or removal (rows None)"""
    L = nat.lib()
    if rows is None:
        return L.lmpc_set_lane_margins(h, None, 0, None)
    arr = (nat.LaneMarginParams * len(rows))(*[nat.LaneMarginParams(r[0], 0, *r[1:]) for r in rows])
    return L.lmpc_set_lane_margins(h, arr, len(rows), nat.ptr(np.ascontiguousarray(idx, np.int32)))


# ---- 1. QPs at every instantiation ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Nh,M", [(n, m) for n, m in nat.SHAPE_GRID])
def test_margins_solve_what_parameter_sets_solve_at_every_instantiation(gold, track, Nh, M):
    _need_gpu()
    Bq = 64
    x0, uold, abc = workloads.ltv_mpc_batch(Bq, N=48)
    abc = np.ascontiguousarray(abc[:, :Nh])
    if M == 0:
        _, base = ftocp.mpc_params(6, 2, Nh, 0.8)
        kw, lm_in, keys, qts = {}, (), ps.MPC_KEYS, None
    else:
        _, _, _, _, qts, base = ftocp.lmpc_params(track, Nh)
        kw, keys = dict(numSS_Points=M, numSS_it=4), ps.LMPC_KEYS
        xP = gold["pid_x"]
        SS = np.zeros((Bq, 6, M)); Qf = np.zeros((Bq, M))
        P = M // 4
        for b in range(Bq):
            i0 = 40 + 3 * b
            for j in range(4):
                blk = xP[i0 + 2 * j:i0 + 2 * j + P].copy()
                blk[:, 0:3] += 1e-3 * (j + 1)
                SS[b, :, P * j:P * j + P] = blk.T
                Qf[b, P * j:P * j + P] = 300.0 - (i0 + np.arange(P)) * 0.3 + 5.0 * j
        lm_in = (SS, Qf)
    mp = nat.make_model_params(TRACK.seg_table, TRACK.TrackLength, 4)

    def handle(margins=None, bxs=None):
        s = BatchedFTOCP(base, batch=Bq, QterminalSlack=qts, **kw)
        if margins is not None:
            nat.check(nat.lib().lmpc_store_create(s._h, C.byref(mp), 6 if M else 0, 5, 256))
            nat.check(_raw(s._h, *margins))
        if bxs is not None:                                            # parameter sets that differ from base only in bx
            sets = []
            for bx in bxs:
                p = copy.deepcopy(base)
                p.bx = np.asarray(bx, float)
                sets.append(p)
            s.set_param_sets(sets, np.arange(Bq) % len(bxs), [qts] * len(bxs) if M else None)
        o = s.solve(x0, uold, abc, *lm_in)
        s.close()
        return o

    bx = np.asarray(base.bx, float).ravel()
    zero = handle(margins=([(1, 0.0, 0.0, 0.0, 0.0)], np.zeros(Bq)))
    ps._same(zero, handle(bxs=[bx]), keys, slice(None))
    if Nh <= 24:
        ps._same(zero, handle(), keys, slice(None))
    # every mode interleaved: 0, a fixed 0.05, an adaptive row planning with its margin0 0.02
    mixed = handle(margins=([(0, 0.0, 0.0, 0.0, 0.0), (1, 0.05, 0.05, 0.0, 0.0), (2, 0.02, 0.1, 0.01, 0.0)], np.arange(Bq) % 3))
    ps._same(mixed, handle(bxs=[bx, lm.planning_bx(bx, 0.05), lm.planning_bx(bx, 0.02)]), keys, slice(None))


# ---- closed loop ------------------------------------------------------------------------------------------------------------
def _par(width, N=12):
    p = rp.lmpc_params(N)[5]
    return SimpleNamespace(**{**vars(p), "bx": np.array([width, width])})


def _controller(Bc, widths=None, warm=False):
    _, _, _, _, Qts, par = rp.lmpc_params(12)
    c = BatchedController(par, Bc, TRACK.seg_table, TRACK.TrackLength, trToUse=4, numSS_Points=48, numSS_it=4,
                          QterminalSlack=Qts, Tmax=1280, ss_cap=7, model_cap=5, warm_start=warm)
    if widths is not None:
        c.set_param_sets([_par(w) for w in widths], np.arange(Bc) % len(widths))
    return c


def _seeded(c, streams, hook=None, reports=0, meas=None):
    if hook is not None:
        hook(c)
    c.enable_rollout(Tcl=1024)
    if reports:
        c.enable_lap_reports(reports)
    if meas is not None:
        c.set_measurement_noise([rp.MeasurementParams(sigma=(s,) * 6, clip=(5 * s,) * 6) for s in meas],
                                np.arange(c.B) % len(meas))
    c.set_noise_streams(streams)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (c.B, 1)), np.tile(X0, (c.B, 1)))


def _laps(c, laps=3, each=None, pooled=False):
    """Drive until every controller has handed over `laps` laps; each(c, done) runs before every hand-over"""
    c.set_lap_budget(laps)
    rows = torch.zeros(c.pool_groups * 3, 288, 9, dtype=torch.float64, device="cuda")
    meta = torch.zeros(c.pool_groups * 3, 4, dtype=torch.int32, device="cuda")
    for n in range(1, 400 * laps + 1):
        c.rollout_step(seed=1234)
        if each is not None:
            each(c, c.rollout_done()[0])
        c.rollout_commit_laps_dev()
        if pooled and n in (320, 520):
            m = c.lane_margin_values()
            c.pool_export(3, 288, 0, rows, meta)
            c.pool_import(c.pool_groups * 3, 2, 288, 0, rows, meta)
            assert np.array_equal(m, c.lane_margin_values())                # an import leaves every margin as it was
        if n % 8 == 0 and c.books()["lap_n"].min() >= laps:
            break
    flags, unsolved = c.rollout_health()
    out = dict(c.books(), flags=flags, unsolved=unsolved, **c.rollout_state())
    out.update({"step_" + k: v for k, v in c.step_results().items()})
    return out


def test_fixed_margin_equals_tightened_parameter_sets_and_reports_judge_the_given_lane():
    _need_gpu()
    m = 0.05
    verdicts = {}

    def record(c, done):
        for b in np.nonzero(done)[0]:
            x, _ = c.rollout_get_lap(int(b))
            verdicts.setdefault(int(b), []).append(lm.lap_left_lane(x, FX, [0.4, 0.4]))
    a = _controller(B)
    try:
        _seeded(a, np.arange(B), hook=lambda c: c.set_lane_margins([G(1, m, m)], np.zeros(B, int)), reports=8)
        assert np.array_equal(a.lane_margin_values(), np.full(B, m))
        got = _laps(a, each=record)
        rep = a.lap_reports()
    finally:
        a.close()
    t = _controller(B, widths=[0.4 - m])
    try:
        _seeded(t, np.arange(B))
        want = _laps(t)
    finally:
        t.close()
    for key in want:
        assert np.array_equal(got[key], want[key]), key
    for b in range(B):
        n = min(int(rep["n"][b]), 8)
        assert n >= 3
        for j in range(n):                                             # judged against bx = 0.4, not the planning 0.35
            assert bool(rep["viol_steps"][b, j] > 0) == verdicts[b][j] == bool(rep["viol_max"][b, j] > 0.0), (b, j)


def test_fixed_margin_lane_rules_judge_the_given_lane():
    """Under a fixed margin with lane rules at lane_tol 0, an own lap is judged against bx = 0.4, not the planning 0.35: its report
    bit and its safe-set key follow the host verdict of its record rows against 0.4."""
    _need_gpu()
    m = 0.05
    verdicts = {}

    def record(c, done):
        for b in np.nonzero(done)[0]:
            x, _ = c.rollout_get_lap(int(b))
            verdicts.setdefault(int(b), []).append(lm.lap_left_lane(x, FX, [0.4, 0.4]))
    a = _controller(B)
    try:
        _seeded(a, np.arange(B), hook=lambda c: (c.set_lane_margins([G(1, m, m)], np.zeros(B, int)),
                                                 c.set_lane_rules([rp.LaneRuleParams(1, 0.0)], np.zeros(B, int))), reports=8)
        got = _laps(a, laps=4, each=record)
        rep = a.lap_reports()
    finally:
        a.close()
    judged = 0
    for b in range(B):
        n = min(int(rep["n"][b]), 8)
        assert n >= 4
        for j in range(n):
            assert bool(rep["flags"][b, j] & nat.REPORT_LANE_UNSAFE) == verdicts[b][j] == bool(rep["viol_steps"][b, j] > 0), (b, j)
        for s in range(got["ss_lap"].shape[1]):                        # own lap j is lap number 4 + j (after 4 seeded copies)
            j = int(got["ss_lap"][b, s]) - 4
            if 0 <= j < len(verdicts[b]):
                assert (int(got["ss_time"][b, s]) >= nat.LANE_UNSAFE_KEY) == verdicts[b][j], (b, s)
                judged += 1
    assert judged > 0


def test_shaped_handle_with_a_margin_equals_tightened_parameter_sets():
    _need_gpu()
    m = 0.03
    shapes, sidx = [(12, 48), (8, 48), (12, 24)], np.arange(B) % 3

    def run(hook):
        c = _controller(B)
        try:
            c.set_shapes(shapes, sidx)
            _seeded(c, np.arange(B), hook=hook)
            return _laps(c, laps=2)
        finally:
            c.close()
    a = run(lambda c: c.set_lane_margins([G(1, m, m)], np.zeros(B, int)))
    t = run(lambda c: c.set_param_sets([_par(0.4 - m)], np.zeros(B, int)))
    for key in KEYS:
        assert np.array_equal(a[key], t[key]), key


def _adaptive(meas):
    widths = (0.4, 0.1, 0.03)
    rows = [G(2, 0.0, 0.02, 0.01, 0.0025), G(2, 0.005, 0.025, 0.01, 0.0), G(1, 0.01, 0.01)]
    idx = (np.arange(B) // 3) % 3
    bx = [widths[b % len(widths)] for b in range(B)]
    c = _controller(B, widths=widths)
    m = {}
    seen = []
    try:
        _seeded(c, np.arange(B), hook=lambda c: c.set_lane_margins(rows, idx), reports=8, meas=meas)
        host = np.array([lm.start(rows[k]) for k in idx])
        assert np.array_equal(c.lane_margin_values(), host)

        def each(c, done):
            for b in np.nonzero(done)[0]:
                x, _ = c.rollout_get_lap(int(b))
                left = lm.lap_left_lane(x, FX, [bx[b]] * 2)
                seen.append((int(b), left))
                host[b] = lm.hand_over(rows[idx[b]], host[b], x, FX, [bx[b]] * 2)
            c.rollout_commit_laps_dev()
            assert np.array_equal(c.lane_margin_values(), host)
            m["last"] = host.copy()
        _laps(c, laps=6, each=lambda c, done: each(c, done))
        return c.lap_reports(), seen, m["last"]
    finally:
        c.close()


def test_adaptive_margins_follow_the_host_rule_without_measurement_noise():
    _need_gpu()
    rep, seen, last = _adaptive(None)
    lefts = sum(l for _, l in seen)
    assert 0 < lefts < len(seen)                                       # the narrow lanes are crossed, the wide one kept
    k = np.zeros(B, int)
    for b, left in seen:
        if k[b] < 8:
            assert bool(rep["viol_steps"][b, k[b]] > 0) == left, (b, k[b])
        k[b] += 1
    assert (last[0::3] > 0).any() or (last[1::3] > 0.005).any()        # some margin moved


def test_adaptive_margins_follow_the_measured_record_under_measurement_noise():
    _need_gpu()
    _, seen, _ = _adaptive((0.0, 0.01))
    assert len(seen) >= 6 * B
    assert 0 < sum(l for _, l in seen) < len(seen)                     # crossings and clean laps both feed the rule


def test_interleaved_rows_equal_one_handle_per_row():
    _need_gpu()
    widths = (0.4, 0.15)
    idx = np.arange(B) % len(ROWS)
    wsel = (np.arange(B) // 3) % 2
    c = _controller(B)
    try:
        c.set_param_sets([_par(w) for w in widths], wsel)
        _seeded(c, np.arange(B), hook=lambda c: c.set_lane_margins(ROWS, idx))
        res = _laps(c, laps=4)
        mres = c.lane_margin_values()
    finally:
        c.close()
    for k, row in enumerate(ROWS):
        members = np.nonzero(idx == k)[0]
        h = _controller(members.size)
        try:
            h.set_param_sets([_par(w) for w in widths], wsel[members])
            _seeded(h, members, hook=lambda h: h.set_lane_margins([row], np.zeros(h.B, int)))
            own = _laps(h, laps=4)
            assert np.array_equal(mres[members], h.lane_margin_values())
        finally:
            h.close()
        for key in KEYS:
            for j, b in enumerate(members):
                assert np.array_equal(res[key][b], own[key][j]), (key, b)


def _late(status, resid):
    return status == 1 and (max(resid[0], resid[1]) > 1.000001e-9 or resid[2] > 1.000001e-11)


def test_warm_start_a_changed_margin_drops_that_record_only():
    """With warm start, a hand-over that changes m_b clears that controller's warm_valid and no other; every sampled warm-started
    QP (every third step and every step after a margin changed) agrees within 1e-6 with a cold host solve of the same QP on the
    controller's planning lane bx - m_b, the warm-start tests' tolerance, wherever neither is a late accept."""
    _need_gpu()
    widths = (0.4, 0.03)
    c = _controller(B, widths=widths, warm=True)
    rows = [G(2, 0.0, 0.02, 0.01, 0.0025)]
    Qts = rp.lmpc_params(12)[4]
    consts = {}
    changed, checked, warm_started = [], 0, 0
    try:
        _seeded(c, np.arange(B), hook=lambda c: c.set_lane_margins(rows, np.zeros(B, int)))
        c.set_lap_budget(4)
        wv = lambda: np.array([c.read_buffer("warm_valid", b, (1,), np.int32)[0] for b in range(B)])   # noqa: E731
        moved_last = False
        for n in range(1, 2000):
            check = n % 3 == 0 or moved_last
            if check:
                x0 = c.rollout_state()["x"].copy()
                old = np.stack([c.read_buffer("OldInput", b, (2,)) for b in range(B)])
                m, v_in, live = c.lane_margin_values(), wv(), c.books()["lap_n"] < 4
            c.rollout_step(seed=1234)
            if check:
                r = c.step_results()
                abc = c.read_buffer("abc", 0, (B, 12, 54))
                xp, up = c.read_buffer("xPred", 0, (B, 13, 6)), c.read_buffer("uPred", 0, (B, 12, 2))
                SS, Qf = c.read_buffer("SS_sel", 0, (B, 6, 48)), c.read_buffer("Qfun_sel", 0, (B, 48))
                for b in np.nonzero(live)[0]:
                    w = widths[b % 2]
                    key = (w, float(m[b]))
                    if key not in consts:
                        consts[key] = hc.make_const(_par(float(lm.planning_bx([w], m[b])[0])), Qts)
                    cold = hc.solve(consts[key], 12, abc[b], x0[b], old[b], SS[b], Qf[b])
                    if not (_late(int(r["status"][b]), r["resid"][b]) or _late(cold["status"], (cold["r_prim"], cold["r_dual"],
                                                                                                cold["gap"]))):
                        assert max(np.abs(xp[b] - cold["x"]).max(), np.abs(up[b] - cold["u"]).max()) < 1e-6, (n, b)
                        checked += 1
                        warm_started += int(v_in[b] >= 1)
            m0, w0 = c.lane_margin_values(), wv()
            c.rollout_commit_laps_dev()
            m1, w1 = c.lane_margin_values(), wv()
            moved = m1 != m0
            moved_last = bool(moved.any())
            changed.extend(np.nonzero(moved)[0].tolist())
            assert (w1[moved] == 0).all()
            assert np.array_equal(w1[~moved], w0[~moved])
            if n % 8 == 0 and c.books()["lap_n"].min() >= 4:
                break
    finally:
        c.close()
    assert changed
    assert checked > 100 and warm_started > checked // 2


def test_rollout_mc_capture_records_margin_rows_and_resumes():
    """rollout_mc.run under a mode 2 table (with measurement noise so that laps cross and margins move): 3 laps captured and
    resumed to 5 equal a straight run to 5 bit for bit, margins included; a start under other margin rows is refused."""
    _need_gpu()
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "benchmarks"))
    try:
        import rollout_mc as rm
    finally:
        sys.path.pop(0)
    Bm = 256
    rows = [G(2, 0.0, 0.1, 0.01, 0.0), G(1, 0.02, 0.02)]                   # step_down 0: a margin that moved stays up
    kw = dict(batch=Bm, local=0, mode="independent", lane_margin_sets=(rows, np.arange(Bm) % 2),
              measurement_sets=([rp.MeasurementParams((0.01,) * 6, (0.05,) * 6)], np.zeros(Bm, int)))
    fin5, bk5 = {}, {}
    o5 = rm.run(laps=5, final=fin5, books=bk5, **kw)
    cap = {}
    rm.run(laps=3, capture=cap, **kw)
    assert cap["diverged_step"] is None and "lane_margin_sets" in cap["tables"]
    fin, bk = {}, {}
    o = rm.run(laps=5, start=cap, final=fin, books=bk, **kw)
    assert o["resume_exact"] and o["closed_loop_steps"] == o5["closed_loop_steps"]
    assert (bk5["lane_margins"][0::2] > 0).any()                       # some adaptive margin moved
    for k in bk5:
        assert np.array_equal(np.asarray(bk5[k]), np.asarray(bk[k])), ("books", k)
    for k in fin5:
        assert np.array_equal(np.asarray(fin5[k]), np.asarray(fin[k])), ("end state", k)
    other = dict(kw, lane_margin_sets=([G(2, 0.0, 0.1, 0.01, 0.0025), rows[1]], np.arange(Bm) % 2))
    with pytest.raises(ValueError, match="lane margins"):
        rm.run(laps=5, start=cap, **other)


def test_snapshot_resumes_bit_for_bit_and_mismatched_records_are_refused():
    _need_gpu()
    idx = np.arange(8) % len(ROWS)
    hook = lambda c: c.set_lane_margins(ROWS, idx)                    # noqa: E731
    saved = {}

    def run(split):
        c = _controller(8, widths=(0.4, 0.15))
        try:
            _seeded(c, np.arange(8), hook=hook)
            c.set_lap_budget(5)
            for n in range(1, 3000):
                c.rollout_step(seed=1234)
                c.rollout_commit_laps_dev()
                if split and "rec" not in saved and n % 8 == 0 and c.books()["lap_n"].min() >= 3:
                    rec, clock = c.snapshot(), c.rollout_clock
                    saved["rec"], saved["m"] = rec.clone(), c.lane_margin_values()
                    d = _controller(8, widths=(0.4, 0.15))
                    hook(d)
                    d.enable_rollout(Tcl=1024)
                    d.set_noise_streams(np.arange(8))
                    d.restore(rec)
                    assert np.array_equal(d.lane_margin_values(), saved["m"])
                    d.rollout_clock = clock
                    d.set_lap_budget(5)
                    c.close()
                    c = d
                if n % 8 == 0 and c.books()["lap_n"].min() >= 5:
                    break
            flags, unsolved = c.rollout_health()
            return dict(c.books(), flags=flags, unsolved=unsolved, margin=c.lane_margin_values(), **c.rollout_state())
        finally:
            c.close()
    a, b = run(False), run(True)
    for key in KEYS + ("margin",):
        assert np.array_equal(a[key], b[key]), key
    rec = saved["rec"]
    off, nb = nat.decode_snapshot_header(rec[0].cpu().numpy())["sections"]["lane_margin"]
    assert nb == 8
    d = _controller(8, widths=(0.4, 0.15))
    try:
        d.enable_rollout(Tcl=1024)
        d.enable_device_books()
        with pytest.raises(ValueError, match="shape"):
            d.restore(rec)                                             # a record with margins, a handle without a table
        hook(d)
        before, m_before = d.snapshot().cpu().numpy(), d.lane_margin_values()
        bad = rec.clone()
        for v in (-1e-3, float("nan"), 0.5, 0.001):      # negative, non-finite, above / below controller 2's margin_max / margin0
            bad[:, off:off + 8] = torch.from_numpy(np.full((8, 1), v).view(np.uint8)).to(bad.device)
            with pytest.raises(nat.NativeError, match="lane margin"):
                d.restore(bad, [2], [2])
        assert np.array_equal(before, d.snapshot().cpu().numpy()) and np.array_equal(m_before, d.lane_margin_values())
        d.set_lane_margins(None)
        L = nat.lib()
        dst = np.array([0], np.int32)
        assert L.lmpc_snapshot_unpack_dev(d._h, nat.ptr(rec), 8, 1, nat.ptr(dst), None) == LMPC_E_INVALID
        assert "lane margin layout" in L.lmpc_last_error().decode()
    finally:
        d.close()


def test_retired_controllers_and_imports_leave_the_margin():
    _need_gpu()
    c = _controller(B, widths=(0.4, 0.03))
    try:
        _seeded(c, np.arange(B), hook=lambda c: c.set_lane_margins([G(2, 0.0, 0.02, 0.01, 0.0)], np.zeros(B, int)))
        _laps(c, laps=2, pooled=True)
        m, n = c.lane_margin_values(), c.books()["lap_n"].copy()
        for _ in range(300):                                           # every controller has retired at its budget
            c.rollout_step(seed=1234)
            c.rollout_commit_laps_dev()
        assert np.array_equal(c.books()["lap_n"], n) and np.array_equal(c.lane_margin_values(), m)
    finally:
        c.close()


def test_refusals_change_nothing():
    _need_gpu()
    L = nat.lib()
    c = _controller(B, widths=(0.4, 0.05))
    try:
        zero = np.zeros(B)
        assert L.lmpc_get_lane_margins(c._h, nat.ptr(np.zeros(B))) == LMPC_E_STATE          # no table
        for bad in ([(3, 0.0, 0.0, 0.0, 0.0)], [(1, -1e-9, 0.0, 0.0, 0.0)], [(1, float("nan"), 0.0, 0.0, 0.0)],
                    [(2, 0.0, float("inf"), 0.0, 0.0)], [(2, 0.02, 0.01, 0.0, 0.0)], [(2, 0.0, 0.01, -0.01, 0.0)],
                    [(1, 0.05, 0.05, 0.0, 0.0)], [(2, 0.0, 0.05, 0.01, 0.0)]):     # the last two: 0.05 closes the narrow lane
            assert _raw(c._h, bad, zero) == LMPC_E_INVALID, bad
        assert _raw(c._h, [(1, 0.0, 0.0, 0.0, 0.0)], np.full(B, 1)) == LMPC_E_INVALID           # bad index
        assert L.lmpc_set_lane_margins(c._h, None, 1, None) == LMPC_E_INVALID
        assert L.lmpc_get_lane_margins(c._h, nat.ptr(np.zeros(B))) == LMPC_E_STATE
        assert _raw(c._h, [(1, 0.04, 0.04, 0.0, 0.0), (2, 0.0, 0.3, 0.01, 0.0)], (np.arange(B) + 1) % 2) == 0
        m = np.zeros(B)
        assert L.lmpc_get_lane_margins(c._h, nat.ptr(m)) == 0 and np.array_equal(m, np.tile([0.0, 0.04], B // 2))
        # the other install order: parameter sets that close a lane under the installed margins
        rows, idx = nat.make_param_sets(c._p, [_par(0.4), _par(0.04)], np.arange(B) % 2, B, 48, 4)
        assert L.lmpc_set_param_sets(c._h, rows, 2, nat.ptr(idx)) == LMPC_E_INVALID
        rows, idx = nat.make_param_sets(c._p, [_par(0.04), _par(0.4)], np.arange(B) % 2, B, 48, 4)
        assert L.lmpc_set_param_sets(c._h, rows, 2, nat.ptr(idx)) == LMPC_E_INVALID
        # the host-slot hand-over under a mode 2 row
        c.enable_rollout(Tcl=1024)
        fin, sl = np.zeros(B, np.int32), -np.ones(B, np.int32)
        assert L.lmpc_rollout_commit_laps(c._h, nat.ptr(fin), nat.ptr(sl), nat.ptr(sl)) == LMPC_E_STATE
        assert _raw(c._h, None, None) == 0
        assert L.lmpc_rollout_commit_laps(c._h, nat.ptr(fin), nat.ptr(sl), nat.ptr(sl)) == 0
    finally:
        c.close()
    # refused calls in the middle of a run leave it as a run without them
    def run(refuse):
        c = _controller(B, widths=(0.4, 0.05))
        try:
            _seeded(c, np.arange(B), hook=lambda c: c.set_lane_margins([G(0), G(1, 0.02, 0.02)], np.arange(B) % 2))
            out = _laps(c, laps=1)
            if refuse:
                for bad in ([(3, 0.0, 0.0, 0.0, 0.0)], [(1, 0.05, 0.05, 0.0, 0.0)]):
                    assert _raw(c._h, bad, np.zeros(B)) == LMPC_E_INVALID
                rows, idx = nat.make_param_sets(c._p, [_par(0.02)], np.zeros(B, int), B, 48, 4)
                assert L.lmpc_set_param_sets(c._h, rows, 1, nat.ptr(idx)) == LMPC_E_INVALID
            out2 = _laps(c, laps=2)
            return out, out2, c.lane_margin_values()
        finally:
            c.close()
    a, b = run(False), run(True)
    for i in range(2):
        for key in KEYS:
            assert np.array_equal(a[i][key], b[i][key]), key
    assert np.array_equal(a[2], b[2])
