"""GPU tier: edge cases of the hot path against the oracle's restatement of the reference
(PredictiveModel.computeIndices PM.py:180-197, LMPC.selectPoints PC.py:478-514) and the error behaviour of the C ABI.

The reference has no tests of its own (SURVEY §4); these are the cases its code branches on:
few / one neighbour (exact distance ties inside one lap are implementation-defined in the reference: np.argsort's default
sort is not stable; the kernel takes the lowest rows), laps of assorted lengths, the two selection-window rules, the window
running off a lap (the reference: IndexError), a full lap pool, unsupported sizes and null arguments."""
import ctypes as C
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import BatchedFTOCP, _native as nat, reference_params as rp   # noqa: E402
from racinglmpc_b200.controller import BatchedController                             # noqa: E402
from oracle import ftocp, ltv_model                                                   # noqa: E402


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _abc_split(abc_b, N):
    return abc_b[:, 0:36].reshape(N, 6, 6), abc_b[:, 36:48].reshape(N, 6, 2), abc_b[:, 48:54]


def _model_controller(track, laps, xLin, uLin, N=12, trToUse=1):
    """B = 1 LTV-MPC controller whose regression model holds `laps`; linearisation points xLin[N+1,6], uLin[N,2]."""
    par = rp.mpc_params(N)
    c = BatchedController(par, 1, track.seg_table(), track.TrackLength, trToUse=trToUse, Tmax=1536, model_cap=trToUse + 1)
    for x, u in laps:
        c.model_add_trajectory(0, x, u)
    c.set_state(xLin=xLin[None], uLin=uLin[None], OldInput=np.zeros((1, 2)), timeStep=[0])
    return c


def _random_lap(rng, T):
    x = np.zeros((T, 6))
    x[:, 0] = 0.8 + 0.3 * rng.standard_normal(T)
    x[:, 1] = 0.05 * rng.standard_normal(T)
    x[:, 2] = 0.3 * rng.standard_normal(T)
    x[:, 3] = 0.05 * rng.standard_normal(T)
    x[:, 4] = np.linspace(0.0, 18.0, T)
    x[:, 5] = 0.05 * rng.standard_normal(T)
    u = np.stack([0.2 * rng.standard_normal(T), 0.5 * rng.standard_normal(T)], axis=1)
    return x, u


def _oracle_abc(track, laps, xLin, uLin, N, trToUse):
    m = ltv_model.LocalLTVModel(6, 2, track, trToUse)
    for x, u in laps:
        m.addTrajectory(x, u)
    out = [m.regressionAndLinearization(xLin[i], uLin[i]) for i in range(N)]
    return np.array([o[0] for o in out]), np.array([o[1] for o in out]), np.array([o[2] for o in out])


@pytest.mark.parametrize("T", [40, 256, 257, 258, 513, 1000])
def test_k1_lap_lengths_across_tile_boundaries(track, T):
    """Rows 0..T-2 are candidates (PM.py:183) on random laps; the tile-edge lengths of the scan (LMPC_K1_TILE) are the
    parametrisation of test_gpu_knn_regression.py."""
    _need_gpu()
    rng = np.random.default_rng(T)
    N = 12
    lap = _random_lap(rng, T)
    idx = rng.integers(0, T - 1, N + 1)
    xLin = lap[0][idx] + 0.01 * rng.standard_normal((N + 1, 6))
    uLin = lap[1][idx[:N]] + 0.01 * rng.standard_normal((N, 2))
    c = _model_controller(track, [lap], xLin, uLin)
    abc, flags = c.identify()
    c.close()
    assert flags[0] == 0
    A, B, Cc = _abc_split(abc[0], N)
    oA, oB, oC = _oracle_abc(track, [lap], xLin, uLin, N, 1)
    assert np.max(np.abs(A - oA)) < 1e-8 and np.max(np.abs(B - oB)) < 1e-8 and np.max(np.abs(Cc - oC)) < 1e-8


def test_k1_fewer_neighbours_than_maxnumpoint_and_the_raising_cases(track):
    """PM.py:187-191: with fewer than MaxNumPoint rows inside the bandwidth h all of them are used.  One neighbour makes the
    reference raise (np.squeeze) -> flag 4."""
    _need_gpu()
    rng = np.random.default_rng(11)
    N, T = 12, 300
    x, u = _random_lap(rng, T)
    x[:, 1] += 100.0                              # everything far away in vy (scaling 1, h = 5) ...
    near = [20, 90, 150, 151, 220, 260]           # ... except six rows
    x[near, 1] -= 100.0
    q = x[150].copy()
    xLin = np.tile(q, (N + 1, 1)); uLin = np.tile(u[150], (N, 1))
    c = _model_controller(track, [(x, u)], xLin, uLin)
    abc, flags = c.identify()
    c.close()
    assert flags[0] == 0
    A, B, Cc = _abc_split(abc[0], N)
    oA, oB, oC = _oracle_abc(track, [(x, u)], xLin, uLin, N, 1)
    assert np.max(np.abs(A - oA)) < 1e-7 and np.max(np.abs(B - oB)) < 1e-7 and np.max(np.abs(Cc - oC)) < 1e-7
    # one neighbour
    x1 = x.copy(); x1[[20, 90, 151, 220, 260], 1] += 100.0
    c = _model_controller(track, [(x1, u)], xLin, uLin)
    _, flags = c.identify()
    c.close()
    assert flags[0] & 4


def _lmpc_controller(track, laps, N=12, ss_cap=6):
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, 1, track.seg_table(), track.TrackLength, trToUse=1, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=1536, ss_cap=ss_cap, model_cap=2)
    for x, u in laps:
        c.add_trajectory(0, x, u)
    return c, numSS_it, numSS_Points


def _oracle_lmpc(track, laps, zt, N=12, numSS_it=None, numSS_Points=None):
    nit, M, _, _, Qts, par = ftocp.lmpc_params(track, N)
    nit, M = numSS_it or nit, numSS_Points or M
    par.timeVarying = False
    par.A, par.B = np.eye(6), np.zeros((6, 2))
    m = ltv_model.LocalLTVModel(6, 2, track, 1)
    o = ftocp.OracleLMPC(M, nit, Qts, par, m, qp=None)
    for x, u in laps:
        o.addTrajectory(x, u, x)
    o.zt = zt.copy()
    o.xLin = np.zeros((N + 1, 6))
    return o


# (numSS_it, numSS_Points) of the handle's grid with P = numSS_Points / numSS_it = 4, 6, 8, 12, 16, 24, 32, 48 and 96 points per lap
K2_SPLITS = [(6, 24), (8, 48), (3, 24), (4, 48), (2, 32), (4, 96), (3, 96), (1, 48), (1, 96)]


def _k2_handle(track, lap_sets, numSS_it, numSS_Points, N=12, shapes=None):
    """One controller per entry of `lap_sets` (its laps in the order driven) with the given safe-set split, or the handle's
    (N, numSS_Points) and per-controller `shapes` = (shapes, index)"""
    _, _, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, len(lap_sets), track.seg_table(), track.TrackLength, trToUse=1, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1536, ss_cap=max(len(laps) for laps in lap_sets), model_cap=2)
    if shapes is not None:
        c.set_shapes(*shapes)
    for b, laps in enumerate(lap_sets):
        for x, u in laps:
            c.add_trajectory(b, x, u)
    return c


def _k2_select(c, zt, x0, timeStep=None, has_pred=None, xPred=None):
    B, N = c.B, c.N
    c.set_state(xLin=np.zeros((B, N + 1, 6)), uLin=np.zeros((B, N, 2)), zt=zt, OldInput=np.zeros((B, 2)),
                timeStep=np.zeros(B, int) if timeStep is None else timeStep, has_pred=np.zeros(B, int) if has_pred is None else has_pred,
                xPred=xPred)
    return c.select(x0)


def _oracle_select(track, laps, zt, x0, numSS_it, numSS_Points, N=12, xPred=None, timeStep=0):
    """The oracle's selection (PC.py:386-416); raises IndexError where the reference does"""
    o = _oracle_lmpc(track, laps, np.asarray(zt, float), N, numSS_it, numSS_Points)
    if xPred is not None:
        o.xPred, o.timeStep = np.array(xPred, float), int(timeStep)
    with np.errstate(invalid="ignore", over="ignore"):        # inf - inf in the distances of (d)
        o.terminal_components(np.array(x0, float))
    return o


def _same_selection(sel, b, o, numSS_it, Mb=None, what=None):
    """Controller b's selection equals the oracle's bit for bit: the leading [6, Mb] / [2, Mb] / [Mb] block of its region (all of
    it without shapes), the argmin row and the lap of every selected lap"""
    Mb = sel["SS_sel"].shape[2] if Mb is None else Mb
    lead = lambda a, rows: a[b].reshape(-1)[:rows * Mb].reshape(rows, Mb)
    assert np.array_equal(lead(sel["SS_sel"], 6), o.SS_PointSelectedTot, equal_nan=True), what
    assert np.array_equal(sel["Qfun_sel"][b][:Mb], o.Qfun_SelectedTot, equal_nan=True), what
    assert np.array_equal(lead(sel["Succ_SS"], 6), o.Succ_SS_PointSelectedTot, equal_nan=True), what
    assert np.array_equal(lead(sel["Succ_uSS"], 2), o.Succ_uSS_PointSelectedTot, equal_nan=True), what
    assert [int(m) for m in sel["min_index"][b]] == [i_min for (_, i_min, _) in o.last_sel_index], what
    order = np.argsort(np.array(o.LapTime), kind="stable")[:numSS_it]
    assert list(order) == [lap for (lap, _, _) in o.last_sel_index], what


def _k2_lap(rng, T, L):
    x, u = _random_lap(rng, T)
    x[:, 4] = np.linspace(0.0, L + 1.5, T)                 # crosses the finish line: computeCost has something to count
    return x, u


def _k2_state(rng, L):
    return np.array([0.8 + 0.3 * rng.standard_normal(), 0.05 * rng.standard_normal(), 0.3 * rng.standard_normal(),
                     0.05 * rng.standard_normal(), rng.uniform(0.5, L - 0.5), 0.05 * rng.standard_normal()])


def _window_fits(mn, T, P):
    """PC.py:492-495 with numPoints = P + 1: [mn - P/2, mn + P/2] when mn - (P+1)/2 >= 0, else [mn, mn + P]; inside T rows?"""
    start = mn - P // 2 if mn - (P + 1) / 2 >= 0 else mn
    return start + P + 1 <= T


def _k2_rows(T, P):
    """Argmin rows of a T-row lap whose window fits -- 0, P/2 and P/2 + 1 (the two rules on either side of the switch) and the
    last row that fits -- and the first row after that whose window does not fit"""
    last = max(mn for mn in range(T) if _window_fits(mn, T, P))
    return [r for r in (0, P // 2, P // 2 + 1, last) if _window_fits(r, T, P)], last + 1


def _plant(x, row, z):
    """z at `row` and again 31 and 32 rows later (another lane, lower for most rows, and the same lane of the 32-row scan): the
    first copy is np.argmin's"""
    for r in (row, row + 31, row + 32):
        if r < x.shape[0]:
            x[r] = z


def test_k2_window_rules_and_first_minimum(track):
    """PC.py:486-495 at every P the handle accepts (K2_SPLITS): the window is [Min - P/2, Min + P/2] when Min - (P+1)/2 >= 0,
    else [Min, Min + P]; np.argmin returns the FIRST minimum (copies of the nearest row 31 and 32 rows later).  Laps of P + 1 rows
    and of one below, at and one above multiples of 32 rows; the argmin at 0, P/2, P/2 + 1 and the last row whose window fits,
    and at the first row whose window does not (the reference: IndexError; the kernel: flag 8)."""
    _need_gpu()
    for numSS_it, numSS_Points in K2_SPLITS:
        _k2_windows_at(track, numSS_it, numSS_Points)


def _k2_windows_at(track, numSS_it, numSS_Points):
    """test_k2_window_rules_and_first_minimum at one (numSS_it, numSS_Points): one controller per lap length and argmin row"""
    split = (numSS_it, numSS_Points)
    P = numSS_Points // numSS_it
    L = track.TrackLength
    k0 = (P + 2) // 32 + 1
    lengths = [P + 1] + [32 * m + d for m in range(k0, k0 + 3) for d in (-1, 0, 1)]
    rng = np.random.default_rng(P)
    cases, lap_sets, zts = [], [], []
    for li in range(len(lengths)):
        for kind in range(5):                              # 0..3: the fitting rows in turn; 4: lap 0 at its first row past the end
            zt = _k2_state(rng, L)
            laps = []
            for j in range(numSS_it):                      # driven in this order, selected in the order of their lengths
                T = lengths[(li + j) % len(lengths)]
                fit, past = _k2_rows(T, P)
                x, u = _k2_lap(rng, T, L)
                _plant(x, past if (kind == 4 and j == 0) else fit[(kind + j) % len(fit)], zt)
                laps.append((x, u))
            cases.append(kind == 4); lap_sets.append(laps); zts.append(zt)
    zt = np.array(zts)
    x0 = np.zeros_like(zt); x0[:, 0] = 0.8; x0[:, 4] = zt[:, 4]
    c = _k2_handle(track, lap_sets, numSS_it, numSS_Points)
    try:
        sel = _k2_select(c, zt, x0)
    finally:
        c.close()
    for b, raises in enumerate(cases):
        if raises:
            assert sel["flags"][b] & 8, (split, b)
            with pytest.raises(IndexError):
                _oracle_select(track, lap_sets[b], zt[b], x0[b], numSS_it, numSS_Points)
        else:
            assert sel["flags"][b] == 0, (split, b)
            _same_selection(sel, b, _oracle_select(track, lap_sets[b], zt[b], x0[b], numSS_it, numSS_Points), numSS_it,
                            what=(split, b))


def _q_laps(rng, L, lengths):
    return [_k2_lap(rng, T, L) for T in lengths]


def test_k2_q_function_shift_and_lap_wrap(track):
    """PC.py:392-393 and 501-512: with a previous prediction that has stages past the finish line (> L; a stage exactly at L does
    not count), an older lap's Qfun is raised by its Qfun[0] and the latest lap's (it-1) by timeStep + N - (stages past); 0, 1 and
    all N + 1 stages past; a stage exactly at L; no prediction yet.  The terminal guess wraps when zt[4] - x0[4] > L/2 (not at
    exactly L/2) and is clamped to 0 when zt[4] - L < 0."""
    _need_gpu()
    numSS_it, numSS_Points, N = 4, 48, 12
    P = numSS_Points // numSS_it
    L = track.TrackLength
    rng = np.random.default_rng(21)
    lengths = [140, 150, 160, 175, 130]                    # the latest lap is the fastest: selected with three older laps
    base = np.linspace(L - 3.0, L - 0.5, N + 1)
    past_specs = {"none": base, "last": np.r_[base[:N], L + 0.25], "all": np.linspace(L + 0.1, L + 3.0, N + 1),
                  "at L, then past": np.r_[base[:N - 1], L, L + 0.25], "last at L": np.r_[base[:N], L]}
    half_x0 = 0.5
    assert (half_x0 + L / 2) - half_x0 == L / 2
    wraps = {"no wrap": (L - 1.0, L - 1.3), "exactly L/2": (half_x0 + L / 2, half_x0), "wrap": (L + 0.7, 0.3),
             "clamped to 0": (0.6 * L, 0.05)}
    cases, lap_sets, zts, x0s, xPreds, ts, hp = [], [], [], [], [], [], []
    for k, (pname, s_pred) in enumerate(list(past_specs.items()) + [("no prediction", past_specs["all"])]):
        for wname, (zt4, x04) in wraps.items():
            zt = _k2_state(rng, L); zt[4] = zt4
            x0 = np.array([0.8, 0, 0, 0, x04, 0.0])
            zeff = zt.copy()
            if zt[4] - x0[4] > L / 2:
                zeff[4] = max(zt[4] - L, 0.0)
            laps = _q_laps(rng, L, lengths)
            for j, (x, _) in enumerate(laps):
                _plant(x, [P // 2 + 1, 0, 40, 100, 20][j], zeff)
            xp = 0.1 * rng.standard_normal((N + 1, 6)); xp[:, 4] = s_pred
            cases.append((pname, wname)); lap_sets.append(laps); zts.append(zt); x0s.append(x0); xPreds.append(xp)
            ts.append([0, 9, 250][len(ts) % 3]); hp.append(0 if pname == "no prediction" else 1)
    c = _k2_handle(track, lap_sets, numSS_it, numSS_Points, N=N)
    try:
        sel = _k2_select(c, np.array(zts), np.array(x0s), timeStep=ts, has_pred=hp, xPred=np.array(xPreds))
    finally:
        c.close()
    for b, case in enumerate(cases):
        assert sel["flags"][b] == 0, case
        o = _oracle_select(track, lap_sets[b], zts[b], x0s[b], numSS_it, numSS_Points, N=N, xPred=xPreds[b] if hp[b] else None,
                           timeStep=ts[b])
        _same_selection(sel, b, o, numSS_it, what=case)
        raw = np.concatenate([o.Qfun[lap][first:first + P] for (lap, _, first) in o.last_sel_index])
        shifted = case[0] in ("last", "all", "at L, then past")
        assert np.array_equal(o.Qfun_SelectedTot, raw) != shifted, case          # the case exercises what it names


def test_k2_shaped_batch_equals_the_oracle_at_each_shape(track):
    """lmpc_set_shapes: a controller of shape (N_b, M_b) selects what the oracle selects at (N_b, M_b) -- its [6, M_b] block
    at the start of its region, P_b = M_b / numSS_it points per lap, and only its N_b + 1 prediction stages counted for the
    Q-function shift (the stale stages beyond N_b are all past the finish line)."""
    _need_gpu()
    numSS_it, HN, HM = 4, 14, 96
    shapes = [(12, 24), (12, 32), (6, 48), (10, 48), (14, 64), (14, 96)]
    B = 2 * len(shapes)
    idx = np.arange(B) % len(shapes)
    L = track.TrackLength
    rng = np.random.default_rng(33)
    lengths = [140, 150, 160, 175, 130]
    lap_sets, zts, xPreds = [], [], []
    for b in range(B):
        Nb, Mb = shapes[idx[b]]
        P = Mb // numSS_it
        zt = _k2_state(rng, L)
        laps = _q_laps(rng, L, lengths)
        for j, (x, _) in enumerate(laps):
            fit, _ = _k2_rows(x.shape[0], P)
            _plant(x, fit[(b + j) % len(fit)], zt)
        xp = 0.1 * rng.standard_normal((HN + 1, 6))
        xp[:, 4] = L + 5.0                                  # stale stages beyond N_b: past the line
        xp[:Nb + 1, 4] = np.linspace(L - 2.0, L - 0.2, Nb + 1)
        if b < len(shapes):
            xp[Nb - 1:Nb + 1, 4] = L + 0.3                  # two of the N_b + 1 stages past the line
        lap_sets.append(laps); zts.append(zt); xPreds.append(xp)
    zt = np.array(zts)
    x0 = np.zeros_like(zt); x0[:, 0] = 0.8; x0[:, 4] = zt[:, 4]
    ts = 3 * np.arange(B)
    c = _k2_handle(track, lap_sets, numSS_it, HM, N=HN, shapes=(shapes, idx))
    try:
        sel = _k2_select(c, zt, x0, timeStep=ts, has_pred=np.ones(B, int), xPred=np.array(xPreds))
    finally:
        c.close()
    for b in range(B):
        Nb, Mb = shapes[idx[b]]
        assert sel["flags"][b] == 0, b
        o = _oracle_select(track, lap_sets[b], zt[b], x0[b], numSS_it, Mb, N=Nb, xPred=xPreds[b][:Nb + 1], timeStep=ts[b])
        _same_selection(sel, b, o, numSS_it, Mb=Mb, what=(b, Nb, Mb))


def test_k2_non_finite_and_huge_inputs_follow_np_argmin(track):
    """np.argmin on any distance vector: the first NaN row if there is one (a NaN in zt, NaN rows in a lap, inf - inf), else the
    first minimum with +inf an ordinary value (a +-inf or 1e301 zt, a lap of inf rows: row 0).  The selection equals the oracle
    where it returns and is flag 8 where it raises; no value of zt, x0 or a lap makes the kernel read outside the lap."""
    _need_gpu()
    numSS_it, numSS_Points = 4, 48
    L = track.TrackLength
    rng = np.random.default_rng(44)
    nan, inf = np.nan, np.inf
    ROWS = [20, 7, 33, 60]                                  # where the finite zt sits in the four laps (driven shortest first)

    def zt_set(j, v):
        return lambda zt, x0, laps: zt.__setitem__(j, v)

    def nan_rows(zt, x0, laps):
        laps[1][0][17, 3] = nan
        laps[1][0][50] = nan

    def inf_lap(zt, x0, laps):
        laps[2][0][:] = inf

    def inf_meets_inf(zt, x0, laps):
        zt[0] = inf
        laps[3][0][25, 0] = inf

    def neg_inf_row(zt, x0, laps):
        laps[1][0][3, 5] = -inf

    def nan_row_past_the_end(zt, x0, laps):
        laps[0][0][97] = nan

    cases = [("nan zt[%d]" % j, zt_set(j, nan), False) for j in range(6)]
    cases += [("+inf zt[0]", zt_set(0, inf), False), ("-inf zt[4]", zt_set(4, -inf), False), ("+inf zt[4]", zt_set(4, inf), False),
              ("-inf zt[2]", zt_set(2, -inf), False), ("1e301 zt[2]", zt_set(2, 1e301), False), ("1e301 zt[4]", zt_set(4, 1e301), False),
              ("nan x0", lambda zt, x0, laps: x0.__setitem__(slice(None), nan), False), ("lap of inf rows", inf_lap, False),
              ("nan rows in a lap", nan_rows, False), ("inf zt meets an inf row", inf_meets_inf, False),
              ("-inf in a row", neg_inf_row, False), ("nan row past the window", nan_row_past_the_end, True)]
    lap_sets, zts, x0s = [], [], []
    for name, mod, _ in cases:
        zt = _k2_state(rng, L)
        x0 = np.array([0.8, 0, 0, 0, zt[4], 0.0])
        laps = _q_laps(rng, L, [100, 110, 120, 130])
        for j, (x, _) in enumerate(laps):
            _plant(x, ROWS[j], zt)
        mod(zt, x0, laps)
        lap_sets.append(laps); zts.append(zt); x0s.append(x0)
    c = _k2_handle(track, lap_sets, numSS_it, numSS_Points)
    try:
        sel = _k2_select(c, np.array(zts), np.array(x0s))
    finally:
        c.close()
    for b, (name, _, raises) in enumerate(cases):
        if raises:
            assert sel["flags"][b] & 8, name
            with pytest.raises(IndexError):
                _oracle_select(track, lap_sets[b], zts[b], x0s[b], numSS_it, numSS_Points)
            continue
        assert sel["flags"][b] == 0, name
        o = _oracle_select(track, lap_sets[b], zts[b], x0s[b], numSS_it, numSS_Points)
        _same_selection(sel, b, o, numSS_it, what=name)
    # the argmin rows these cases are about
    mins = {name: [int(m) for m in sel["min_index"][b]] for b, (name, _, _) in enumerate(cases)}
    for j in range(6):
        assert mins["nan zt[%d]" % j] == [0, 0, 0, 0]
    assert mins["1e301 zt[4]"] == [0, 0, 0, 0] and mins["+inf zt[0]"] == [0, 0, 0, 0]
    assert mins["nan x0"] == ROWS and mins["-inf in a row"] == ROWS
    assert mins["lap of inf rows"] == [20, 7, 0, 60]
    assert mins["nan rows in a lap"] == [20, 17, 33, 60]
    assert mins["inf zt meets an inf row"] == [0, 0, 0, 25]


def test_k2_window_past_the_lap_end_is_flagged(track):
    """The reference indexes past the array (IndexError, PC.py:497) when the nearest point is within 6 rows of a lap's end
    and addPoint has not grown it; the kernel reports bit 8 and leaves the selection of that lap untouched."""
    _need_gpu()
    rng = np.random.default_rng(4)
    laps = [_random_lap(rng, 100) for _ in range(4)]
    zt = laps[1][0][97].copy()
    c, _, _ = _lmpc_controller(track, laps)
    c.set_state(xLin=np.zeros((1, 13, 6)), uLin=np.zeros((1, 12, 2)), zt=zt[None], OldInput=np.zeros((1, 2)), timeStep=[0], has_pred=[0])
    sel = c.select(np.array([[0.8, 0, 0, 0, zt[4], 0.0]]))
    c.close()
    assert sel["flags"][0] & 8
    with pytest.raises(IndexError):
        o = _oracle_lmpc(track, laps, zt)
        o.terminal_components(np.array([0.8, 0, 0, 0, zt[4], 0.0]))


def test_add_point_on_a_full_lap_is_flagged(track):
    _need_gpu()
    rng = np.random.default_rng(6)
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(12)
    c = BatchedController(par, 1, track.seg_table(), track.TrackLength, trToUse=1, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=64, ss_cap=5, model_cap=2)
    for _ in range(4):
        c.add_trajectory(0, *_random_lap(rng, 63))
    c.add_point(np.zeros(6), np.zeros(2))              # row 64 of 64: fits
    assert c.get_lap(0, 3)[0].shape[0] == 64
    # no room: LMPC.addPoint would np.append (PC.py:466-476); the fixed pool must not drop the point silently: the host
    # entry reports it (the device-resident rollout accumulates flag bit 16 in its health record instead)
    with pytest.raises(nat.NativeError, match="Tmax"):
        c.add_point(np.zeros(6), np.zeros(2))
    assert c.get_lap(0, 3)[0].shape[0] == 64
    assert c.step_results()["flags"][0] & 16
    c.close()


def test_add_point_refuses_non_finite_values(track):
    """A state or input with a NaN or an inf is not appended (PC.py:466-476 would store it): the host entry refuses it with
    LMPC_E_INVALID and leaves every lap as it was; a finite point still appends."""
    _need_gpu()
    rng = np.random.default_rng(7)
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(12)
    c = BatchedController(par, 2, track.seg_table(), track.TrackLength, trToUse=1, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=256, ss_cap=5, model_cap=2)
    try:
        for b in range(2):
            for _ in range(4):
                c.add_trajectory(b, *_random_lap(rng, 100))
        before = [c.get_lap(b, 3) for b in range(2)]
        for j, v in ((0, np.nan), (4, np.inf), (5, -np.inf), (6, np.nan), (7, np.inf)):
            x, u = np.full((2, 6), 0.5), np.zeros((2, 2))
            (x if j < 6 else u)[1, j % 6] = v
            with pytest.raises(nat.NativeError, match="non-finite"):
                c.add_point(x, u)
            for b in range(2):
                assert all(np.array_equal(a, e) for a, e in zip(c.get_lap(b, 3), before[b])), (j, b)
        c.add_point(np.full((2, 6), 0.5), np.zeros((2, 2)))
        assert all(c.get_lap(b, 3)[0].shape[0] == 101 for b in range(2))
    finally:
        c.close()


def test_c_abi_rejects_bad_arguments_without_raising_through_the_boundary():
    _need_gpu()
    L = nat.lib()
    par = rp.mpc_params(12)
    p = nat.make_params(par, 0, 0, None, 0.0, 0.0, 0)
    h = C.c_void_p()
    assert L.lmpc_create(C.byref(p), 0, 0, C.byref(h)) != 0                     # empty batch
    assert b"batch" in L.lmpc_last_error() or L.lmpc_last_error()
    p_bad = nat.make_params(rp.mpc_params(13), 0, 0, None, 0.0, 0.0, 0)          # horizon without an instantiation
    rc = L.lmpc_create(C.byref(p_bad), 4, 0, C.byref(h))
    if rc == 0:                                                                   # accepted at create: must fail at solve
        x0 = np.zeros((4, 6)); u0 = np.zeros((4, 2)); abc = np.zeros((4, 13, 54))
        out = [np.zeros((4, 14, 6)), np.zeros((4, 13, 2)), np.zeros((4, 26)), np.zeros(4, np.int32), np.zeros(4, np.int32), np.zeros((4, 3))]
        assert L.lmpc_solve_mpc_host(h, nat.ptr(x0), nat.ptr(u0), nat.ptr(abc), 13 * 54, 54, *[nat.ptr(a) for a in out]) != 0
        L.lmpc_destroy(h)
    assert L.lmpc_create(C.byref(p), 4, 0, C.byref(h)) == 0
    x0 = np.zeros((4, 6)); u0 = np.zeros((4, 2)); abc = np.zeros((4, 12, 54))
    out = [np.zeros((4, 13, 6)), np.zeros((4, 12, 2)), np.zeros((4, 24)), np.zeros(4, np.int32), np.zeros(4, np.int32), np.zeros((4, 3))]
    assert L.lmpc_solve_mpc_host(h, None, nat.ptr(u0), nat.ptr(abc), 12 * 54, 54, *[nat.ptr(a) for a in out]) != 0      # null x0
    assert L.lmpc_solve_mpc_host(h, nat.ptr(x0), nat.ptr(u0), nat.ptr(abc), 7, 54, *[nat.ptr(a) for a in out]) != 0      # bad strides
    assert L.lmpc_step_host(h, 0, nat.ptr(x0), *([None] * 10)) != 0                                                        # no lap store yet
    assert L.lmpc_ss_add_point(h, nat.ptr(x0), nat.ptr(u0)) != 0
    assert L.lmpc_rollout_step(h, 0, None, 0) != 0
    # an all-zero model is a legal (if useless) QP: the call itself must succeed and report per-instance status
    assert L.lmpc_solve_mpc_host(h, nat.ptr(x0), nat.ptr(u0), nat.ptr(abc), 12 * 54, 54, *[nat.ptr(a) for a in out]) == 0
    L.lmpc_destroy(h)


def test_lmpc_qp_with_short_horizon_matches_oracle(gold, track):
    """LMPC-type QP at N = 6 (BASELINE configs[4] lists LMPC at N in {6, 12}): the first six stages of a golden LMPC step."""
    _need_gpu()
    from oracle import osqp_port
    from racinglmpc_b200.batched import pack_abc
    N = 6
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    _, _, _, _, oQts, opar = ftocp.lmpc_params(track, N)
    opar.timeVarying = True
    keys = [(4, 60), (5, 90), (6, 40)]
    B = len(keys)
    x0 = np.stack([gold["lmpc_%d_%d_x0" % k] for k in keys])
    uold = np.stack([gold["lmpc_%d_%d_OldInput" % k].ravel() for k in keys])
    A = [gold["lmpc_%d_%d_A" % k][:N] for k in keys]; Bm = [gold["lmpc_%d_%d_B" % k][:N] for k in keys]
    Cm = [gold["lmpc_%d_%d_C" % k][:N] for k in keys]
    abc = np.stack([pack_abc(a, b, c) for a, b, c in zip(A, Bm, Cm)])
    SS = np.stack([gold["lmpc_%d_%d_SS_sel" % k] for k in keys]); Qf = np.stack([gold["lmpc_%d_%d_Qfun_sel" % k] for k in keys])
    s = BatchedFTOCP(par, batch=B, numSS_Points=numSS_Points, numSS_it=numSS_it, QterminalSlack=Qts)
    o = s.solve(x0, uold, abc, SS, Qf)
    s.close()
    assert np.all(o["status"] == 1), (o["status"], o["iters"])
    for b in range(B):
        opar.A, opar.B = list(A[b]), list(Bm[b])
        F, bb = ftocp.build_ineq(opar)
        G, E, Lv = ftocp.build_eq(opar, list(A[b]), list(Bm[b]), list(Cm[b]))
        H, q = ftocp.build_cost(opar, uold[b][None, :])
        F2, b2, G2, E2, L2, H2, q2 = ftocp.add_safe_set(F, bb, G, E, Lv, H, q, 6, N, SS[b], Qf[b], oQts)
        P, qq, Am, l, u = ftocp.osqp_form(H2, q2, F2, b2, G2, E2 @ x0[b] + L2)
        z, info = osqp_port.tight_qp(P, qq, Am, l, u)
        assert info["status"] == 1
        assert np.max(np.abs(o["xPred"][b].ravel() - z[:6 * (N + 1)])) < 1e-6
        assert np.max(np.abs(o["uPred"][b].ravel() - z[6 * (N + 1):6 * (N + 1) + 2 * N])) < 1e-6
