"""GPU tier: per-controller regression models (lmpc_set_regression_sets).

Host-driven K1: the knn_fixtures groups that share N and dt, interleaved in one handle (the largest trToUse, Tmax and model_cap of
them) with one regression set per group, give the flags and models of one handle per group bit for bit and meet the exact
reference; the same groups with scaling and bandwidth moved to both ends of the admitted range give the same models bit for bit.
Device-resident closed loop: four interleaved sets (h, MaxNumPoint, lamb and trToUse each changed) equal one handle per set created
with those constants, traced or not, and a crossed design of 2 regression sets x 2 QP tunings equals one handle per cell.  The
reference constants as one set equal no sets, nsets == 0 reverts, refusals change nothing, and a run captured at one lap and
resumed to two equals a straight run."""
import contextlib
import copy
import ctypes as C
import dataclasses
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import closed_loop as cl                                           # noqa: E402
import knn_fixtures as kf                                          # noqa: E402
import regression_sets as rs                                       # noqa: E402
from closed_loop import N, KEYS                                    # noqa: E402
from racinglmpc_b200 import reference_params as rp                # noqa: E402
from racinglmpc_b200 import _native as nat                        # noqa: E402
from racinglmpc_b200.controller import BatchedController          # noqa: E402
from racinglmpc_b200.reference_params import RegressionParams, TrackParams   # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LMPC_E_INVALID, LMPC_E_STATE = -1, -4
B = 256
REF = RegressionParams.reference(4)
# the four sets of the closed-loop tests: one field changed each
FOUR = [dataclasses.replace(REF, h=2.0), dataclasses.replace(REF, MaxNumPoint=4), dataclasses.replace(REF, lamb=1e-3),
        dataclasses.replace(REF, trToUse=2)]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


# ------------------------------------------------------------------------------------------------------------ host-driven K1
def _shared_groups():
    return [g for g in kf.groups() if g.N == 12 and g.consts["dt"] == 0.1]


def _identify(groups, sets=True):
    """One handle for every fixture of `groups`, interleaved (fixture j of every group in turn); with `sets`, one regression set per
    group.  Returns (abc, flags, [(group index, fixture)] per instance)."""
    inst = []
    for j in range(max(len(g.fixtures) for g in groups)):
        inst += [(gi, g.fixtures[j]) for gi, g in enumerate(groups) if j < len(g.fixtures)]
    Bh = len(inst)
    c = BatchedController(rp.mpc_params(12), Bh, kf.TRACK.seg_table(), kf.TRACK.TrackLength,
                          trToUse=max(g.trToUse for g in groups), Tmax=max(g.Tmax for g in groups),
                          model_cap=max(g.model_cap for g in groups), model_kwargs=dict(dt=0.1))
    try:
        if sets:
            c.set_regression([rs.set_of(g) for g in groups], np.array([gi for gi, _ in inst]))
        for b, (_, fx) in enumerate(inst):
            for x, u in fx.laps:
                c.model_add_trajectory(b, x, u)
        c.set_state(xLin=np.stack([fx.xLin for _, fx in inst]), uLin=np.stack([fx.uLin for _, fx in inst]),
                    OldInput=np.zeros((Bh, 2)), timeStep=np.zeros(Bh))
        abc, flags = c.identify()
    finally:
        c.close()
    return abc, flags, inst


def _one_handle(g):
    Bg = len(g.fixtures)
    c = BatchedController(rp.mpc_params(g.N), Bg, kf.TRACK.seg_table(), kf.TRACK.TrackLength, trToUse=g.trToUse, Tmax=g.Tmax,
                          model_cap=g.model_cap, model_kwargs=g.consts)
    try:
        for b, fx in enumerate(g.fixtures):
            for x, u in fx.laps:
                c.model_add_trajectory(b, x, u)
        c.set_state(xLin=np.stack([fx.xLin for fx in g.fixtures]), uLin=np.stack([fx.uLin for fx in g.fixtures]),
                    OldInput=np.zeros((Bg, 2)), timeStep=np.zeros(Bg))
        return c.identify()
    finally:
        c.close()


def test_interleaved_groups_equal_one_handle_per_group_and_the_exact_reference():
    _need_gpu()
    groups = _shared_groups()
    assert {"default_N12", "laps_trToUse1", "laps_trToUse4", "laps_trToUse8", "k1_h50_ridge", "k3_h0.5",
            "negative_scaling"} <= {g.name for g in groups}
    abc, flags, inst = _identify(groups)
    own = [_one_handle(g) for g in groups]
    pos = [0] * len(groups)
    for b, (gi, fx) in enumerate(inst):
        oabc, oflags = own[gi]
        j = pos[gi]
        pos[gi] += 1
        assert int(flags[b]) == int(oflags[j]) == fx.flags, (groups[gi].name, fx.name)
        assert np.array_equal(abc[b], oabc[j]), (groups[gi].name, fx.name)
        if fx.flags:
            continue
        m = kf.exact_model(fx, groups[gi])
        for i in range(groups[gi].N):
            A, Bm, Cc = m.model(fx.xLin[i], fx.uLin[i])
            tol, _ = kf.tolerance(m.systems)
            gA, gB, gC = kf.abc_split(abc[b, i])
            assert float(np.max(np.abs(kf.rows012(gA, gB, gC) - kf.rows012(A, Bm, Cc)))) <= tol, (fx.name, i)
            assert float(np.max(np.abs(kf.rows345(gA, gB, gC) - kf.rows345(A, Bm, Cc)))) <= 1e-14, (fx.name, i)


def test_scaling_at_both_ends_of_the_range_gives_the_same_models():
    """scaling and h times 2^-28 and 2^32: every distance scales exactly, so flags and models equal the unscaled sets bit for bit."""
    _need_gpu()
    base = [g for g in _shared_groups() if g.name in ("default_N12", "k1_h50_ridge", "k3_h0.5", "negative_scaling")]
    abc0, flags0, _ = _identify(base)
    for k in (rs.LOW, rs.HIGH):
        abc, flags, _ = _identify([rs.scaled(g, k) for g in base])
        assert np.array_equal(flags, flags0), k
        assert np.array_equal(abc, abc0), k


# ------------------------------------------------------------------------------------------------------ device closed loop
def _store_controller(reg):
    """closed_loop.controller, with the store created with `reg`'s constants instead of installing a set."""
    def make(Bc, track=None, par=None, qts=None, **_):
        numSS_it, numSS_Points, _, _, Qts, base = rp.lmpc_params(N)
        track = TrackParams.l_shaped() if track is None else track
        return BatchedController(base if par is None else par, Bc, track.seg_table, track.TrackLength, trToUse=reg.trToUse,
                                 numSS_Points=numSS_Points, numSS_it=numSS_it, QterminalSlack=Qts if qts is None else qts,
                                 Tmax=1280, ss_cap=7, model_cap=5,
                                 model_kwargs=dict(MaxNumPoint=reg.MaxNumPoint, h=reg.h, lamb=reg.lamb, scaling=reg.scaling))
    return make


@contextlib.contextmanager
def _store_with(reg):
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(cl, "controller", _store_controller(reg))
        yield


# a store created with a smaller trToUse keeps fewer model laps: its model-pool books differ, what it regresses on does not
MODEL_BOOKS = ("md_time", "md_seq")


def _same(a, b, sel, what, model_books=True):
    keys = KEYS if model_books else tuple(k for k in KEYS if k not in MODEL_BOOKS)
    (ar, al), (br, bl) = a, b
    for key in keys:
        assert np.array_equal(ar[key][sel], br[key][sel]), (what, key)
    for (i, slot), v in al.items():
        if sel[i] and (i, slot) in bl:
            assert all(np.array_equal(p, q) for p, q in zip(v, bl[(i, slot)])), (what, i, slot)


def _reject(c):
    """Refused calls, each returning LMPC_E_INVALID; the handle must stay as it was."""
    L = nat.lib()
    idx = np.arange(B, dtype=np.int32) % 4
    good, _ = nat.make_regression_sets(FOUR, idx, B, trToUse=4)

    def copy_of(mod):
        t = (nat.RegressionParams * 4)()
        C.memmove(t, good, C.sizeof(t))
        mod(t)
        return t
    bad = [copy_of(lambda t: setattr(t[1], "trToUse", 5)), copy_of(lambda t: setattr(t[2], "trToUse", 0)),
           copy_of(lambda t: setattr(t[0], "MaxNumPoint", 8)), copy_of(lambda t: setattr(t[3], "h", 0.0)),
           copy_of(lambda t: setattr(t[3], "h", float("nan"))), copy_of(lambda t: setattr(t[1], "lamb", -1.0)),
           copy_of(lambda t: t[2].scaling.__setitem__(0, 2.0 ** 33)), copy_of(lambda t: t[2].scaling.__setitem__(4, 1e-12)),
           copy_of(lambda t: t[0].scaling.__setitem__(1, float("inf")))]
    cases = [(t, 4, idx) for t in bad] + [(good, 4, np.full(B, 4, np.int32)), (good, 4, np.full(B, -1, np.int32)), (good, 0, idx),
                                          (None, 4, idx), (good, 4, None)]
    for tab, n, ix in cases:
        assert L.lmpc_set_regression_sets(c._h, tab, n, nat.ptr(ix) if ix is not None else None) == LMPC_E_INVALID
    big = (nat.RegressionParams * (B + 1))(*([good[0]] * (B + 1)))
    assert L.lmpc_set_regression_sets(c._h, big, B + 1, nat.ptr(np.zeros(B, np.int32))) == LMPC_E_INVALID


@pytest.fixture(scope="module")
def runs():
    """A batch of FOUR (set b % 4) with refused calls before the run, one handle per set created with its constants, no sets."""
    _need_gpu()
    ridx = np.arange(B) % 4

    def install(c):
        c.set_regression(FOUR, ridx)
        _reject(c)

    n, het, het_laps = cl.run(B, hook=install)
    # MaxNumPoint = 4 is slower to learn: most of its controllers have not finished an LMPC lap in the run's 1200 steps, the
    # others all have; the comparison covers the whole run either way
    assert het["lap_n"][ridx != 1].min() >= 1, "not every controller of sets 0, 2, 3 finished an LMPC lap in %d steps" % n
    refs = []
    for reg in FOUR:
        with _store_with(reg):
            refs.append(cl.run(B, steps=n)[1:])
    none = cl.run(B, steps=n)[1:]
    return dict(n=n, ridx=ridx, het=(het, het_laps), refs=refs, none=none)


def test_batch_of_regression_sets_equals_one_handle_per_set(runs):
    for k in range(4):
        _same(runs["het"], runs["refs"][k], runs["ridx"] == k, "regression set %d" % k, model_books=FOUR[k].trToUse == 4)
    h = runs["het"][0]
    assert len({float(h["lap_hist"][runs["ridx"] == k, 0].mean()) for k in range(4)} | {float(runs["none"][0]["lap_hist"][:, 0].mean())}) > 1


def test_traced_batch_gives_the_same_results(runs):
    _, het, laps = cl.run(B, hook=lambda c: c.set_regression(FOUR, runs["ridx"]), steps=runs["n"], trace=True)
    for k in range(4):
        _same((het, laps), runs["refs"][k], runs["ridx"] == k, "traced, regression set %d" % k, model_books=FOUR[k].trToUse == 4)


def test_reference_as_one_set_equals_no_sets_and_reverts(runs):
    n, every = runs["n"], np.ones(B, bool)
    one = cl.run(B, hook=lambda c: c.set_regression([REF], np.zeros(B, np.int32)), steps=n)[1:]
    _same(one, runs["none"], every, "reference as one set vs no sets")

    def install_then_revert(c):
        c.set_regression(FOUR, runs["ridx"])
        with pytest.raises(ValueError):
            c.set_regression(None, runs["ridx"])          # reverting takes no index
        with pytest.raises(ValueError):
            c.set_regression(FOUR)                        # sets need one
        with pytest.raises(ValueError):
            c.set_regression([dataclasses.replace(REF, trToUse=5)], np.zeros(B, np.int32))
        c.set_regression(None)

    _same(cl.run(B, hook=install_then_revert, steps=n)[1:], runs["none"], every, "nsets == 0 reverts")


def test_without_a_store_the_call_is_a_state_error():
    _need_gpu()
    L = nat.lib()
    p = nat.make_params(rp.mpc_params(12))
    h = C.c_void_p()
    nat.check(L.lmpc_create(C.byref(p), 4, 0, C.byref(h)))
    try:
        t, idx = nat.make_regression_sets([RegressionParams.reference(1)], np.zeros(4), 4, trToUse=1)
        assert L.lmpc_set_regression_sets(h, t, 1, nat.ptr(idx)) == LMPC_E_STATE
    finally:
        L.lmpc_destroy(h)


def test_crossed_regression_sets_and_tunings_equal_one_handle_per_cell():
    """2 regression sets x 2 QP tunings: controller b runs tuning b % 2 with regression set (b // 2) % 2."""
    _need_gpu()
    _, _, _, _, Qts, base = rp.lmpc_params(N)
    ps = []
    for k in range(2):
        p = copy.deepcopy(base)
        p.dR = (0.5, 2.0)[k] * np.asarray(base.dR, float)
        ps.append(p)
    regs = [FOUR[0], FOUR[3]]
    b = np.arange(B)
    pidx, ridx = b % 2, (b // 2) % 2
    n, het, het_laps = cl.run(B, psets=(ps, pidx, [Qts, Qts]), hook=lambda c: c.set_regression(regs, ridx))
    for i in range(2):
        for j in range(2):
            with _store_with(regs[j]):
                ref = cl.run(B, par=ps[i], qts=Qts, steps=n)[1:]
            _same((het, het_laps), ref, (pidx == i) & (ridx == j), "tuning %d, regression set %d" % (i, j),
                  model_books=regs[j].trToUse == 4)


def _rollout_mc():
    sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
    try:
        import rollout_mc
    finally:
        sys.path.pop(0)
    return rollout_mc


def test_capture_and_resume_with_regression_sets():
    """rollout_mc.run with regression sets installed: 1 lap captured and resumed to 2 equals a straight run to 2 laps."""
    _need_gpu()
    rm = _rollout_mc()
    Bs = 256
    kw = dict(batch=Bs, local=0, regression_sets=([FOUR[0], FOUR[2], FOUR[3], REF], np.arange(Bs) % 4))
    fin2, bk2, cap2 = {}, {}, {}
    o2 = rm.run(laps=2, final=fin2, books=bk2, capture=cap2, **kw)
    cap = {}
    rm.run(laps=1, capture=cap, **kw)
    assert cap["diverged_step"] is None
    fin, bk, capr = {}, {}, {}
    o = rm.run(laps=2, start=cap, final=fin, books=bk, capture=capr, **kw)
    assert o["resume_exact"] and o["closed_loop_steps"] == o2["closed_loop_steps"]
    assert capr["exchange_steps"] == cap2["exchange_steps"]
    assert torch.equal(capr["records"], cap2["records"])
    for k in bk2:
        assert np.array_equal(np.asarray(bk2[k]), np.asarray(bk[k])), ("books", k)
    for k in fin2:
        assert np.array_equal(np.asarray(fin2[k]), np.asarray(fin[k])), ("end state", k)
    for k in ("lap_stats_rank0", "per_regression_rank0", "instances_with_flags_rank0", "unsolved_steps_rank0"):
        assert o2.get(k) == o.get(k), k
    assert len(o2["per_regression_rank0"]) == 4
