"""GPU tier: per-controller noise models and common random numbers of the device closed loop (lmpc_rollout_set_noise,
lmpc_rollout_set_noise_streams).

A batch of several noise sets is several one-set batches in one launch, and the heterogeneous PID lap follows the test-side PID and
dynModel (tests/support/noise_model.py) with each controller's set.  The reference's noise installed as one set equals a handle
without sets, identity streams equal no streams, and both revert.  A zero-noise set makes the closed loop independent of the
seed.  Streams move a controller's draws: controllers on one stream drive the closed loop of that stream, tuning pairs on one
stream share their PID lap and their seeded stores.  Refused calls leave the handle as it was, and a run captured and resumed with
noise sets and streams installed equals a straight run."""
import copy
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                # noqa: E402
from racinglmpc_b200 import _native as nat                        # noqa: E402
from racinglmpc_b200.controller import BatchedController          # noqa: E402
from racinglmpc_b200.reference_params import NoiseParams          # noqa: E402
import closed_loop as cl                                          # noqa: E402
import noise_model as nm                                          # noqa: E402
from closed_loop import N, X0, KEYS                               # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LMPC_E_INVALID = -1
REF = NoiseParams.reference()
B = 256

# interleaved sets of test 1: none, the reference, scaled simulator, scaled PID, other clips
SETS = [NoiseParams.scaled(0, 0), REF, NoiseParams.scaled(10, 1), NoiseParams.scaled(1, 0.5), NoiseParams.scaled(100, 0.5),
        NoiseParams((0.02, 0.03, 0.01), (0.01, 0.2, 0.004), 0.05, (0.4, 0.3), (0.1, 0.5)),
        NoiseParams((0.3, 0.0, 0.2), (0.5, 0.5, 0.0), 0.02, (0.0, 0.5), (0.3, 0.0))]
# the four sets of the batch tests
FOUR = [REF, NoiseParams.scaled(0, 1), NoiseParams.scaled(10, 1), NoiseParams.scaled(1, 0.5)]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


class _Fake:
    def __init__(self, z):
        self._it = iter(np.asarray(z, float).ravel())

    def standard_normal(self):
        return next(self._it)


def test_noise_sets_pid_lap_matches_the_test_side_model(track):
    """Seven noise sets interleaved, host-given draws: one PID step to 1e-12 in both frames, a 300-step PID lap to 1e-9."""
    _need_gpu()
    Bs, K = 2 * len(SETS), 300
    idx = np.arange(Bs) % len(SETS)
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, Bs, track.seg_table(), track.TrackLength, trToUse=4, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=1536, ss_cap=6, model_cap=5)
    c.set_noise(SETS, idx)
    c.set_noise_streams(np.zeros(Bs, np.int32))          # host-given draws do not use the streams
    c.enable_rollout(Tcl=1024)
    c.rollout_set_state(np.tile(X0, (Bs, 1)), np.tile(X0, (Bs, 1)))
    zs = np.random.default_rng(11).standard_normal((Bs, K, 5))
    car = rp.VehicleParams.reference()
    for k in range(K):
        c.rollout_pid_step(0.8, z_pid=zs[:, k, 0:2], z_sim=zs[:, k, 2:5])
        if k == 0:
            st = c.rollout_state()
            for b in range(Bs):
                fake = _Fake(zs[b, 0])
                pid = nm.PIDFollower(0.8, SETS[idx[b]], rng=fake)
                pid.solve(X0)
                xo, go = nm.dyn_model(track, X0, X0, pid.uPred[0], car, SETS[idx[b]], rng=fake)
                assert np.max(np.abs(st["x"][b] - xo)) < 1e-12 and np.max(np.abs(st["xglob"][b] - go)) < 1e-12, b
    st = c.rollout_state()
    assert np.all(st["cl_len"] == K)
    for b in range(Bs):
        fake = _Fake(zs[b])
        xo, uo, go, last = nm.closed_loop(track, [X0, X0], nm.PIDFollower(0.8, SETS[idx[b]], rng=fake), car, SETS[idx[b]],
                                          max_steps=K, rng=fake)
        xg, ug = c.rollout_get_lap(b)
        assert np.max(np.abs(xg - xo)) < 1e-9 and np.max(np.abs(ug - uo)) < 1e-9, b
        assert np.max(np.abs(st["x"][b] - last[0])) < 1e-9 and np.max(np.abs(st["xglob"][b] - last[1])) < 1e-9, b
    # the sets act: without noise the two copies of set 0 drive identically, with noise the copies differ
    x = st["x"]
    assert np.array_equal(x[0], x[len(SETS)]) and not np.array_equal(x[2], x[2 + len(SETS)])
    c.close()


def _reject(c):
    """Refused calls, each returning LMPC_E_INVALID; the handle must stay as it was."""
    L = nat.lib()
    idx = np.arange(B, dtype=np.int32) % 4
    good, _ = nat.make_noise_sets(FOUR, idx, B)

    def copy_of(mod):
        t = (nat.NoiseParams * 4)()
        C.memmove(t, good, C.sizeof(t))
        mod(t)
        return t
    bad = [copy_of(lambda t: t[1].sim_sigma.__setitem__(2, -0.01)), copy_of(lambda t: t[2].pid_clip.__setitem__(0, float("nan"))),
           copy_of(lambda t: setattr(t[3], "sim_gain", float("inf"))), copy_of(lambda t: t[0].sim_clip.__setitem__(1, -1e-300))]
    cases = [(t, 4, idx) for t in bad] + [(good, 4, np.full(B, 4, np.int32)), (good, 4, np.full(B, -1, np.int32)), (good, 0, idx),
                                          (None, 4, idx), (good, 4, None)]
    for tab, n, ix in cases:
        assert L.lmpc_rollout_set_noise(c._h, tab, n, nat.ptr(ix) if ix is not None else None) == LMPC_E_INVALID
    big = (nat.NoiseParams * (B + 1))(*([good[0]] * (B + 1)))
    assert L.lmpc_rollout_set_noise(c._h, big, B + 1, nat.ptr(np.zeros(B, np.int32))) == LMPC_E_INVALID
    s = np.arange(B, dtype=np.int32)[::-1].copy()
    s[B // 2] = -1
    assert L.lmpc_rollout_set_noise_streams(c._h, nat.ptr(s)) == LMPC_E_INVALID


@pytest.fixture(scope="module")
def runs():
    """A batch of FOUR (noise set b % 4, Philox) with refused calls before the run, and one handle per set."""
    _need_gpu()
    nidx = np.arange(B) % 4

    def install(c):
        c.set_noise(FOUR, nidx)
        _reject(c)

    n, het, het_laps = cl.run(B, hook=install)
    assert het["lap_n"].min() >= 1, "not every controller finished an LMPC lap in %d steps" % n
    refs = [cl.run(B, hook=lambda c, v=v: c.set_noise([v], np.zeros(B, np.int32)), steps=n)[1:] for v in FOUR]
    none = cl.run(B, steps=n)[1:]
    return dict(n=n, nidx=nidx, het=(het, het_laps), refs=refs, none=none)


def test_batch_of_noise_sets_equals_one_handle_per_set(runs):
    """Refused calls before the run changed nothing; the sets drove different laps."""
    for k in range(4):
        cl.same(runs["het"], runs["refs"][k], runs["nidx"] == k, "noise set %d" % k)
    h = runs["het"][0]
    assert len({float(h["lap_hist"][runs["nidx"] == k, 0].mean()) for k in range(4)}) == 4


def test_traced_batch_gives_the_same_results(runs):
    _, het, laps = cl.run(B, hook=lambda c: c.set_noise(FOUR, runs["nidx"]), steps=runs["n"], trace=True)
    for k in range(4):
        cl.same((het, laps), runs["refs"][k], runs["nidx"] == k, "traced, noise set %d" % k)


def test_defaults_and_revert(runs):
    """The reference as one set equals no sets; identity streams equal no streams; nsets == 0 and streams=None revert."""
    n, every = runs["n"], np.ones(B, bool)
    cl.same(runs["none"], runs["refs"][0], every, "reference as one set vs no sets")
    ident = cl.run(B, hook=lambda c: c.set_noise_streams(np.arange(B)), steps=n)[1:]
    cl.same(ident, runs["none"], every, "identity streams vs no streams")

    def install_then_revert(c):
        c.set_noise(FOUR, runs["nidx"])
        c.set_noise_streams(np.zeros(B, np.int32))
        with pytest.raises(ValueError):
            c.set_noise(None, runs["nidx"])          # reverting takes no index
        with pytest.raises(ValueError):
            c.set_noise(FOUR)                        # sets need one
        with pytest.raises(ValueError):
            c.set_noise_streams(np.full(B, -1))
        c.set_noise(None)
        c.set_noise_streams(None)

    reverted = cl.run(B, hook=install_then_revert, steps=n)[1:]
    cl.same(reverted, runs["none"], every, "nsets == 0 and streams=None revert")


def test_zero_noise_is_independent_of_the_seed(runs):
    """A zero-noise set under two seeds, and the reference's noise with host-given draws of zeros: one closed loop."""
    n, every = runs["n"], np.ones(B, bool)
    def quiet(c, seeds=None):
        c.set_noise([NoiseParams.scaled(0, 0)], np.zeros(B, np.int32))
        if seeds:
            nm.with_draws(c, seeds=seeds)
    a = cl.run(B, hook=quiet, steps=n)[1:]
    b = cl.run(B, hook=lambda c: quiet(c, seeds=(99, 7)), steps=n)[1:]
    z = cl.run(B, hook=lambda c: nm.with_draws(c, zeros=True), steps=n)[1:]
    cl.same(a, b, every, "zero noise, two seeds")
    cl.same(a, z, every, "zero noise vs host draws of zeros")
    # every controller of a noise-free batch drives the same closed loop
    for key in ("x", "lap_hist", "ss_time"):
        assert np.all(a[0][key] == a[0][key][0]), key


def _same_mapped(a, b, dst, src, what):
    """Controller dst[i] of run a equals controller src[i] of run b bit for bit (KEYS and the stored laps both runs kept)."""
    (ar, al), (br, bl) = a, b
    for key in KEYS:
        assert np.array_equal(ar[key][dst], br[key][src]), (what, key)
    m = dict(zip(dst.tolist(), src.tolist()))
    hit = 0
    for (i, slot), v in al.items():
        if i in m and (m[i], slot) in bl:
            assert all(np.array_equal(p, q) for p, q in zip(v, bl[(m[i], slot)])), (what, i, slot)
            hit += 1
    return hit


def test_streams_move_the_draws(runs):
    """Every controller on stream 0 drives controller 0's closed loop; a permutation of streams permutes the closed loops."""
    n = runs["n"]
    b = np.arange(B)
    zero = cl.run(B, hook=lambda c: c.set_noise_streams(np.zeros(B, np.int32)), steps=n)[1:]
    _same_mapped(zero, runs["none"], b, np.zeros(B, int), "stream 0 everywhere")
    perm = np.random.default_rng(5).permutation(B)
    p = cl.run(B, hook=lambda c: c.set_noise_streams(perm), steps=n)[1:]
    _same_mapped(p, runs["none"], b, perm, "permuted streams")
    assert not np.array_equal(p[0]["x"], runs["none"][0]["x"])


def test_tuning_pairs_on_one_stream_share_their_noise():
    """Two tunings interleaved (tuning b % 2) on streams b // 2: controller b equals controller b // 2 of a handle on which every
    controller runs b's tuning without streams, so each pair shares its PID lap, its seeded stores and every later draw."""
    _need_gpu()
    _, _, _, _, Qts, base = rp.lmpc_params(N)
    ps = []
    for k in range(2):
        p = copy.deepcopy(base)
        p.dR = (0.5, 2.0)[k] * np.asarray(base.dR, float)
        ps.append(p)
    b = np.arange(B)
    pidx = b % 2
    n, het, het_laps = cl.run(B, psets=(ps, pidx, [Qts, Qts]), hook=lambda c: c.set_noise_streams(b // 2))
    assert het["lap_n"].min() >= 1
    for i in range(2):
        ref = cl.run(B, par=ps[i], qts=Qts, steps=n)[1:]
        sel = b[pidx == i]
        _same_mapped((het, het_laps), ref, sel, sel // 2, "tuning %d on stream b // 2" % i)
    # the tunings drive different LMPC laps
    assert not np.array_equal(het["lap_hist"][0::2, 0], het["lap_hist"][1::2, 0])


def _rollout_mc():
    sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
    try:
        import rollout_mc
    finally:
        sys.path.pop(0)
    return rollout_mc


def test_capture_and_resume_with_noise_sets_and_streams():
    """rollout_mc.run with noise sets and streams installed: 1 lap captured and resumed to 2 equals a straight run to 2 laps."""
    _need_gpu()
    rm = _rollout_mc()
    Bs = 256
    kw = dict(batch=Bs, local=0, noise_sets=(FOUR, np.arange(Bs) % 4), noise_streams=np.arange(Bs) // 2)
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
    for k in ("lap_stats_rank0", "per_noise_rank0", "instances_with_flags_rank0", "unsolved_steps_rank0"):
        assert o2.get(k) == o.get(k), k
    assert len(o2["per_noise_rank0"]) == 4
