"""GPU tier: per-group readiness of the pooled exchange (lmpc_rollout_group_stats, lmpc_pool_export_groups_dev,
rollout_mc.run(readiness="group")).

The per-group progress numbers equal a numpy reduction of the books, the closed-loop state and the health counters; the row
of one group is lmpc_rollout_stats and an empty group reports the sentinel.  A masked export ships the unmasked groups exactly
as the plain export and invalid rows for the others, and after the import the controllers of a masked group equal a handle
that skipped the exchange.  Without groups "group" readiness is "batch" readiness bit for bit.  With it, the controllers of
one circuit in a three-circuit batch equal a batch on that circuit alone, exchange steps included, and a crossed design runs
end to end with the oval groups exchanging earlier than under "batch" readiness."""
import copy
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp, sharding     # noqa: E402
from racinglmpc_b200 import _native as nat                       # noqa: E402
from racinglmpc_b200.reference_params import TrackParams         # noqa: E402
import closed_loop as cl                                         # noqa: E402
from closed_loop import N, X0, KEYS                              # noqa: E402
from group_stats import INT32_MAX, group_stats                   # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LMPC_E_INVALID = -1
THREE = [TrackParams.l_shaped(), TrackParams.goggle(), TrackParams.oval()]
OVAL = 2
TPAD, SHARE = 288, 2
KBEST = SHARE + 1


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _rollout_mc():
    sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
    try:
        import rollout_mc
    finally:
        sys.path.pop(0)
    return rollout_mc


def _buffers(rows_n):
    dev = torch.device("cuda", 0)
    return (torch.zeros(rows_n, TPAD, 9, dtype=torch.float64, device=dev), torch.zeros(rows_n, 4, dtype=torch.int32, device=dev))


def _seeded(B, tidx, groups, G):
    """Three circuits (track = tidx), pool groups installed, PID lap, seeding: ready for LMPC steps."""
    c = cl.controller(B)
    c.set_tracks(THREE, tidx)
    c.set_pool_groups(groups, G)
    c.enable_rollout(Tcl=1024)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    return c


def _steps(c, n):
    for _ in range(n):
        c.rollout_step(seed=1234)
        c.rollout_commit_laps_dev()


def _snapshot(c):
    """KEYS of every controller and every stored safe-set lap."""
    bk = c.books()
    flags, unsolved = c.rollout_health()
    run = dict(bk, flags=flags, unsolved=unsolved, **c.rollout_state())
    laps = {}
    for b in range(c.B):
        for slot in range(7):
            T = C.c_int(0)
            x, u, q = np.zeros((1280, 6)), np.zeros((1280, 2)), np.zeros(1280)
            nat.check(nat.lib().lmpc_ss_get_lap(c._h, b, slot, C.byref(T), nat.ptr(x), nat.ptr(u), nat.ptr(q)))
            laps[(b, slot)] = (x[:T.value].copy(), u[:T.value].copy(), q[:T.value].copy())
    return run, laps


def test_group_stats_equal_a_numpy_reduction():
    """Three circuits, one group per circuit plus an empty fourth group: at several points of the closed loop the rows equal the
    reduction of lap_n, cl_len and the health flags per group; the empty group reports (INT32_MAX, 0, INT32_MAX, 0); without
    groups the one row is rollout_stats."""
    _need_gpu()
    B, G = 48, 4
    tidx = (np.arange(B) % 3).astype(np.int32)
    c = _seeded(B, tidx, tidx, G)
    seen_laps = set()
    for n in (8, 120, 90, 100, 80):
        _steps(c, n)
        got = c.rollout_group_stats()
        assert got.dtype == np.int32 and got.shape == (G, 4)
        lap_n, cl_len, flags = c.books()["lap_n"], c.rollout_state()["cl_len"], c.rollout_health()[0]
        assert np.array_equal(got, group_stats(lap_n, cl_len, flags, tidx, G)), (n, got)
        assert got[3].tolist() == [INT32_MAX, 0, INT32_MAX, 0]
        seen_laps.update(int(v) for v in got[:3, 0])
        c.set_pool_groups(None)
        one = c.rollout_group_stats()
        assert one.shape == (1, 4) and one[0].tolist() == list(c.rollout_stats())
        assert np.array_equal(one, group_stats(lap_n, cl_len, flags, np.zeros(B, int), 1))
        c.set_pool_groups(tidx, G)
    assert len(seen_laps) >= 2                                  # the groups were at different laps at some point
    c.close()


def test_masked_export_and_import():
    """Three handles driven identically (groups = circuit): a full exchange, an exchange with group 1 masked out, none.
    The all-ones mask exports what the plain export does; the masked export ships invalid rows for group 1 and the same rows
    for the others; after the import (and 60 more steps) group 1 equals the handle without exchange and the others equal the
    full exchange.  Bad masks are refused and change nothing."""
    _need_gpu()
    L = nat.lib()
    B, G, at = 48, 3, 330
    tidx = (np.arange(B) % 3).astype(np.int32)
    hs = [_seeded(B, tidx, tidx, G) for _ in range(3)]
    for c in hs:
        _steps(c, at)
    full, masked, skipped = hs
    rows_a, meta_a = _buffers(G * KBEST)
    full.pool_export(KBEST, TPAD, 0, rows_a, meta_a)
    rows_1, meta_1 = _buffers(G * KBEST)
    full.pool_export(KBEST, TPAD, 0, rows_1, meta_1, groups=np.ones(G, bool))
    assert torch.equal(rows_a, rows_1) and torch.equal(meta_a, meta_1)
    assert (meta_a[:, 2] >= 0).all()                           # every group ships laps here

    rows_m, meta_m = _buffers(G * KBEST)
    for bad in (np.array([1, 2, 0], np.int32), np.array([1, -1, 1], np.int32)):
        assert L.lmpc_pool_export_groups_dev(masked._h, KBEST, TPAD, 0, nat.ptr(bad), nat.ptr(rows_m), nat.ptr(meta_m)) == LMPC_E_INVALID
    assert L.lmpc_pool_export_groups_dev(masked._h, KBEST, TPAD, 0, None, nat.ptr(rows_m), nat.ptr(meta_m)) == LMPC_E_INVALID
    assert not rows_m.any() and not meta_m.any()               # a refused call writes nothing
    rows_n, meta_n = _buffers(G * KBEST)
    masked.pool_export(KBEST, TPAD, 0, rows_n, meta_n)         # the next export is unchanged by the refusals
    assert torch.equal(rows_n, rows_a) and torch.equal(meta_n, meta_a)

    masked.pool_export(KBEST, TPAD, 0, rows_m, meta_m, groups=[1, 0, 1])
    g1 = slice(KBEST, 2 * KBEST)
    assert meta_m[g1].cpu().numpy().tolist() == [[0, INT32_MAX, -1, 1]] * KBEST and not rows_m[g1].any()
    for g in (0, 2):
        s = slice(g * KBEST, (g + 1) * KBEST)
        assert torch.equal(rows_m[s], rows_a[s]) and torch.equal(meta_m[s], meta_a[s])

    took_full = full.pool_import(G * KBEST, SHARE, TPAD, 0, rows_a, meta_a, count=True)
    took_masked = masked.pool_import(G * KBEST, SHARE, TPAD, 0, rows_m, meta_m, count=True)
    assert took_full > took_masked > 0
    g = tidx == 1
    for what in ("after the import", "60 steps later"):
        snap = [_snapshot(c) for c in hs]
        cl.same(snap[1], snap[2], g, "masked group vs no exchange, " + what)
        cl.same(snap[1], snap[0], ~g, "other groups vs full exchange, " + what)
        for c in hs:
            _steps(c, 60)
    for c in hs:
        c.close()


def _same_books(a, b, what):
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), (what, k)


def test_group_readiness_without_groups_is_batch_readiness():
    """No pool groups: readiness="group" makes the same decisions at the same steps as "batch" -- books, end state, solver
    report, health, exchange count, exchange steps and launches are identical."""
    _need_gpu()
    rm = _rollout_mc()
    B, laps = 256, 3
    res = {}
    for name, kw in (("batch", {}), ("group", {"readiness": "group"}), ("batch_one_group", {"pool_groups": (np.zeros(B, np.int32), 1)})):
        fin, bk = {}, {}
        out = rm.run(batch=B, laps=laps, local=0, final=fin, books=bk, **kw)
        res[name] = (out, fin, bk)
    (ob, fb, bb), (og, fg, bg), (o1, _, _) = res["batch"], res["group"], res["batch_one_group"]
    assert np.all(bb["lap_n"] >= laps)
    _same_books(bb, bg, "books")
    _same_books(fb, fg, "end state")
    for k in ("closed_loop_steps", "exchanges", "laps_filed_rank0", "lap_stats_rank0", "kernel_launches_rank0",
              "instances_with_flags_rank0", "unsolved_steps_rank0", "late_accepts_rank0", "allgather_bytes_per_rank"):
        assert ob[k] == og[k], k
    assert "readiness" not in ob and "exchange_steps_per_group_rank0" not in ob       # the default output is unchanged
    assert og["readiness"] == "group" and len(og["exchange_steps_per_group_rank0"][0]) == og["exchanges"] == laps - 1
    assert og["exchange_steps_per_group_rank0"] == o1["exchange_steps_per_group_rank0"]


def test_circuits_under_group_readiness_follow_their_own_schedule():
    """Three circuits in one batch, grouped per circuit, readiness="group", 400 steps (no run reaches its 4 laps, so the done
    rule ends none early): the controllers of circuit k equal, bit for bit, a same-size batch on circuit k alone grouped as
    "circuit-k positions" / "the rest", and exchange at the same steps.  Under "batch" readiness the same comparison is
    reported, not asserted: there the oval's schedule follows the slowest circuit."""
    _need_gpu()
    rm = _rollout_mc()
    B, laps, steps = 48, 4, 400
    tidx = (np.arange(B) % 3).astype(np.int32)
    for readiness in ("group", "batch"):
        het_bk, het_fin = {}, {}
        het = rm.run(batch=B, laps=laps, local=0, max_steps=steps, books=het_bk, final=het_fin, track_sets=(THREE, tidx),
                     pool_groups=(tidx, 3), readiness=readiness)
        assert het["closed_loop_steps"] == steps
        for k in range(3):
            mine = tidx == k
            bk, fin = {}, {}
            ref = rm.run(batch=B, laps=laps, local=0, max_steps=steps, books=bk, final=fin, track_sets=([THREE[k]], np.zeros(B, np.int32)),
                         pool_groups=(np.where(mine, 0, 1).astype(np.int32), 2), readiness=readiness)
            assert ref["closed_loop_steps"] == steps
            same = all(np.array_equal(np.asarray(het_bk[key])[mine], np.asarray(bk[key])[mine]) for key in het_bk) and \
                all(np.array_equal(np.asarray(het_fin[key])[mine], np.asarray(fin[key])[mine]) for key in ("x", "xglob", "done", "cl_len"))
            xs_het, xs_ref = het["exchange_steps_per_group_rank0"][k], ref["exchange_steps_per_group_rank0"][0]
            print("readiness=%s circuit %d: identical to the one-circuit batch: %s; exchange steps %s vs %s" % (readiness, k, same, xs_het, xs_ref))
            if readiness == "group":
                assert same, k
                assert xs_het == xs_ref and len(xs_het) >= 1, (k, xs_het, xs_ref)


def test_crossed_design_end_to_end_under_group_readiness():
    """3 circuits x 2 lane widths pooled per cell with readiness="group": every controller finishes, every group exchanges
    laps - 1 times and files laps, no late acceptance, no more flagged controllers per circuit than the independent mode, and
    every oval group exchanges for the first time before the batch-readiness run does."""
    _need_gpu()
    rm = _rollout_mc()
    B, laps = 192, 2
    _, _, _, _, Qts, base = rp.lmpc_params(N)
    ps = []
    for w in (0.4, 0.3):
        q = copy.deepcopy(base)
        q.bx = np.array([w, w])
        ps.append(q)
    b = np.arange(B)
    tidx, pidx = b % 3, (b // 3) % 2
    groups, G = sharding.design_groups(tidx, pidx)
    runs = {}
    for name, mode, readiness in (("independent", "independent", "batch"), ("batch", "pooled", "batch"), ("group", "pooled", "group")):
        bk = {}
        out = rm.run(batch=B, laps=laps, mode=mode, local=0, books=bk, max_steps=1200, track_sets=(THREE, tidx),
                     param_sets=(ps, pidx, [Qts, Qts]), pool_groups=(groups, G) if mode == "pooled" else None, readiness=readiness)
        assert np.all(bk["lap_n"] >= laps), name
        assert out["late_accepts_rank0"] == 0, name
        runs[name] = (out, bk)
    out, bk = runs["group"]
    assert out["readiness"] == "group" and out["pool_groups"] == G == 6
    xs = out["exchange_steps_per_group_rank0"]
    assert all(len(s) == laps - 1 for s in xs), xs
    assert all(f > 0 for f in out["laps_filed_per_group_rank0"])
    flagged = {m: (r[1]["flags_or"] != 0) for m, r in runs.items()}
    for k in range(3):
        on = tidx == k
        assert flagged["group"][on].sum() <= flagged["independent"][on].sum(), (k, flagged["group"][on].sum())
    batch_first = runs["batch"][0]["exchange_steps_per_group_rank0"][0][0]
    for g in range(G):
        if tidx[np.nonzero(groups == g)[0][0]] == OVAL:
            assert xs[g][0] < batch_first, (g, xs[g], batch_first)
    print("crossed design: exchange steps per group, group readiness %s; batch readiness first exchange at %d" % (xs, batch_first))
