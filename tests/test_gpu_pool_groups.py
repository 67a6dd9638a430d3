"""GPU tier: the pooled safe-set exchange within pool groups (lmpc_set_pool_groups).

One group holding everyone is the ungrouped exchange bit for bit, and reverting returns to it.  A grouped exchange equals the
host books that restate the reference's lists, where every controller imports the fastest laps of its own group -- on one
handle and on two handles that stand for two ranks.  Groups that each drive one circuit keep the circuits apart: each circuit's
controllers equal, bit for bit, a one-circuit handle where they pool among themselves.  Refused calls leave the handle as it
was, a gathered row of a group the handle does not have is never handed out, and a crossed design runs end to end through
benchmarks/rollout_mc.py."""
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
from racinglmpc_b200.controller import BatchedController         # noqa: E402
from racinglmpc_b200.reference_params import TrackParams         # noqa: E402
import closed_loop as cl                                         # noqa: E402
from closed_loop import N, X0, KEYS                              # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LMPC_E_INVALID, LMPC_E_STATE = -1, -4
THREE = [TrackParams.l_shaped(), TrackParams.goggle(), TrackParams.oval()]
TPAD, SHARE = 288, 2
KBEST = SHARE + 1


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _buffers(rows_n, tpad=TPAD):
    dev = torch.device("cuda", 0)
    return (torch.zeros(rows_n, tpad, 9, dtype=torch.float64, device=dev), torch.zeros(rows_n, 4, dtype=torch.int32, device=dev))


def _exchange(c):
    """One exchange of a handle with itself (one rank): export G * kbest rows, import them.  Returns (rows, meta, took)."""
    rows, meta = _buffers(c.pool_groups * KBEST)
    c.pool_export(KBEST, TPAD, 0, rows, meta)
    took = c.pool_import(c.pool_groups * KBEST, SHARE, TPAD, 0, rows, meta, count=True)
    return rows.cpu().numpy(), meta.cpu().numpy(), took


def _pooled_loop(B, steps, xsteps, track=None, tracks=None, tidx=None, hook=None, at=None):
    """Device closed loop (PID lap, seeding, LMPC steps) with an exchange at every step in `xsteps` -- a fixed schedule, not
    the progress poll.  `hook(c)` runs once the tables are installed, `at(c)` once before the first exchange.  Returns
    (run, laps, exchanges): the KEYS of every controller, the stored safe-set laps of every fifth one, (rows, meta, took) per
    exchange."""
    c = cl.controller(B, track=track)
    if tracks is not None:
        c.set_tracks(tracks, tidx)
    if hook is not None:
        hook(c)
    c.enable_rollout(Tcl=1024)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    xs = []
    for n in range(1, steps + 1):
        c.rollout_step(seed=1234)
        c.rollout_commit_laps_dev()
        if n in xsteps:
            if at is not None and not xs:
                at(c)
            xs.append(_exchange(c))
    bk = c.books()
    flags, unsolved = c.rollout_health()
    st = c.rollout_state()
    laps = {}
    for b in range(0, B, 5):
        for slot in range(7):
            T = C.c_int(0)
            x, u, q = np.zeros((1280, 6)), np.zeros((1280, 2)), np.zeros(1280)
            nat.check(nat.lib().lmpc_ss_get_lap(c._h, b, slot, C.byref(T), nat.ptr(x), nat.ptr(u), nat.ptr(q)))
            laps[(b, slot)] = (x[:T.value].copy(), u[:T.value].copy(), q[:T.value].copy())
    c.close()
    return dict(bk, flags=flags, unsolved=unsolved, **st), laps, xs


XSTEPS = (120, 250, 330)


def test_one_group_equals_no_groups_bit_for_bit():
    """ngroups = 1 (all zeros) exports the same rows and meta and leaves the same closed loop, lap books and stored laps as a
    handle without groups; installing three groups and reverting with ngroups = 0 equals a handle that never had groups."""
    _need_gpu()
    B, steps = 64, 360
    none = _pooled_loop(B, steps, XSTEPS)
    one = _pooled_loop(B, steps, XSTEPS, hook=lambda c: c.set_pool_groups(np.zeros(B, np.int32), 1))

    def revert(c):
        c.set_pool_groups(np.arange(B) % 3, 3)
        assert c.pool_groups == 3
        c.set_pool_groups(None)
        assert c.pool_groups == 1
    reverted = _pooled_loop(B, steps, XSTEPS, hook=revert)
    everyone = np.ones(B, bool)
    for other, what in ((one, "one group"), (reverted, "reverted")):
        cl.same(none[:2], other[:2], everyone, what)
        assert len(other[2]) == len(none[2]) == len(XSTEPS)
        for (ra, ma, ta), (rb, mb, tb) in zip(none[2], other[2]):
            assert np.array_equal(ra, rb) and np.array_equal(ma, mb) and ta == tb, what
    assert not none[2][0][1][:, 3].any()                       # meta[:, 3] = 0 without groups
    assert sum(t for _, _, t in none[2]) > 0


def _host_seeded(gold, track, B):
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    xP, uP = gold["pid_x"].copy(), gold["pid_u"].copy()
    c = BatchedController(par, B, track.seg_table(), track.TrackLength, trToUse=4, numSS_Points=numSS_Points,
                          numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1536, ss_cap=7, model_cap=5)
    for b in range(B):
        for _ in range(4):
            c.model_add_trajectory(b, xP, uP)
        for _ in range(4):
            c.add_trajectory(b, xP, uP)
    c.set_state(xLin=np.tile(xP[1:N + 2], (B, 1, 1)), uLin=np.tile(uP[1:N + 1], (B, 1, 1)),
                zt=np.tile(np.array([0.0, 0, 0, 0, 10.0, 0]), (B, 1)), OldInput=np.zeros((B, 2)), timeStep=np.zeros(B, np.int32),
                has_pred=np.zeros(B, np.int32))
    c.enable_rollout(Tcl=512)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    return c


def _check_books(ca, cb, lo, laps_a):
    """Device books of handle cb (controllers lo, lo+1, ... of the host controller ca) equal ca's host books."""
    numSS_it = ca.numSS_it
    bk = cb.books()
    for i in range(cb.B):
        b = lo + i
        host = sorted((ca.LapTime[b][ln], ln) for ln in ca.ss_book[b].slot_of)
        devb = sorted((int(t), int(l)) for t, l in zip(bk["ss_time"][i], bk["ss_lap"][i]) if l >= 0)
        assert host == devb, (b, host, devb)
        assert int(bk["it"][i]) == ca.it[b]
        order = [int(bk["ss_lap"][i][s]) for s in bk["sel"][i]]
        assert order == [int(j) for j in np.argsort(np.array(ca.LapTime[b]), kind="stable")[:numSS_it]], b
        hostm = sorted((T, ln) for T, ln in ca.model_laps[b] if ln in ca.model_book[b].slot_of)
        devm = sorted((int(t), int(q)) for t, q in zip(bk["md_time"][i], bk["md_seq"][i]) if q >= 0)
        assert hostm == devm, (b, hostm, devm)
        assert [int(bk["md_seq"][i][s]) for s in bk["used"][i]] == [ln for _, ln in ca.model_laps[b][:4]], b
        assert list(bk["lap_hist"][i][:len(laps_a[b])]) == laps_a[b]


def _host_grouped_exchange(ca, grp, Tpad):
    """The host restatement: every controller imports the `SHARE` fastest latest-own laps of its own group that it does not own
    (export_laps / import_laps with sharding.pooled_fastest(groups=)).  Returns (best per group, lap times)."""
    B = ca.B
    rows = torch.zeros(B, Tpad, 9, dtype=torch.float64, device="cuda")
    lens = torch.zeros(B, dtype=torch.int32, device="cuda")
    own = [ca.it[b] - 1 for b in range(B)]
    ca.export_laps(own, Tpad, rows, lens)
    times = np.array([ca.LapTime[b][own[b]] for b in range(B)])
    best = [[int(i) for i in g] for g in sharding.pooled_fastest(times, KBEST, groups=grp)]
    for j in range(SHARE):
        src = np.full(B, -1, np.int32)
        lt = np.zeros(B, np.int64)
        for b in range(B):
            cand = [g for g in best[grp[b]] if g != b]
            src[b], lt[b] = cand[j], times[cand[j]]
        ca.import_laps(src, lt, Tpad, rows, lens)
    return best, times


def _drive(ca, cbs, zs, laps_a, k):
    """One closed-loop step of the host-book controller ca and of the device-book handles cbs (consecutive controller ranges of
    ca) with the same explicit draws zs[k]."""
    ca.rollout_step(z=zs[k])
    lo = 0
    for cb in cbs:
        cb.rollout_step(z=zs[k][lo:lo + cb.B])
        lo += cb.B
    done, n = ca.rollout_done()
    if done.any():
        for b in np.nonzero(done)[0]:
            laps_a[b].append(int(n[b]))
        ca.rollout_finish_laps(done, n)
    lo = 0
    for cb in cbs:
        cb.rollout_commit_laps_dev()
        sa, sb = ca.rollout_state(), cb.rollout_state()
        assert np.array_equal(sa["x"][lo:lo + cb.B], sb["x"]) and np.array_equal(sa["cl_len"][lo:lo + cb.B], sb["cl_len"]), k
        lo += cb.B


def _until_two_laps(ca, cbs, zs, laps_a):
    k = 0
    while min(len(l) for l in laps_a) < 2:
        _drive(ca, cbs, zs, laps_a, k)
        k += 1
        assert k < 560
    for _ in range(40):                                     # well into the next lap: lap it-1 has grown by addPoint rows
        _drive(ca, cbs, zs, laps_a, k)
        k += 1
    return k


def test_grouped_exchange_matches_the_host_books(gold, track):
    """B = 12 controllers in 3 groups with different noise levels: after one grouped exchange the device books equal the host
    books in which every controller imported the fastest laps of its own group; meta is group-major with meta[:, 3] = g and
    each group's global ids and lap times are the host ranking; the books keep agreeing as the loop goes on."""
    _need_gpu()
    B, G = 12, 3
    grp = np.array([0, 1, 2, 2, 1, 0, 0, 2, 1, 1, 2, 0], np.int32)
    ca, cb = _host_seeded(gold, track, B), _host_seeded(gold, track, B)
    cb.enable_device_books()
    cb.set_pool_groups(grp, G)
    zs = np.random.default_rng(7).standard_normal((760, B, 3)) * np.linspace(0.5, 3.0, B)[None, :, None]
    laps_a = [[] for _ in range(B)]
    k = _until_two_laps(ca, [cb], zs, laps_a)
    _check_books(ca, cb, 0, laps_a)

    best, times = _host_grouped_exchange(ca, grp, TPAD)
    rows, meta = _buffers(G * KBEST)
    cb.pool_export(KBEST, TPAD, 0, rows, meta)
    took = cb.pool_import(G * KBEST, SHARE, TPAD, 0, rows, meta, count=True)
    m = meta.cpu().numpy()
    assert m[:, 3].tolist() == np.repeat(np.arange(G), KBEST).tolist()
    for g in range(G):
        blk = m[g * KBEST:(g + 1) * KBEST]
        assert [int(x) for x in blk[:, 2]] == best[g], (g, blk, best[g])
        assert [int(x) for x in blk[:, 1]] == [int(times[i]) for i in best[g]]
        assert all(grp[i] == g for i in best[g])
    assert took >= 1
    _check_books(ca, cb, 0, laps_a)
    for _ in range(60):
        _drive(ca, [cb], zs, laps_a, k)
        k += 1
    _check_books(ca, cb, 0, laps_a)
    ca.close(); cb.close()


def test_two_ranks_on_one_gpu_match_the_host_books_over_the_union(gold, track):
    """Two handles stand for two ranks (global ids 0.. and B..).  Their exports, concatenated as an all-gather lays them out
    ([2][G][kbest]), are imported into both; each handle's books equal the host books of one 2B-controller batch that pools the
    union by group with global ids.  The host controller b sees the same draws as controller b of its rank."""
    _need_gpu()
    B, G = 8, 3
    grp = (np.arange(2 * B) * 7 // 3) % G
    grp = grp.astype(np.int32)
    ca = _host_seeded(gold, track, 2 * B)
    r0, r1 = _host_seeded(gold, track, B), _host_seeded(gold, track, B)
    for r, lo in ((r0, 0), (r1, B)):
        r.enable_device_books()
        r.set_pool_groups(grp[lo:lo + B], G)
    zs = np.random.default_rng(11).standard_normal((760, 2 * B, 3)) * np.linspace(0.5, 3.0, 2 * B)[None, :, None]
    laps_a = [[] for _ in range(2 * B)]
    k = _until_two_laps(ca, [r0, r1], zs, laps_a)

    best, times = _host_grouped_exchange(ca, grp, TPAD)
    (rows0, meta0), (rows1, meta1) = _buffers(G * KBEST), _buffers(G * KBEST)
    r0.pool_export(KBEST, TPAD, 0, rows0, meta0)
    r1.pool_export(KBEST, TPAD, B, rows1, meta1)
    rows_all, meta_all = torch.cat([rows0, rows1]), torch.cat([meta0, meta1])
    assert r0.pool_import(2 * G * KBEST, SHARE, TPAD, 0, rows_all, meta_all, count=True) >= 1
    assert r1.pool_import(2 * G * KBEST, SHARE, TPAD, B, rows_all, meta_all, count=True) >= 1
    m = meta_all.cpu().numpy()
    for g in range(G):
        ranked = sorted((int(t), int(i)) for t, i, gg in zip(m[:, 1], m[:, 2], m[:, 3]) if gg == g and i >= 0)
        assert [i for _, i in ranked[:KBEST]] == best[g], g
    _check_books(ca, r0, 0, laps_a)
    _check_books(ca, r1, B, laps_a)
    for _ in range(60):
        _drive(ca, [r0, r1], zs, laps_a, k)
        k += 1
    _check_books(ca, r0, 0, laps_a)
    _check_books(ca, r1, B, laps_a)
    ca.close(); r0.close(); r1.close()


def test_circuits_pooled_per_group_are_isolated():
    """Three circuits, groups = track index, exchanges at fixed steps: the controllers of circuit k equal, bit for bit, those of
    a same-size handle where everyone drives circuit k and the circuit-k controllers form group 0.  Mid-run, a grouping that
    spans two circuits is refused on both sides with LMPC_E_STATE and changes nothing."""
    _need_gpu()
    B, steps = 48, 360
    tidx = (np.arange(B) % 3).astype(np.int32)
    L = nat.lib()

    def refuse_spanning(c):
        c.set_pool_groups(np.zeros(B, np.int32), 1)             # one group over three circuits: accepted, checked at exchange
        rows, meta = _buffers(KBEST)
        assert L.lmpc_pool_export_dev(c._h, KBEST, TPAD, 0, nat.ptr(rows), nat.ptr(meta)) == LMPC_E_STATE
        assert L.lmpc_pool_import_dev(c._h, KBEST, SHARE, TPAD, 0, nat.ptr(rows), nat.ptr(meta), None) == LMPC_E_STATE
        c.set_pool_groups(tidx, 3)

    het = _pooled_loop(B, steps, XSTEPS, tracks=THREE, tidx=tidx, hook=lambda c: c.set_pool_groups(tidx, 3), at=refuse_spanning)
    assert all(x[2] > 0 for x in het[2])
    for k in range(3):
        mine = tidx == k
        ref = _pooled_loop(B, steps, XSTEPS, track=THREE[k], hook=lambda c: c.set_pool_groups(np.where(mine, 0, 1), 2))
        cl.same(het[:2], ref[:2], mine, "circuit %d" % k)
        for (_, mh, _), (_, mr, _) in zip(het[2], ref[2]):
            assert np.array_equal(mh[k * KBEST:(k + 1) * KBEST, :3], mr[0:KBEST, :3]), k
    assert len({float(het[0]["lap_hist"][tidx == k, 0].mean()) for k in range(3)}) == 3


def test_refusals_leave_the_handle_unchanged():
    """Bad ngroups, a bad index and a NULL / ngroups mismatch return LMPC_E_INVALID; the call before lmpc_store_create returns
    LMPC_E_STATE; n_src > 64 G returns LMPC_E_INVALID.  After the refusals the handle exports the groups it had.  A gathered row
    of a group outside [0, G) is never handed out: books and laps filed equal those of an import without it."""
    _need_gpu()
    L = nat.lib()
    B = 8
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    p = nat.make_params(par, numSS_Points, numSS_it, Qts)
    h = C.c_void_p()
    nat.check(L.lmpc_create(C.byref(p), B, 0, C.byref(h)))
    ok = np.zeros(B, np.int32)
    assert L.lmpc_set_pool_groups(h, 1, nat.ptr(ok)) == LMPC_E_STATE
    L.lmpc_destroy(h)

    def seeded():
        c = cl.controller(B)
        c.enable_rollout(Tcl=1024)
        c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
        for _ in range(300):
            c.rollout_pid_step(0.8, seed=11)
        c.rollout_seed_from_record_dev(copies=4)
        c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
        for _ in range(30):
            c.rollout_step(seed=5)
            c.rollout_commit_laps_dev()
        c.sync()
        return c

    a, b = seeded(), seeded()
    grp = (np.arange(B) % 2).astype(np.int32)
    a.set_pool_groups(grp, 2)
    b.set_pool_groups(grp, 2)
    bad = [(-1, ok), (65, ok), (B + 1, ok), (2, np.full(B, 2, np.int32)), (2, np.full(B, -1, np.int32)), (0, ok), (2, None)]
    for ng, ix in bad:
        assert L.lmpc_set_pool_groups(a._h, ng, nat.ptr(ix) if ix is not None else None) == LMPC_E_INVALID, ng
    with pytest.raises(ValueError):
        a.set_pool_groups(np.full(B, 3), 2)
    assert a.pool_groups == 2
    rows, meta = _buffers(2 * KBEST + 1)
    meta[-1] = 77                                              # sentinel: the export writes G * kbest rows, no more
    a.pool_export(KBEST, TPAD, 0, rows, meta)
    m = meta.cpu().numpy()
    assert m[:2 * KBEST, 3].tolist() == [0] * KBEST + [1] * KBEST and m[-1].tolist() == [77] * 4
    assert L.lmpc_pool_import_dev(a._h, 64 * 2 + 1, SHARE, TPAD, 0, nat.ptr(rows), nat.ptr(meta), None) == LMPC_E_INVALID

    # a row of group 5 (and one of group -1) that would be the fastest of all: never handed out
    n = 2 * KBEST
    rb, mb = _buffers(n)
    b.pool_export(KBEST, TPAD, 0, rb, mb)
    assert torch.equal(rb, rows[:n]) and torch.equal(mb, meta[:n])
    stray_r = torch.cat([rows[:n], rows[0:1], rows[KBEST:KBEST + 1]])
    stray_m = torch.cat([meta[:n], meta[0:1], meta[KBEST:KBEST + 1]])
    stray_m[n, 1], stray_m[n, 2], stray_m[n, 3] = 1, 7, 5
    stray_m[n + 1, 1], stray_m[n + 1, 2], stray_m[n + 1, 3] = 1, 6, -1
    took_a = a.pool_import(n + 2, SHARE, TPAD, 0, stray_r, stray_m, count=True)
    took_b = b.pool_import(n, SHARE, TPAD, 0, rb, mb, count=True)
    assert took_a == took_b and took_b >= 1
    ba, bb = a.books(), b.books()
    for key in ("ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt", "sel", "used"):
        assert np.array_equal(ba[key], bb[key]), key
    a.close(); b.close()


def test_crossed_design_end_to_end():
    """rollout_mc.run in the pooled mode over the 3 circuits x 2 lane widths (bx through lmpc_set_param_sets), pooled per cell
    (design_groups), against the same batch in the independent mode: every controller finishes its laps, every group files
    laps, no late acceptance, and pooling flags no more controllers than the independent mode.  The oval laps ~30 % faster than
    the other two circuits, so when the batch is ready its controllers hold laps that have just ended; the export ships only
    laps with `ship_after` rows past the finish line (lmpc_set_pool_min_overrun), which an importer's safe-set window needs."""
    _need_gpu()
    sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
    try:
        import rollout_mc
    finally:
        sys.path.pop(0)
    B, laps = 192, 2
    _, _, _, _, Qts, base = rp.lmpc_params(N)
    ps = []
    for w in (0.4, 0.3):
        q = copy.deepcopy(base)
        q.bx = np.array([w, w])
        ps.append(q)
    b = np.arange(B)
    tidx, pidx = b % 3, (b // 3) % 2
    groups = sharding.design_groups(tidx, pidx)
    assert groups[1] == 6
    runs = {}
    for mode in ("independent", "pooled"):
        bk = {}
        out = rollout_mc.run(batch=B, laps=laps, mode=mode, local=0, books=bk, max_steps=1200, track_sets=(THREE, tidx),
                             param_sets=(ps, pidx, [Qts, Qts]), pool_groups=groups if mode == "pooled" else None)
        assert np.all(bk["lap_n"] >= laps), mode
        assert out["late_accepts_rank0"] == 0, mode
        runs[mode] = (out, bk)
    out, bk = runs["pooled"]
    assert out["exchanges"] == laps - 1 and out["pool_groups"] == 6
    assert out["allgather_bytes_per_rank"] == 6 * KBEST * (TPAD * 9 * 8 + 16)
    filed = out["laps_filed_per_group_rank0"]
    assert len(filed) == 6 and all(f > 0 for f in filed) and sum(filed) == out["laps_filed_rank0"]
    flagged = {m: (r[1]["flags_or"] != 0) for m, r in runs.items()}
    for k in range(3):
        on = tidx == k
        assert flagged["pooled"][on].sum() <= flagged["independent"][on].sum(), (k, flagged["pooled"][on].sum())


def test_export_ships_invalid_rows_for_short_groups_and_short_overruns():
    """A group with fewer controllers on the rank than kbest, or none, ships its laps followed by rows with global id -1; a
    latest lap whose shipped rows (at most Tpad) reach fewer rows past its finish line than lmpc_set_pool_min_overrun asks is not
    shipped, one with enough is."""
    _need_gpu()
    L = nat.lib()
    B, steps = 8, 30
    c = cl.controller(B)
    c.enable_rollout(Tcl=1024)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    for _ in range(300):
        c.rollout_pid_step(0.8, seed=11)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    for _ in range(steps):                                  # addPoint appends `steps` rows past the seeded lap's finish line
        c.rollout_step(seed=5)
        c.rollout_commit_laps_dev()
    c.sync()
    assert L.lmpc_set_pool_min_overrun(c._h, -1) == LMPC_E_INVALID
    grp = np.array([0, 0, 0, 0, 0, 0, 0, 1], np.int32)      # group 1: one controller, group 2: none
    c.set_pool_groups(grp, 3)
    # the seeded lap has 300 rows (lap time 300): Tpad = 400 ships all of them and the `steps` rows past the finish line,
    # Tpad = 320 cuts the rows past the finish line to 20
    for tpad, min_over, valid in ((400, 0, [3, 1, 0]), (400, steps, [3, 1, 0]), (400, steps + 1, [0, 0, 0]), (320, 20, [3, 1, 0]),
                                 (320, 21, [0, 0, 0])):
        c.set_pool_min_overrun(min_over)
        rows, meta = _buffers(3 * KBEST, tpad)
        c.pool_export(KBEST, tpad, 100, rows, meta)
        m = meta.cpu().numpy()
        assert m[:, 3].tolist() == np.repeat(np.arange(3), KBEST).tolist()
        for g in range(3):
            blk = m[g * KBEST:(g + 1) * KBEST]
            gids = [int(x) for x in blk[:, 2]]
            assert gids[valid[g]:] == [-1] * (KBEST - valid[g]), (min_over, g, gids)
            assert all(grp[x - 100] == g for x in gids[:valid[g]]), (g, gids)
            assert np.all(blk[:valid[g], 0] - blk[:valid[g], 1] >= min_over)
            assert np.all(blk[valid[g]:, 0] == 0) and not rows[g * KBEST + valid[g]:(g + 1) * KBEST].any()
    c.close()


def test_group_limit_is_the_librarys_own():
    """With more than 64 controllers, ngroups = 65 is refused by the group limit (not by ngroups <= batch); 64 is accepted."""
    _need_gpu()
    L = nat.lib()
    B = 80
    c = cl.controller(B, Tmax=64, ss_cap=6, model_cap=5)
    assert L.lmpc_set_pool_groups(c._h, 65, nat.ptr((np.arange(B) % 65).astype(np.int32))) == LMPC_E_INVALID
    assert "LMPC_MAX_POOL_GROUPS" in L.lmpc_last_error().decode()
    nat.check(L.lmpc_set_pool_groups(c._h, 64, nat.ptr((np.arange(B) % 64).astype(np.int32))))
    rows, meta = _buffers(64 * KBEST)
    c.pool_export(KBEST, TPAD, 0, rows, meta)               # no laps stored: every row is invalid, every group labelled
    m = meta.cpu().numpy()
    assert m[:, 3].tolist() == np.repeat(np.arange(64), KBEST).tolist() and np.all(m[:, 2] == -1)
    c.close()
