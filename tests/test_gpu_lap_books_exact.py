"""GPU tier: the device lap books and the pooled exchange (csrc/lapbooks.cuh) against the unbounded lists of
tests/support/lapbook_exact.py, through public entry points only, compared after every event.

Own laps go in through a snapshot: the test writes fingerprinted rows into the closed-loop record of the controllers that finish,
sets cl_len = T and done = 1, restores, and calls lmpc_rollout_commit_laps_dev, so each controller follows its own sequence of
lap lengths with no simulator step.  Imports go in through lmpc_pool_import_dev with crafted rows and meta.  After every event the
slot tables must hold the model's laps with the model's times, the resident laps, the selection in order, is_prev, the addPoint
target, usedIt, the lap history and health bit 64; every few events the stored rows of every lap a kernel reads must equal the
model's lap bit for bit."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import _native as nat, reference_params as rp     # noqa: E402
from racinglmpc_b200.controller import BatchedController               # noqa: E402
from racinglmpc_b200.reference_params import TrackParams               # noqa: E402
import lapbook_exact as lx                                             # noqa: E402

GRID = [(4, 6, 4, 5), (4, 7, 4, 5), (4, 4, 4, 4), (4, 5, 4, 4), (1, 2, 1, 1), (2, 4, 8, 8), (8, 10, 8, 9)]
TMAX, TCL, TPAD = 40, 56, 32          # laps longer than Tmax, and shipped rows cut at Tpad < Tmax
B, G = 16, 2
ROUNDS, XEVERY = 50, 4                # own-lap rounds; an import round before every XEVERY-th
TRACK = TrackParams.l_shaped()
INT_MAX = 0x7FFFFFFF


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _controller(cfg, batch, Tmax=TMAX, Tcl=TCL):
    numSS_it, ss_cap, trToUse, model_cap = cfg
    _, _, _, _, Qts, par = rp.lmpc_params(12)
    M = 24 if (24 // numSS_it) % 2 == 0 else 32          # a built numSS_Points with an even numSS_Points / numSS_it
    c = BatchedController(par, batch, TRACK.seg_table, TRACK.TrackLength, trToUse=trToUse, numSS_Points=M,
                          numSS_it=numSS_it, QterminalSlack=Qts, Tmax=Tmax, ss_cap=ss_cap, model_cap=model_cap)
    c.enable_rollout(Tcl=Tcl)
    c.enable_device_books()               # empty device books: snapshots work from the start
    return c


class _Records:
    """A host copy of every controller's snapshot record with named views of its sections."""

    def __init__(self, c):
        self.raw = c.snapshot().cpu().numpy().copy()
        self.sect = nat.decode_snapshot_header(self.raw[0])["sections"]

    def view(self, name, dtype, shape):
        off, n = self.sect[name]
        return self.raw[:, off:off + n].view(dtype).reshape((self.raw.shape[0],) + shape)

    def restore(self, c):
        c.restore(torch.from_numpy(self.raw).to("cuda"))


def _lap_lengths(rng, kind, n):
    """One controller's own lap lengths: ties from {k, k+1}, strictly decreasing, strictly increasing, T in {1, 2}, around
    and above Tmax (up to Tcl), or uniform."""
    k = int(rng.integers(3, TMAX - 3))
    return {0: lambda: k + rng.integers(0, 2, n), 1: lambda: TCL - np.arange(n) % TCL, 2: lambda: 1 + np.arange(n) % TCL,
            3: lambda: rng.integers(1, 3, n), 4: lambda: rng.integers(TMAX - 3, TCL + 1, n),
            5: lambda: rng.integers(1, TCL + 1, n)}[kind]().astype(int)


def _check_books(c, models, fresh_dead=()):
    bk = c.books()
    flags, _ = c.rollout_health()
    for b, m in enumerate(models):
        if b in fresh_dead:
            assert flags[b] & 64, b
        if m.dead:
            continue
        ctx = (b, m.times, [(t, s) for t, s, _ in m.md])
        assert not flags[b] & 64, ctx
        assert bk["it"][b] == m.it and bk["md_cnt"][b] == m.seq, ctx
        ss = {int(ln): int(t) for t, ln in zip(bk["ss_time"][b], bk["ss_lap"][b]) if ln >= 0}
        assert all(m.times[ln] == t for ln, t in ss.items()), ctx
        assert m.resident() <= set(ss), ctx
        md = {int(s): int(t) for t, s in zip(bk["md_time"][b], bk["md_seq"][b]) if s >= 0}
        by_seq = m.md_by_seq()
        assert all(by_seq[s][0] == t for s, t in md.items()), ctx
        if m.it >= 1:
            sel, _ = m.sel()
            assert [int(bk["ss_lap"][b][s]) for s in bk["sel"][b]] == sel, ctx
            assert list(bk["is_prev"][b]) == m.is_prev(), ctx
            assert bk["ss_lap"][b][bk["prev_slot"][b]] == m.it - 1, ctx
        else:
            assert bk["prev_slot"][b] == -1
        if m.md:
            assert [int(bk["md_seq"][b][u]) for u in bk["used"][b]] == m.used(), ctx
        n = len(m.lap_hist)
        assert bk["lap_n"][b] == n and list(bk["lap_hist"][b][:min(n, 16)]) == m.lap_hist[:16], ctx
    return bk


def _check_pools(c, models, bk, cfg):
    """The rows of every selected slot, every used slot and the addPoint target equal the model's lap bit for bit."""
    _, ss_cap, _, model_cap = cfg
    r = _Records(c)
    sx, su = r.view("ss_x", np.float64, (ss_cap, TMAX, 6)), r.view("ss_u", np.float64, (ss_cap, TMAX, 2))
    sq, sl = r.view("ss_q", np.float64, (ss_cap, TMAX)), r.view("ss_len", np.int32, (ss_cap,))
    mx, mu = r.view("model_x", np.float64, (model_cap, TMAX, 6)), r.view("model_u", np.float64, (model_cap, TMAX, 2))
    ml = r.view("model_len", np.int32, (model_cap,))
    for b, m in enumerate(models):
        if m.dead or m.it < 1:
            continue
        for s in set(bk["sel"][b]) | {bk["prev_slot"][b]}:
            x, u, q = m.ss_rows[bk["ss_lap"][b][s]]
            T = x.shape[0]
            assert sl[b, s] == T, (b, s)
            assert np.array_equal(sx[b, s, :T], x) and np.array_equal(su[b, s, :T], u) and np.array_equal(sq[b, s, :T], q), (b, s)
        by_seq = m.md_by_seq()
        for s in set(bk["used"][b]):
            x, u = by_seq[bk["md_seq"][b][s]][1]
            T = x.shape[0]
            assert ml[b, s] == T and np.array_equal(mx[b, s, :T], x) and np.array_equal(mu[b, s, :T], u), (b, s)


def _own_round(c, models, rng, lengths, lap):
    r = _Records(c)
    clx, clu = r.view("cl_x", np.float64, (TCL, 6)), r.view("cl_u", np.float64, (TCL, 2))
    cl_len, done = r.view("cl_len", np.int32, (1,)), r.view("done", np.int32, (1,))
    done[:] = 0
    fin = [b for b in range(B) if not models[b].dead and rng.random() > 0.05]
    for b in fin:
        T = int(lengths[b][lap[b]])
        lap[b] += 1
        x = rng.standard_normal((T, 6))
        x[:, 4] = rng.uniform(0.0, 1.3 * TRACK.TrackLength, T)      # rows past the finish line reset computeCost
        u = rng.standard_normal((T, 2))
        clx[b, :T], clu[b, :T], cl_len[b], done[b] = x, u, T, 1
        models[b].own(T, x, u)
    r.restore(c)
    c.rollout_commit_laps_dev()
    return {b for b in fin if models[b].dead}


def _import_round(c, models, rng, grp):
    """Crafted gathered rows: lap times tying stored laps and own latest laps, other controllers' and foreign gids, the
    importer's own gid, invalid rows (gid < 0, len < 2) mid-ranking, groups outside [0, G), Tpad < len, lt > Tmax, and
    sometimes n_src = 64 G with more than 64 rows in one group."""
    n_src = G * lx.POOL_MAXSRC if rng.random() < 0.3 else int(rng.integers(3, 24))
    share = int(rng.integers(1, 4))
    pool = [t for m in models for t in m.times[-3:]] or [5]
    meta = np.zeros((n_src, 4), np.int32)
    for i in range(n_src):
        lt = int(rng.choice(pool)) if rng.random() < 0.7 else int(rng.integers(1, TCL + 8))
        gid = int(rng.integers(0, B)) if rng.random() < 0.7 else int(rng.choice([-1, B + 3, B + 40]))
        ln = int(rng.integers(0, 2)) if rng.random() < 0.1 else int(rng.integers(lt, lt + 12))
        g = int(rng.integers(0, G)) if rng.random() < 0.9 else int(rng.choice([-1, G, G + 5]))
        if n_src > 64 and i < 70:
            g = 0                                                      # more than 64 rows in group 0
        meta[i] = (ln, lt, gid, g)
    rows = rng.standard_normal((n_src, TPAD, 9))
    order = lx.pool_rank(meta, G)
    dead_before = {b for b, m in enumerate(models) if m.dead}
    filed = 0
    for b, m in enumerate(models):
        for i in lx.pool_pick(order[grp[b]], meta, b, share):
            if m.dead:
                break
            filed += m.imp(int(meta[i, 1]), int(meta[i, 0]), rows[i], TPAD) == "filed"
    took = c.pool_import(n_src, share, TPAD, 0, torch.from_numpy(rows).to("cuda"), torch.from_numpy(meta).to("cuda"), count=True)
    fresh = {b for b, m in enumerate(models) if m.dead} - dead_before
    if not any(m.dead for m in models):                # a controller past flag 64 is no longer followed, its imports included
        assert took == filed
    return fresh


@pytest.mark.parametrize("cfg", GRID, ids=lambda c: "nit%d_ss%d_tr%d_md%d" % c)
def test_device_books_follow_the_unbounded_lists_event_by_event(cfg):
    _need_gpu()
    rng = np.random.default_rng(1000 + GRID.index(cfg))
    c = _controller(cfg, B)
    grp = np.arange(B) % G
    c.set_pool_groups(grp, G)
    models = [lx.Books(*cfg, Tmax=TMAX, TrackLength=TRACK.TrackLength) for _ in range(B)]
    lengths = [_lap_lengths(rng, b % 6, ROUNDS + 1) for b in range(B)]
    lap = [0] * B
    filed_any = dropped_any = 0
    for r in range(ROUNDS):
        if r % XEVERY == 0:
            before = [m.seq - m.it for m in models]
            fresh = _import_round(c, models, rng, grp)
            bk = _check_books(c, models, fresh)
            dropped_any += sum((m.seq - m.it) > x for m, x in zip(models, before))
            filed_any += int(bk["it"].sum())
        fresh = _own_round(c, models, rng, lengths, lap)
        bk = _check_books(c, models, fresh)
        if r % 5 == 4:
            _check_pools(c, models, bk, cfg)
    if cfg == (4, 4, 4, 4):
        assert any(m.dead for m in models)              # the tightest tables raise flag 64
    else:
        assert max(len(m.lap_hist) for m in models) >= 44
        assert dropped_any > 0                          # imports the safe set dropped reached the model list
    c.close()


def test_books_set_derives_the_selection_and_the_export_ships_the_chosen_laps():
    """B = 1100 (the 1024-thread loop of pool_local_best_kernel takes a second pass), three pool groups, tied lap times across
    controllers, controllers with no lap, kbest above the eligible laps of a group, min_overrun at the boundary and one row
    short, a ship mask.  The books go in through lmpc_books_set, which must derive sel, is_prev, prev_slot and used itself."""
    _need_gpu()
    cfg, Bx, Tmax, Tpad, kbest = (4, 7, 4, 5), 1100, 32, 24, 8
    numSS_it, ss_cap, trToUse, model_cap = cfg
    rng = np.random.default_rng(99)
    c = _controller(cfg, Bx, Tmax=Tmax, Tcl=Tmax)
    grp = np.where(np.arange(Bx) < 600, 0, np.where(np.arange(Bx) < 1090, 1, 2)).astype(np.int32)
    c.set_pool_groups(grp, 3)
    ss_time = np.full((Bx, ss_cap), INT_MAX, np.int32); ss_lap = -np.ones((Bx, ss_cap), np.int32)
    md_time = np.full((Bx, model_cap), INT_MAX, np.int32); md_seq = -np.ones((Bx, model_cap), np.int32)
    it = np.zeros(Bx, np.int32); md_cnt = np.zeros(Bx, np.int32)
    r = _Records(c)
    sx, su = r.view("ss_x", np.float64, (ss_cap, Tmax, 6)), r.view("ss_u", np.float64, (ss_cap, Tmax, 2))
    sq, sl = r.view("ss_q", np.float64, (ss_cap, Tmax)), r.view("ss_len", np.int32, (ss_cap,))
    models, rows_of, over = [], {}, np.zeros(Bx, int)
    for b in range(Bx):
        m = lx.Books(*cfg, Tmax=Tmax)
        nl = 0 if b % 97 == 5 else int(rng.integers(4, 7))             # some controllers have no lap
        slots = rng.permutation(ss_cap)[:nl]
        for j in range(nl):
            T = int(rng.integers(5, 8)) if b < 1090 else int(rng.integers(18, 21))
            m.own(T)
            ss_time[b, slots[j]], ss_lap[b, slots[j]] = T, j
        for j in range(min(nl, model_cap)):
            md_time[b, j], md_seq[b, j] = m.md[j][0], m.md[j][1]      # the model list's first laps, ascending
        it[b], md_cnt[b] = nl, min(nl, model_cap)
        if nl:                                         # lap it-1 with `over` rows past its finish line (addPoint's rows)
            s, T = slots[nl - 1], m.times[nl - 1]
            over[b] = int(rng.choice([0, 2, 3, 5])) if b < 1090 else (0, 2, 3, 11)[b % 4]
            n = T + over[b]
            x, u, q = rng.standard_normal((n, 6)), rng.standard_normal((n, 2)), rng.standard_normal(n)
            sx[b, s, :n], su[b, s, :n], sq[b, s, :n], sl[b, s] = x, u, q, n
            rows_of[b] = (x, u, q)
        models.append(m)
    r.restore(c)                                       # stored rows only: the restored books are still the empty ones
    nat.check(c._lib.lmpc_books_set(c._h, nat.ptr(ss_time), nat.ptr(ss_lap), nat.ptr(it), nat.ptr(md_time), nat.ptr(md_seq),
                                    nat.ptr(md_cnt)))
    bk = c.books()
    for b in range(Bx):
        m = models[b]
        if m.it == 0:
            assert bk["prev_slot"][b] == -1
            continue
        assert [ss_lap[b][s] for s in bk["sel"][b]] == m.sel()[0], b
        assert list(bk["is_prev"][b]) == m.is_prev() and ss_lap[b][bk["prev_slot"][b]] == m.it - 1, b
        stored = sorted((int(md_time[b, j]), int(md_seq[b, j])) for j in range(md_cnt[b]))
        assert [md_seq[b][u] for u in bk["used"][b]] == [s for _, s in stored][:trToUse] + \
            [stored[-1][1]] * (trToUse - len(stored)), b
    dev = torch.device("cuda", 0)
    for min_over, ship in ((0, None), (3, None), (3, [1, 0, 1])):
        c.set_pool_min_overrun(min_over)
        rows = torch.zeros(3 * kbest, Tpad, 9, dtype=torch.float64, device=dev)
        meta = torch.zeros(3 * kbest, 4, dtype=torch.int32, device=dev)
        c.pool_export(kbest, Tpad, 0, rows, meta, groups=ship)
        rows, meta = rows.cpu().numpy(), meta.cpu().numpy()
        for g in range(3):
            cands = [(models[b].times[-1], b, rows_of[b][0].shape[0]) for b in range(Bx) if grp[b] == g and models[b].it]
            best = lx.pool_local_best(cands, kbest, Tpad, min_over) if ship is None or ship[g] else [-1] * kbest
            if g == 2 and min_over == 3:
                assert best[-1] == -1                   # kbest above the eligible laps: -1 rows are shipped
            for j, b in enumerate(best):
                row = g * kbest + j
                if b < 0:
                    assert list(meta[row]) == [0, INT_MAX, -1, g] and not rows[row].any(), (min_over, g, j)
                    continue
                x, u, q = rows_of[b]
                T = min(x.shape[0], Tpad)
                assert list(meta[row]) == [T, models[b].times[-1], b, g], (min_over, g, j)
                want = np.zeros((Tpad, 9))
                want[:T, 0:6], want[:T, 6:8], want[:T, 8] = x[:T], u[:T], q[:T]
                assert np.array_equal(rows[row], want), (min_over, g, j)
    c.close()
