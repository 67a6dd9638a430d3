"""GPU tier: controller snapshots (lmpc_snapshot_pack_dev / lmpc_snapshot_unpack_dev, BatchedController.snapshot / restore /
clone, rollout_mc.run(capture=..., start=...)).

A handle restored from another's records into buffers that held a different experiment drives on bit for bit like the
original, through a lap hand-over, with and without warm start and with a trace on the destination: the carried buffers are
the whole state.  Re-packing returns the records unpacked; clones inside a handle stay identical under equal draws; a broadcast
equals separate unpacks; a record drives whatever car the destination has.  Every refusal (layout, track, corrupted field,
repeated destination) leaves the handle exactly as it was.  A run captured at 3 laps and resumed to 5 equals a run to 5."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import reference_params as rp                 # noqa: E402
from racinglmpc_b200 import _native as nat                         # noqa: E402
from racinglmpc_b200.controller import BatchedController           # noqa: E402
from racinglmpc_b200.reference_params import TrackParams, VehicleParams   # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LMPC_E_INVALID, LMPC_E_STATE = -1, -4
N = 12
X0 = np.array([0.5, 0, 0, 0, 0, 0.0])
L_TRACK = TrackParams.l_shaped()


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _ctrl(B, warm=False, Tmax=1280, ss_cap=7, track=L_TRACK, Tcl=1024):
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
    c = BatchedController(par, B, track.seg_table, track.TrackLength, trToUse=4, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=Tmax, ss_cap=ss_cap, model_cap=5, warm_start=warm)
    if Tcl:
        c.enable_rollout(Tcl=Tcl)
    return c


def _seeded(B, pid_seed=4321, **kw):
    """PID lap (Philox) and device seeding: ready for LMPC steps."""
    c = _ctrl(B, **kw)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=pid_seed)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    return c


def _steps(c, n, seed=1234, z=None):
    for k in range(n):
        c.rollout_step(seed=seed, z=None if z is None else z(k))
        c.rollout_commit_laps_dev()


def _view(c):
    """Everything a caller can read per controller: books, closed loop, health, the last step's solver report, stored laps."""
    out = dict(c.books(), **c.rollout_state())
    out["flags_or"], out["unsolved"] = c.rollout_health()
    for k, v in c.step_results().items():
        out["step_" + k] = v
    L = nat.lib()
    for b in range(c.B):
        for slot in range(c.ss_cap):
            T = C.c_int(0)
            x, u, q = np.zeros((c.Tmax, 6)), np.zeros((c.Tmax, 2)), np.zeros(c.Tmax)
            nat.check(L.lmpc_ss_get_lap(c._h, b, slot, C.byref(T), nat.ptr(x), nat.ptr(u), nat.ptr(q)))
            out["lap_%d_%d" % (b, slot)] = np.concatenate([x[:T.value].ravel(), u[:T.value].ravel(), q[:T.value]])
    return out


def _same(a, b, what):
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.shape == y.shape and np.array_equal(x, y), (what, k)


def _sect(rec_row, name):
    off, nb = nat.decode_snapshot_header(rec_row[:C.sizeof(nat.SnapshotHeader)])["sections"][name]
    return off, nb


@pytest.mark.parametrize("warm,B", [(False, 12), (True, 12), (False, 5)])
def test_round_trip_into_a_dirty_handle(warm, B):
    """A learns (PID lap, seeding, 100 LMPC steps); B, same layout, runs another experiment first (other seeds, another car, a
    trace, 151 steps: its simulator double buffer is on the other half).  After pack(A) -> unpack(B), B's tables set to A's and the
    clock copied, 260 more steps of both give bit-identical books, stored laps, end states, health, solver reports and records,
    through a lap hand-over.  An odd batch puts buffers carved out of a larger allocation (the lap history) off 16-byte
    alignment."""
    _need_gpu()
    a = _seeded(B, warm=warm)
    _steps(a, 100)
    b = _seeded(B, pid_seed=99, warm=warm)
    b.set_vehicles([VehicleParams.from_friction(0.6)], np.zeros(B, np.int32))
    inst = np.array([0, B // 2, B - 1], np.int32)
    nat.check(nat.lib().lmpc_rollout_trace_create(b._h, len(inst), nat.ptr(inst), 64))
    _steps(b, 151, seed=77)                                      # 1000 + 151 simulator steps against A's 1000 + 100
    rec = a.snapshot()
    assert rec.dtype == torch.uint8 and tuple(rec.shape) == (B, a.snapshot_bytes) and rec.device == torch.device("cuda", 0)
    b.set_vehicles(None)
    b.restore(rec)
    b.rollout_clock = a.rollout_clock
    assert torch.equal(b.snapshot(), rec)                        # re-pack identity
    lap_n0 = a.books()["lap_n"].copy()
    _steps(a, 260)
    _steps(b, 260)
    assert (a.books()["lap_n"] > lap_n0).any()                   # a lap was handed over after the restore
    _same(_view(a), _view(b), "dirty round trip, warm=%s" % warm)
    assert torch.equal(a.snapshot(), b.snapshot())
    a.close(); b.close()


def test_clone_within_a_handle_and_permutation():
    """clone([3] -> [7, 11]) under host draws in which rows 7 and 11 equal row 3 keeps the three bit-identical through a lap
    hand-over; clone(perm -> arange) followed by permuted draws equals the permuted original."""
    _need_gpu()
    B = 16
    rng = np.random.default_rng(5)
    Z = rng.standard_normal((300, B, 3))
    c = _seeded(B)
    _steps(c, 100)
    c.clone([3], [7, 11])
    Zc = Z.copy()
    Zc[:, 7] = Zc[:, 3]
    Zc[:, 11] = Zc[:, 3]
    lap0 = c.books()["lap_n"][3]
    _steps(c, 300, z=lambda k: Zc[k])
    assert c.books()["lap_n"][3] > lap0
    r = c.snapshot([3, 7, 11])
    assert torch.equal(r[0], r[1]) and torch.equal(r[0], r[2])
    c.close()

    perm = rng.permutation(B).astype(np.int32)
    p, q = _seeded(B), _seeded(B)
    _steps(p, 100); _steps(q, 100)
    p.clone(perm, np.arange(B))                                 # controller i <- old controller perm[i]
    _steps(p, 200, z=lambda k: Z[k][perm])
    _steps(q, 200, z=lambda k: Z[k])
    assert torch.equal(p.snapshot(), q.snapshot(perm))
    p.close(); q.close()


def test_broadcast_equals_single_unpacks():
    """rec_of mapping 2 records onto 8 controllers of a 24-controller handle equals 8 single-record unpacks."""
    _need_gpu()
    src = _seeded(8)
    _steps(src, 120)
    recs = src.snapshot([2, 5])
    dst = np.array([1, 3, 4, 9, 10, 15, 20, 22], np.int32)
    rec_of = np.array([0, 1, 1, 0, 0, 1, 0, 1], np.int32)
    h1, h2 = _seeded(24), _seeded(24)
    h1.restore(recs, dst, rec_of)
    for d, r in zip(dst, rec_of):
        h2.restore(recs[r:r + 1], [d])
    assert torch.equal(h1.snapshot(), h2.snapshot())
    assert torch.equal(h1.snapshot(dst), recs[torch.from_numpy(rec_of).long().cuda()])
    for h in (src, h1, h2):
        h.close()


def _unchanged(c, before, what):
    view, rec = before
    _same(view, _view(c), what)
    assert torch.equal(rec, c.snapshot()), what


def _raw_unpack(c, rec, dst=None, rec_of=None):
    dst = np.arange(rec.shape[0], dtype=np.int32) if dst is None else np.asarray(dst, np.int32)
    ro = None if rec_of is None else np.asarray(rec_of, np.int32)
    return nat.lib().lmpc_snapshot_unpack_dev(c._h, nat.ptr(rec), int(rec.shape[0]), int(dst.size), nat.ptr(dst), nat.ptr(ro))


def test_refusals_leave_the_handle_as_it_was():
    """Another Tmax, ss_cap, N or warm setting, another track, a corrupted field, a repeated destination: LMPC_E_INVALID (the
    Python layer raises ValueError first where it can), the handle unchanged (books, state, re-pack)."""
    _need_gpu()
    B = 6
    dst = _seeded(B)
    _steps(dst, 40)
    good = _seeded(B, pid_seed=11)
    _steps(good, 60)
    base = good.snapshot()
    nb = dst.snapshot_bytes
    before = (_view(dst), dst.snapshot())

    def fit(rec):                                               # a foreign record in a buffer of this handle's record size
        out = torch.zeros((rec.shape[0], nb), dtype=torch.uint8, device=rec.device)
        k = min(nb, rec.shape[1])
        out[:, :k] = rec[:, :k]
        return out

    others = [("Tmax", dict(Tmax=1024)), ("ss_cap", dict(ss_cap=6)), ("warm_start", dict(warm=True))]
    for field, kw in others:
        o = _seeded(B, **kw)
        rec = o.snapshot()
        with pytest.raises(ValueError, match=field):
            dst.restore(fit(rec))
        assert _raw_unpack(dst, fit(rec)) == LMPC_E_INVALID
        assert field in nat.lib().lmpc_last_error().decode()
        o.close()
    numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(14)
    o = BatchedController(par, B, L_TRACK.seg_table, L_TRACK.TrackLength, trToUse=4, numSS_Points=numSS_Points, numSS_it=numSS_it,
                          QterminalSlack=Qts, Tmax=1280, ss_cap=7, model_cap=5)
    o.enable_rollout(Tcl=1024)
    o.enable_device_books()
    assert _raw_unpack(dst, fit(o.snapshot())) == LMPC_E_INVALID
    assert "N" in nat.lib().lmpc_last_error().decode()
    o.close()
    _unchanged(dst, before, "after the layout refusals")

    oval = _ctrl(B, track=TrackParams.oval())
    oval.enable_device_books()
    with pytest.raises(nat.NativeError, match="track"):
        oval.restore(base)
    oval.close()

    row = base[0].cpu().numpy()
    hdr = nat.decode_snapshot_header(row[:C.sizeof(nat.SnapshotHeader)])
    lay = dst.snapshot_layout()

    def ints(rec, name, k, v):
        off, _ = _sect(rec, name)
        rec[off + 4 * k:off + 4 * k + 4] = np.frombuffer(np.int32(v).tobytes(), np.uint8)

    corrupt = [("magic", lambda r: r.__setitem__(slice(0, 4), 0)),
               ("version", lambda r: r.__setitem__(slice(4, 8), np.frombuffer(np.int32(7).tobytes(), np.uint8))),
               ("safe-set lap length", lambda r: ints(r, "ss_len", 2, lay["Tmax"] + 1)),
               ("model lap length", lambda r: ints(r, "model_len", 1, -1)),
               ("sel", lambda r: ints(r, "sel", 0, lay["ss_cap"])),
               ("prev_slot", lambda r: ints(r, "prev_slot", 0, lay["ss_cap"])),
               ("used", lambda r: ints(r, "used", 1, lay["model_cap"])),
               ("safe-set lap number", lambda r: ints(r, "ss_lap", 0, 1 << 20)),
               ("model arrival number", lambda r: ints(r, "md_seq", 0, 1 << 20)),
               ("it", lambda r: ints(r, "it", 0, -1)),
               ("lap_n", lambda r: ints(r, "lap_n", 0, -1)),
               ("timeStep", lambda r: ints(r, "timeStep", 0, -3)),
               ("cl_len", lambda r: ints(r, "cl_len", 0, lay["Tcl"] + 1)),
               ("done", lambda r: ints(r, "done", 0, 2)),
               ("is_prev", lambda r: ints(r, "is_prev", 1, 2)),
               ("has_pred", lambda r: ints(r, "has_pred", 0, -1)),
               ("md_cnt", lambda r: ints(r, "md_cnt", 0, -1)),
               ("track row", lambda r: r.__setitem__(slice(C.sizeof(nat.SnapshotHeader) - 8, C.sizeof(nat.SnapshotHeader)), 1))]
    assert hdr["Tcl"] == lay["Tcl"] and hdr["sections"]["ss_len"][1] == 4 * lay["ss_cap"]
    for field, spoil in corrupt:
        bad = base.cpu().numpy().copy()
        spoil(bad[3])
        t = torch.from_numpy(bad).cuda()
        assert _raw_unpack(dst, t) == LMPC_E_INVALID, field
        msg = nat.lib().lmpc_last_error().decode()
        assert ("record 3" in msg and field in msg), (field, msg)
    assert _raw_unpack(dst, base, dst=[0, 1, 1], rec_of=[0, 1, 2]) == LMPC_E_INVALID
    assert _raw_unpack(dst, base, dst=[0, B], rec_of=[0, 1]) == LMPC_E_INVALID
    assert _raw_unpack(dst, base, dst=[0, 1], rec_of=[0, B]) == LMPC_E_INVALID
    with pytest.raises(ValueError):
        dst.restore(base, [0, 0])
    _unchanged(dst, before, "after the corrupted records")
    for c in (dst, good):
        c.close()

    # warm start: the destination has stepped (problem type LMPC); the source has not (its records carry no warm problem type)
    wdst = _seeded(B, warm=True)
    _steps(wdst, 20)
    wsrc = _seeded(B, warm=True, pid_seed=5)
    wbase = wsrc.snapshot()
    assert nat.decode_snapshot_header(wbase[0, :C.sizeof(nat.SnapshotHeader)].cpu().numpy())["warm_mode"] == -1
    wbefore = (_view(wdst), wdst.snapshot())
    mode_word = 4 * 14                                          # lmpc_snapshot_header.warm_mode
    for field, spoil in (("warm_valid", lambda r: ints(r, "warm_valid", 0, 1)),     # a valid warm record without a problem type
                         ("warm_mode", lambda r: r.__setitem__(slice(mode_word, mode_word + 4), np.frombuffer(np.int32(5).tobytes(), np.uint8))),
                         ("warm_mode", lambda r: r.__setitem__(slice(mode_word, mode_word + 4), np.frombuffer(np.int32(0).tobytes(), np.uint8)))):
        bad = wbase.cpu().numpy().copy()
        spoil(bad[2])
        assert _raw_unpack(wdst, torch.from_numpy(bad).cuda()) == LMPC_E_INVALID, field
        msg = nat.lib().lmpc_last_error().decode()
        assert ("record 2" in msg and field in msg), (field, msg)
    _unchanged(wdst, wbefore, "after the warm-start refusals")
    wdst.restore(wbase)                                          # records without a problem type fit any handle
    for c in (wdst, wsrc):
        c.close()


def test_a_record_drives_the_destination_car_and_fixes_the_tracks():
    """A record restored onto a controller with another car drives that car: equal to restoring first and installing the car
    after.  After an unpack lmpc_set_tracks returns LMPC_E_STATE."""
    _need_gpu()
    B = 8
    src = _seeded(B)
    _steps(src, 100)
    rec, clock = src.snapshot(), src.rollout_clock
    mu = [VehicleParams.from_friction(0.6)]
    p = _ctrl(B)
    p.set_vehicles(mu, np.zeros(B, np.int32))
    p.restore(rec)
    q = _ctrl(B)
    q.restore(rec)
    q.set_vehicles(mu, np.zeros(B, np.int32))
    for h in (p, q):
        h.rollout_clock = clock
    _steps(p, 150); _steps(q, 150); _steps(src, 150)
    assert torch.equal(p.snapshot(), q.snapshot())
    assert not torch.equal(p.snapshot(), src.snapshot())        # the other car drove differently
    sets, idx = nat.make_track_sets([TrackParams.oval()], np.zeros(B, np.int32), B)
    assert nat.lib().lmpc_set_tracks(q._h, sets, 1, nat.ptr(idx)) == LMPC_E_STATE
    # the same circuit installed from a struct with values in its padding and past nseg: still the circuit of the records
    lsets, lidx = nat.make_track_sets([L_TRACK], np.zeros(B, np.int32), B)
    n3 = lsets[0].nseg * 3
    lsets[0].seg[n3:] = [7.0] * (3 * nat.MAX_SEG - n3)
    C.memmove(C.addressof(lsets[0]) + 4, b"\x55\x55\x55\x55", 4)    # the 4 bytes between nseg and seg
    r = _ctrl(B)
    nat.check(nat.lib().lmpc_set_tracks(r._h, lsets, 1, nat.ptr(lidx)))
    r.restore(rec)
    assert torch.equal(r.snapshot(), rec)
    for h in (src, p, q, r):
        h.close()


def _rollout_mc():
    sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
    try:
        import rollout_mc
    finally:
        sys.path.pop(0)
    return rollout_mc


def _mirrored(track_spec):
    s = np.array(track_spec, dtype=float)
    s[:, 1] = -s[:, 1]
    return TrackParams.from_spec(s)


@pytest.mark.parametrize("case", ["independent", "pooled_batch", "three_circuits_group"])
def test_resume_equals_uninterrupted(case):
    """rollout_mc.run at batch 256: 3 laps captured, the handle destroyed, resumed to 5 laps on a fresh handle equals a run to 5
    laps bit for bit: books, end states, health, exchange steps.  The three-circuit case pools per circuit under group readiness
    (the L-shaped circuit, its mirror image, and the L-shaped circuit driven the other way round)."""
    _need_gpu()
    rm = _rollout_mc()
    B = 256
    kw = dict(batch=B, local=0)
    if case == "independent":
        kw["mode"] = "independent"
    elif case == "three_circuits_group":
        spec = TrackParams.l_shaped_spec()
        rev = spec[::-1].copy()
        rev[:, 1] = -rev[:, 1]
        three = [L_TRACK, _mirrored(spec), TrackParams.from_spec(rev)]
        tidx = (np.arange(B) % 3).astype(np.int32)
        kw.update(track_sets=(three, tidx), pool_groups=(tidx, 3), readiness="group")
    fin5, bk5, cap5 = {}, {}, {}
    o5 = rm.run(laps=5, final=fin5, books=bk5, capture=cap5, **kw)      # capture: the exchange steps of every mode
    cap = {}
    o3 = rm.run(laps=3, capture=cap, **kw)
    assert cap["diverged_step"] is None, cap["diverged_step"]
    assert cap["records"].shape[0] == B and cap["steps"] == o3["closed_loop_steps"]
    assert {k: v for k, v in cap["layout"].items() if k != "bytes"} == rm.layout()
    fin, bk, capr = {}, {}, {}
    o = rm.run(laps=5, start=cap, final=fin, books=bk, capture=capr, **kw)
    assert capr["exchange_steps"] == cap5["exchange_steps"], (case, cap5["exchange_steps"], capr["exchange_steps"])
    assert (len(cap5["exchange_steps"][0]) > len(cap["exchange_steps"][0])) == (case != "independent")
    assert torch.equal(capr["records"], cap5["records"])
    assert o["resume_exact"] and o["resumed_from_step"] == cap["steps"]
    assert o["closed_loop_steps"] == o5["closed_loop_steps"]
    for k in bk5:
        assert np.array_equal(np.asarray(bk5[k]), np.asarray(bk[k])), (case, "books", k)
    for k in fin5:
        assert np.array_equal(np.asarray(fin5[k]), np.asarray(fin[k])), (case, "end state", k)
    for k in ("lap_stats_rank0", "instances_with_flags_rank0", "unsolved_steps_rank0", "exchange_steps_per_group_rank0"):
        assert o5.get(k) == o.get(k), (case, k)
    with pytest.raises(ValueError, match="laps"):
        rm.run(laps=3, start=cap, **kw)
