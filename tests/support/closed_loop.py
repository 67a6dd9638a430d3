"""Device closed loops of the per-controller GPU tests (tests/test_gpu_vehicle_sets.py, tests/test_gpu_track_sets.py).

``run`` drives one handle through the reference's whole program on the device -- PID lap, seeding, LMPC laps -- with any
combination of per-controller QP parameters, vehicles and tracks installed, and returns what the run left behind; ``same``
asserts that two such runs agree bit for bit on the chosen controllers.
"""
import ctypes as C

import numpy as np

from racinglmpc_b200 import reference_params as rp
from racinglmpc_b200 import _native as nat
from racinglmpc_b200.controller import BatchedController
from racinglmpc_b200.reference_params import TrackParams

N = 12
X0 = np.array([0.5, 0, 0, 0, 0, 0.0])

# what run() returns per controller: end state, lap books and health counters
KEYS = ("x", "xglob", "done", "cl_len", "lap_hist", "lap_n", "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt", "flags", "unsolved")


def controller(B, track=None, par=None, qts=None, trToUse=4, ss_cap=7, model_cap=5, Tmax=1280):
    """A controller created with `track` (default: the reference's L track) through lmpc_store_create."""
    numSS_it, numSS_Points, _, _, Qts, base = rp.lmpc_params(N)
    track = TrackParams.l_shaped() if track is None else track
    return BatchedController(base if par is None else par, B, track.seg_table, track.TrackLength, trToUse=trToUse,
                             numSS_Points=numSS_Points, numSS_it=numSS_it, QterminalSlack=Qts if qts is None else qts,
                             Tmax=Tmax, ss_cap=ss_cap, model_cap=model_cap)


def run(B, track=None, tracks=None, tidx=None, vehicles=None, vidx=None, par=None, qts=None, psets=None, steps=None,
        trace=False, hook=None):
    """Device PID lap (Philox), seeding, then LMPC rollout steps until every controller has finished one LMPC lap (or `steps`
    steps).  `hook(c)` runs once the tables are installed; `trace` traces controllers 0-3.  Returns (steps, run, laps): the
    KEYS of every controller and the stored safe-set laps of every fifth one."""
    c = controller(B, track=track, par=par, qts=qts)
    if psets is not None:
        c.set_param_sets(*psets)
    if vehicles is not None:
        c.set_vehicles(vehicles, vidx)
    if tracks is not None:
        c.set_tracks(tracks, tidx)
    if hook is not None:
        hook(c)
    c.enable_rollout(Tcl=1024)
    if trace:
        inst = np.array([0, 1, 2, 3], np.int32)
        nat.check(nat.lib().lmpc_rollout_trace_create(c._h, len(inst), nat.ptr(inst), 16))
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    for _ in range(1000):
        c.rollout_pid_step(0.8, seed=4321)
    c.rollout_seed_from_record_dev(copies=4)
    c.rollout_set_state(np.tile(X0, (B, 1)), np.tile(X0, (B, 1)))
    n = 0
    while (steps is None and n < 1200) or (steps is not None and n < steps):
        c.rollout_step(seed=1234)
        c.rollout_commit_laps_dev()
        n += 1
        if steps is None and n % 8 == 0 and c.rollout_stats()[0] >= 1:
            break
    bk = c.books()
    flags, unsolved = c.rollout_health()
    st = c.rollout_state()
    laps = {}
    for b in range(0, B, 5):                        # stored safe-set laps of every fifth controller
        for slot in range(7):
            T = C.c_int(0)
            x, u, q = np.zeros((1280, 6)), np.zeros((1280, 2)), np.zeros(1280)
            nat.check(nat.lib().lmpc_ss_get_lap(c._h, b, slot, C.byref(T), nat.ptr(x), nat.ptr(u), nat.ptr(q)))
            laps[(b, slot)] = (x[:T.value].copy(), u[:T.value].copy(), q[:T.value].copy())
    c.close()
    return n, dict(bk, flags=flags, unsolved=unsolved, **st), laps


def same(a, b, sel, what):
    """(run, laps) pairs a and b agree bit for bit on the controllers selected by the boolean mask `sel`."""
    a_run, a_laps = a
    b_run, b_laps = b
    for key in KEYS:
        assert np.array_equal(a_run[key][sel], b_run[key][sel]), (what, key)
    for (i, slot), v in a_laps.items():
        if sel[i] and (i, slot) in b_laps:
            assert all(np.array_equal(p, q) for p, q in zip(v, b_laps[(i, slot)])), (what, i, slot)
