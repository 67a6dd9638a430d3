#!/usr/bin/env python
"""Generate tests/golden/track_golden.npz by running the REAL reference Map and Simulator.dynModel on the three circuits of
Track.py: the L-shaped track it drives (Track.py:30-40), the goggle-shaped track (Track.py:15-28) and the oval (Track.py:43-48).

Run in the build container only (needs /root/reference; the GPU box has no copy):
    python tests/golden/make_track_golden.py

Map.__init__ builds its table from one `spec` assignment (the other two circuits are commented out).  For every circuit this
script parses Track.py with ``ast``, replaces the right-hand side of that assignment by a name bound to the circuit's spec,
compiles the result IN MEMORY (nothing of the reference is written anywhere) and records:
  - PointAndTangent and TrackLength;
  - Map.curvature and Map.getGlobalPosition at 64 s values (segment starts, interiors, the lap end, values beyond one lap and
    a negative one), NaN and ok = 0 where the reference raises;
  - Simulator.dynModel (the reference's own SysModel on the patched Map) on 16 states with fixed noise draws.
The test-side restatements (reference_params.TrackParams.from_spec, tests/support/track_model.py, vehicle_model.dyn_model) are
checked against it bit for bit on the way.
"""
import ast
import os
import sys
import types
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "support"))
REF = "/root/reference/src"
OUT = os.path.dirname(os.path.abspath(__file__))

import track_model                                                       # noqa: E402
import vehicle_model as vm                                               # noqa: E402
from racinglmpc_b200.reference_params import TrackParams, VehicleParams  # noqa: E402

NAMES = ("l_shaped", "goggle", "oval")
SPECS = (TrackParams.l_shaped_spec(), TrackParams.goggle_spec(), TrackParams.oval_spec())
NS, NX = 64, 16


def patched_map(src, path, spec):
    """Track.Map whose __init__ builds its table from ``spec``."""
    tree = ast.parse(src, path)
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "Map")
    init = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "__init__")
    hits = [st for st in init.body if isinstance(st, ast.Assign) and len(st.targets) == 1
            and isinstance(st.targets[0], ast.Name) and st.targets[0].id == "spec"]
    assert len(hits) == 1, len(hits)
    hits[0].value = ast.copy_location(ast.Name(id="_GOLDEN_SPEC", ctx=ast.Load()), hits[0].value)
    mod = types.ModuleType("Track_patched")
    mod.__file__ = path
    exec(compile(ast.fix_missing_locations(tree), path, "exec"), mod.__dict__)
    mod._GOLDEN_SPEC = np.array(spec)
    return mod.Map


def s_points(P, L, rng):
    """64 s values: every segment start, segment interiors, 0, the lap end, values beyond one and two laps, one negative."""
    starts = list(P[:, 3])
    mids = list(P[:, 3] + 0.5 * P[:, 4])
    fixed = [0.0, L, -0.1, L + 0.25, 2 * L + 1.0, L + starts[min(2, len(starts) - 1)]]
    s = starts + mids + fixed
    s += list(rng.uniform(0.0, 3 * L, NS - len(s)))
    return np.array(s[:NS])


def states(L, rng):
    """16 (x, x_glob, u) across the whole circuit (straights and curves), lateral offsets, side slip and yaw rate."""
    s = np.linspace(0.3, L - 0.6, NX)
    x = np.zeros((NX, 6)); g = np.zeros((NX, 6)); u = np.zeros((NX, 2))
    x[:, 0] = rng.uniform(0.6, 1.8, NX)
    x[:, 1] = rng.uniform(-0.15, 0.15, NX)
    x[:, 2] = rng.uniform(-0.8, 0.8, NX)
    x[:, 3] = rng.uniform(-0.2, 0.2, NX)
    x[:, 4] = s
    x[:, 5] = rng.uniform(-0.3, 0.3, NX)
    g[:, 0:3] = x[:, 0:3]
    g[:, 3] = rng.uniform(-np.pi, np.pi, NX)
    g[:, 4:6] = rng.uniform(-3.0, 3.0, (NX, 2))
    u[:, 0] = rng.uniform(-0.4, 0.4, NX)
    u[:, 1] = rng.uniform(-1.0, 1.0, NX)
    return x, g, u


def main():
    for sub in ("fnc/simulator", "fnc", ""):
        sys.path.append(os.path.join(REF, sub))
    import SysModel as SM
    import Track as TR
    path = os.path.join(REF, "fnc/simulator/Track.py")
    src = open(path).read()
    rng = np.random.default_rng(17)
    out = {}
    for k, (name, spec) in enumerate(zip(NAMES, SPECS)):
        rmap = patched_map(src, path, spec)(0.4)
        P, L = rmap.PointAndTangent, rmap.TrackLength
        mine = TrackParams.from_spec(spec)
        assert np.array_equal(mine.table6, P) and mine.TrackLength == L, name
        if name == "l_shaped":
            orig = TR.Map(0.4)
            assert np.array_equal(orig.PointAndTangent, P) and orig.TrackLength == L
        tm = track_model.from_table(P)
        s = s_points(P, L, rng)
        ey = rng.uniform(-0.3, 0.3, NS)
        cur = np.full(NS, np.nan); xy = np.full((NS, 2), np.nan); ok_c = np.zeros(NS, np.int32); ok_g = np.zeros(NS, np.int32)
        for i in range(NS):
            try:
                cur[i] = rmap.curvature(s[i]); ok_c[i] = 1
            except Exception:
                pass
            try:
                xy[i] = rmap.getGlobalPosition(s[i], ey[i]); ok_g[i] = 1
            except Exception:
                pass
        x, g, u = states(L, rng)
        z = np.zeros((NX, 3)); xn = np.zeros((NX, 6)); gn = np.zeros((NX, 6))
        sim = SM.Simulator(rmap)
        for i in range(NX):
            np.random.seed(1000 * k + i)
            z[i] = [np.random.randn() for _ in range(3)]
            np.random.seed(1000 * k + i)
            xn[i], gn[i] = sim.dynModel(x[i].copy(), g[i].copy(), u[i].copy())
            draws = iter(z[i])
            a, b = vm.dyn_model(tm, x[i], g[i], u[i], VehicleParams.reference(),
                                rng=types.SimpleNamespace(standard_normal=lambda: next(draws)))
            assert np.array_equal(a, xn[i]) and np.array_equal(b, gn[i]), (name, i)
        out.update({name + "_table": P, name + "_length": np.array(L), name + "_s": s, name + "_ey": ey, name + "_curvature": cur,
                    name + "_curvature_ok": ok_c, name + "_xy": xy, name + "_xy_ok": ok_g, name + "_x": x, name + "_x_glob": g,
                    name + "_u": u, name + "_z": z, name + "_x_next": xn, name + "_x_glob_next": gn})
        print(name, "rows", P.shape[0], "TrackLength %.17g" % L, "raises", int((ok_c == 0).sum()), int((ok_g == 0).sum()))
    np.savez_compressed(os.path.join(OUT, "track_golden.npz"), **out)
    print("wrote", os.path.join(OUT, "track_golden.npz"))


if __name__ == "__main__":
    main()
