#!/usr/bin/env python
"""Generate tests/golden/vehicle_golden.npz by running the REAL reference Simulator.dynModel on other vehicles.

Run in the build container only (needs /root/reference; the GPU box has no copy):
    python tests/golden/make_vehicle_golden.py

SysModel.py hard-codes its vehicle in ten assignments at the top of Simulator.dynModel (SysModel.py:61-70).  For every vehicle
under test this script parses SysModel.py with ``ast``, replaces the right-hand sides of those ten assignments by the vehicle's
values, compiles the result IN MEMORY (nothing of the reference is written anywhere) and records dynModel's two outputs on 16
states (straight and curved segments, ey != 0, vy, wz != 0) with fixed noise draws.  The test-side restatement for any vehicle
(tests/support/vehicle_model.py) is checked against it bit for bit on the way.
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

import vehicle_model as vm                                # noqa: E402
from oracle.track import TrackTable                       # noqa: E402
from racinglmpc_b200.reference_params import VehicleParams  # noqa: E402

FIELDS = vm.VEHICLE_FIELDS


def vehicles():
    """The reference; friction 0.5 and 1.1; heavy and light cars; another axle split; other tyre shapes; front/rear friction apart."""
    ref = VehicleParams.reference()
    f = VehicleParams.from_friction
    split = f(0.8)
    return [ref, f(0.5), f(1.1), f(0.8, m=2.6, Iz=0.032), f(0.8, m=1.5, Iz=0.018), f(0.8, lf=0.10, lr=0.15),
            f(0.8, Cf=1.4, Bf=1.3, Cr=1.1, Br=0.8),
            VehicleParams(split.m, split.lf, split.lr, split.Iz, 0.9 * split.m * 9.81 / 2.0, split.Cf, split.Bf,
                          0.6 * split.m * 9.81 / 2.0, split.Cr, split.Br)]


def states(track):
    """16 (x, x_glob, u): s across the whole track (straights and curves), lateral offsets, side slip and yaw rate."""
    rng = np.random.default_rng(11)
    s = np.linspace(0.3, track.TrackLength - 0.6, 16)
    x = np.zeros((16, 6)); g = np.zeros((16, 6)); u = np.zeros((16, 2))
    x[:, 0] = rng.uniform(0.6, 1.8, 16)
    x[:, 1] = rng.uniform(-0.15, 0.15, 16)
    x[:, 2] = rng.uniform(-0.8, 0.8, 16)
    x[:, 3] = rng.uniform(-0.2, 0.2, 16)
    x[:, 4] = s
    x[:, 5] = rng.uniform(-0.3, 0.3, 16)
    g[:, 0:3] = x[:, 0:3]
    g[:, 3] = rng.uniform(-np.pi, np.pi, 16)
    g[:, 4:6] = rng.uniform(-3.0, 3.0, (16, 2))
    u[:, 0] = rng.uniform(-0.4, 0.4, 16)
    u[:, 1] = rng.uniform(-1.0, 1.0, 16)
    return x, g, u


def patched_simulator(src, path, veh):
    """SysModel.Simulator with the ten vehicle assignments of dynModel replaced by ``veh``'s values."""
    tree = ast.parse(src, path)
    sim = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "Simulator")
    dyn = next(n for n in sim.body if isinstance(n, ast.FunctionDef) and n.name == "dynModel")
    done = set()
    for st in dyn.body:
        if isinstance(st, ast.Assign) and len(st.targets) == 1 and isinstance(st.targets[0], ast.Name) and st.targets[0].id in FIELDS:
            name = st.targets[0].id
            assert name not in done, name
            st.value = ast.copy_location(ast.Constant(float(getattr(veh, name))), st.value)
            done.add(name)
    assert done == set(FIELDS), done
    mod = types.ModuleType("SysModel_patched")
    mod.__file__ = path
    exec(compile(ast.fix_missing_locations(tree), path, "exec"), mod.__dict__)
    return mod.Simulator


def main():
    for sub in ("fnc/simulator", "fnc", ""):
        sys.path.append(os.path.join(REF, sub))
    import Track as TR
    path = os.path.join(REF, "fnc/simulator/SysModel.py")
    src = open(path).read()
    rmap, omap = TR.Map(0.4), TrackTable(0.4)
    assert rmap.TrackLength == omap.TrackLength
    x, g, u = states(omap)
    vs = vehicles()
    V, S = len(vs), x.shape[0]
    z = np.zeros((V, S, 3))
    xn = np.zeros((V, S, 6)); gn = np.zeros((V, S, 6))
    for k, veh in enumerate(vs):
        Sim = patched_simulator(src, path, veh)(rmap)
        for i in range(S):
            np.random.seed(1000 * k + i)
            z[k, i] = [np.random.randn() for _ in range(3)]
            np.random.seed(1000 * k + i)
            a, b = Sim.dynModel(x[i].copy(), g[i].copy(), u[i].copy())
            xn[k, i], gn[k, i] = a, b
            draws = iter(z[k, i])
            oa, ob = vm.dyn_model(omap, x[i], g[i], u[i], veh, rng=types.SimpleNamespace(standard_normal=lambda: next(draws)))
            assert np.array_equal(oa, a) and np.array_equal(ob, b), (k, i, np.abs(oa - a).max(), np.abs(ob - b).max())
    # the reference vehicle through the unpatched module as well: row 0 is SysModel.py's own car
    import SysModel as SM
    for i in range(S):
        np.random.seed(i)
        a, b = SM.Simulator(rmap).dynModel(x[i].copy(), g[i].copy(), u[i].copy())
        np.random.seed(i)
        pa, pb = patched_simulator(src, path, vs[0])(rmap).dynModel(x[i].copy(), g[i].copy(), u[i].copy())
        assert np.array_equal(a, pa) and np.array_equal(b, pb), i
    vt = np.array([[getattr(v, f) for f in FIELDS] for v in vs])
    np.savez_compressed(os.path.join(OUT, "vehicle_golden.npz"), vehicles=vt, fields=np.array(FIELDS), x=x, x_glob=g, u=u, z=z,
                        x_next=xn, x_glob_next=gn)
    print("wrote", os.path.join(OUT, "vehicle_golden.npz"), "%d vehicles x %d states" % (V, S))
    print("spread of x_next over the vehicles (max over states):", np.abs(xn - xn[0]).max(axis=(1, 2)))


if __name__ == "__main__":
    main()
