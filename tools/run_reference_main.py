#!/usr/bin/env python
"""tools/run_reference_main.py — boundary acceptance (SURVEY §7.1 step 2 / §8b): the reference's own `src/main.py`, UNCHANGED,
driven by the drop-in modules of this repository.

main.py imports its controllers by module name from `fnc/controller` (main.py:24-31), so putting a directory with modules named
`PredictiveControllers` / `PredictiveModel` earlier on sys.path swaps the implementation.  Two back ends:

  b200     racinglmpc_b200/compat  (ctypes -> liblmpc_b200.so -> CUDA kernels; needs an H100)
  oracle   tests/support/oracle_compat  (the oracle: reference arithmetic + OSQP-algorithm port at 1e-9; CPU)

Everything else main.py imports (Simulator, Map, PID, Regression, initControllerParameters, plot) is the reference's own code.
The reference tree is NOT part of this repository: `stage` copies /root/reference/src into the git-ignored baseline/_ref/
(which travels to the GPU box with the gpurun snapshot) and writes a matplotlib stub next to it (matplotlib is not installed;
main.py only plots after the laps are printed).  main.py does not seed NumPy; the launcher seeds it (seed 0) before
`runpy`-ing the file so that the two back ends see the same noise.

  python tools/run_reference_main.py stage                  (build container: /root/reference present)
  python tools/run_reference_main.py run --backend oracle   (CPU, ~10 min)  -> gpurun_out/main_py_oracle.json
  python tools/run_reference_main.py run --backend b200     (GPU box)       -> gpurun_out/main_py_b200.json
  python tools/run_reference_main.py compare                 lap-time printouts of the two runs
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGE = os.path.join(ROOT, "baseline", "_ref")
SRC = os.path.join(STAGE, "reference_src")
STUBS = os.path.join(STAGE, "stubs")
OUT = os.path.join(ROOT, "gpurun_out")

_STUB = '''"""matplotlib stand-in for running the reference's main.py headless: every attribute is a callable that returns another one."""
class _Any:
    def __call__(self, *a, **k): return _Any()
    def __getattr__(self, name): return _Any()
    def __iter__(self): return iter([_Any()])          # `line, = ax.plot(...)` (plot.py:132-133)
    def __getitem__(self, i): return _Any()
def __getattr__(name): return _Any()
'''

_LAUNCH = '''import sys, runpy
import numpy as np
np.random.seed(%d)
sys.argv = ["main.py"]
runpy.run_path("main.py", run_name="__main__")
'''


def stage():
    ref = "/root/reference/src"
    if not os.path.isdir(ref):
        raise SystemExit("stage: /root/reference/src is not available here (run this in the build container)")
    if os.path.isdir(SRC):
        shutil.rmtree(SRC)
    shutil.copytree(ref, SRC, ignore=shutil.ignore_patterns("*.gif", "__pycache__"))
    for mod in ("", "pyplot", "animation", "patches"):
        d = os.path.join(STUBS, "matplotlib")
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, (mod or "__init__") + ".py"), "w") as f:
            f.write(_STUB)
    print("staged", SRC, "and the matplotlib stub")


def run(backend, seed, timeout):
    if not os.path.isdir(SRC):
        raise SystemExit("run: no staged reference tree (python tools/run_reference_main.py stage)")
    compat = os.path.join(ROOT, "racinglmpc_b200", "compat") if backend == "b200" else os.path.join(ROOT, "tests", "support", "oracle_compat")
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([compat, STUBS, ROOT])
    p = subprocess.run([sys.executable, "-c", _LAUNCH % seed], cwd=SRC, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=timeout)
    laps = [(int(m.group(1)), float(m.group(2))) for m in re.finditer(r"Lap time at iteration\s+(\d+)\s+is\s+([0-9.]+)", p.stdout)]
    done = [(int(m.group(1)), float(m.group(2))) for m in re.finditer(r"Completed lap:\s+(\d+)\s+in\s+([0-9.]+)", p.stdout)]
    os.makedirs(OUT, exist_ok=True)
    res = {"backend": backend, "seed": seed, "returncode": p.returncode, "lap_times_s": laps, "completed": done, "tail": p.stdout[-1500:]}
    with open(os.path.join(OUT, "main_py_%s.json" % backend), "w") as f:
        json.dump(res, f)
    print("main.py with the %s back end: rc %d, %d laps printed; last lines:" % (backend, p.returncode, len(laps)))
    print("\n".join(p.stdout.strip().splitlines()[-6:]))
    return res


def compare():
    a = json.load(open(os.path.join(OUT, "main_py_b200.json")))
    b = json.load(open(os.path.join(OUT, "main_py_oracle.json")))
    la, lb = dict(a["lap_times_s"]), dict(b["lap_times_s"])
    rows, same = [], 0
    for i in sorted(set(la) | set(lb)):
        rows.append((i, la.get(i), lb.get(i)))
        same += int(la.get(i) == lb.get(i))
    first_diff = next((i for i, x, y in rows if x != y), None)
    print("laps printed: b200 %d, oracle %d; identical lap times: %d; first difference at iteration %s" % (len(la), len(lb), same, first_diff))
    for i, x, y in rows:
        print("  it %2d   b200 %6s s   oracle %6s s%s" % (i, x, y, "" if x == y else "   <-"))
    return rows


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("cmd", choices=["stage", "run", "compare"])
    ap.add_argument("--backend", choices=["b200", "oracle"], default="b200")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--timeout", type=int, default=3000)
    a = ap.parse_args()
    if a.cmd == "stage":
        stage()
    elif a.cmd == "run":
        run(a.backend, a.seed, a.timeout)
    else:
        compare()
