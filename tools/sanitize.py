#!/usr/bin/env python
"""Small-batch run of every kernel for compute-sanitizer (memcheck / racecheck / synccheck / initcheck):
    compute-sanitizer --tool racecheck python tools/sanitize.py
Exercises: ftocp_kernel<12,0> and <12,48> (host + device entry points), knn_ltv_regress, ss_select, shift_state,
ss_add_point, rollout_cost, sim_step (with noise sets and noise streams), measure (with measurement sets), knn_ltv_regress with regression sets, commit_laps, ss_export_laps, ss_import_laps; round 2: the long-horizon kernel
that reads its model in place (N = 48), warm-started solves, pid_input, seed_books, commit_laps_books, rollout_stats, the pooled
exchange (pool_local_best / export / rank / import), trace_step and track_global_position, and a controller made
non-finite in the closed loop (ss_select on a NaN terminal guess, ss_add_point refusing the point), all with per-lap reports on
(the report paths of sim_step, seed_books and commit_laps_books, lap_reports_reset)."""
import os
import sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from racinglmpc_b200 import BatchedFTOCP, workloads, reference_params as rp
from racinglmpc_b200.controller import BatchedController

B, N = 8, 12
x0, uold, abc = workloads.ltv_mpc_batch(B, N=N)
s = BatchedFTOCP(rp.mpc_params(N), batch=B)
o = s.solve(x0, uold, abc)
assert np.all(o["status"] == 1)
s.close()
data = workloads.lmpc_batch(B)
numSS_it, numSS_Points, _, _, Qts, par = rp.lmpc_params(N)
c = BatchedController(par, B, workloads.track_seg_table(), rp.TRACK_LENGTH, trToUse=5, numSS_Points=numSS_Points,
                      numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1280, ss_cap=8, model_cap=7)
workloads.restore_lmpc_batch(c, data)
o = c.step(data["x0"])
assert np.all(o["status"] == 1) and np.all(o["flags"] == 0)
c.add_point(data["x0"], o["uPred"][:, 0])
c.enable_rollout(Tcl=64)
c.rollout_set_state(data["x0"], data["x0"])
# per-controller noise sets and shared noise streams: the simulator reads its row and its stream per controller
c.set_noise([rp.NoiseParams.reference(), rp.NoiseParams.scaled(10, 0.5)], np.arange(B) % 2)
c.set_noise_streams(np.arange(B) // 2)
# per-controller measurement noise: measure_kernel reads its row and its stream, the QP, addPoint and the record read its output
c.set_measurement_noise([rp.MeasurementParams.zero(), rp.MeasurementParams((0.01,) * 6, (0.05,) * 6)], np.arange(B) % 2)
# per-controller regression sets: K1 stages its row per warp; fewer laps, other h / MaxNumPoint / lamb / scaling per controller
r = rp.RegressionParams.reference(5)
c.set_regression([r, rp.RegressionParams(2, 3, 0.5, 1e-6, (2.0 ** 32, 1.0, 0.0, 1.0, -(2.0 ** -32)))], np.arange(B) % 2)
for _ in range(3):
    c.rollout_step(seed=1)
done, n = c.rollout_done()
c.rollout_finish_laps(np.array([1] + [0] * (B - 1), np.int32), n)
c.sync()
# pooled-safe-set exchange: export a stored lap of every instance, hand instance 0's lap to the others
lens = torch.zeros(B, dtype=torch.int32, device="cuda")
rows9 = torch.zeros(B, 512, 9, dtype=torch.float64, device="cuda")
c.export_laps([1] * B, 512, rows9, lens)
took = c.import_laps(np.array([-1] + [0] * (B - 1)), np.full(B, 100), 512, rows9, lens)
assert len(took) == B - 1
o = c.step(data["x0"])
# instance 0 was handed a fake 3-row lap above (flag 8: selection window past the lap end); all others must be clean
assert np.all(o["status"][1:] == 1) and np.all(o["flags"][1:] == 0), (o["status"], o["flags"])
f, n_uns = c.rollout_health()
r = c.step_results()
c.close()
# ---- round 2 ---------------------------------------------------------------------------------------------------------------
from racinglmpc_b200 import export
x0, uold, abc = workloads.ltv_mpc_batch(4, N=48)
s = BatchedFTOCP(rp.mpc_params(48), batch=4)          # stage model streamed from global memory
o = s.solve(x0, uold, abc)
assert np.all(o["status"] == 1)
s.close()
B = 8
c = BatchedController(par, B, workloads.track_seg_table(), rp.TRACK_LENGTH, trToUse=4, numSS_Points=numSS_Points,
                      numSS_it=numSS_it, QterminalSlack=Qts, Tmax=1280, ss_cap=7, model_cap=5, warm_start=True)
xs = np.tile(np.array([0.5, 0, 0, 0, 0, 0.0]), (B, 1))
c.enable_rollout(Tcl=1024)
c.enable_lap_reports(2)                              # per-lap reports: the report paths of the step, hand-over and seeding
c.rollout_set_state(xs, xs)
c.set_measurement_noise([rp.MeasurementParams((0.01,) * 6, (0.05,) * 6)], np.zeros(B, np.int32))   # the PID lap measures too
for _ in range(int(os.environ.get("SANITIZE_PID_STEPS", "1000"))):
    c.rollout_pid_step(0.8, seed=7)
c.rollout_seed_from_record_dev(copies=4)
c.rollout_set_state(xs, xs)
tr = export.RolloutTrace(c, [0, 3], cap_steps=64)
for _ in range(6):
    c.rollout_step(seed=3)                               # warm-started from the second step on
    c.rollout_commit_laps_dev()
# a controller whose state stops being finite: K2 on its non-finite terminal guess, addPoint refusing its point (flag 512)
st = c.rollout_state()
xb = st["x"].copy()
xb[1, 0] = np.nan
c.rollout_set_state(xb, st["xglob"])
for _ in range(3):
    c.rollout_step(seed=3)
    c.rollout_commit_laps_dev()
assert c.rollout_health()[0][1] & 512
rep = c.lap_reports()                                # the non-finite controller's running row holds viol_max = +inf
print("stats", c.rollout_stats())
rows = torch.zeros(3, 288, 9, dtype=torch.float64, device="cuda")
meta = torch.zeros(3, 4, dtype=torch.int32, device="cuda")
c.pool_export(3, 288, 0, rows, meta)
print("filed", c.pool_import(3, 2, 288, 0, rows, meta, count=True))
c.rollout_step(seed=3)
t = tr.get(0)
gt = np.load(os.path.join(ROOT, "tests", "golden", "track_global.npz"))
xy, ok = export.global_position(gt["table"], float(gt["track_length"]), gt["s"][:32], gt["ey"][:32])
assert np.all(ok[np.isfinite(gt["s"][:32])] >= 0)
c.sync()
c.close()
print("sanitize workload done")
