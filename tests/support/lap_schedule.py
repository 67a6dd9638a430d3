"""Host restatement of the lap schedules of the device closed loop (lmpc_rollout_set_lap_schedule, csrc/lap_schedule.cuh).

Given the laps every controller had handed over as each step started (lap_n of the lap books), ``rows_read`` says which row of a
scheduled table every controller reads at every step: row_of_lap[b][min(lap_n, L - 1)], its own index without a schedule or on a
PID step, and nothing (-1) while it is retired by a lap budget.
"""
import numpy as np

RETIRED = -1


def rows_read(lap_n, own, schedule=None, budget=None, pid=None):
    """lap_n [steps, B]: lap_n at the start of every step; own [B]: the table index (set_of_instance); schedule [B, L] or None;
    budget [B] or None; pid [steps] booleans (a PID step reads `own` and retires nobody) or None.  Returns [steps, B] rows."""
    lap_n = np.asarray(lap_n, np.int64)
    steps, B = lap_n.shape
    own = np.broadcast_to(np.asarray(own, np.int64), (B,))
    out = np.empty((steps, B), np.int64)
    for t in range(steps):
        if pid is not None and pid[t]:
            out[t] = own
            continue
        if schedule is None:
            out[t] = own
        else:
            s = np.asarray(schedule)
            out[t] = s[np.arange(B), np.minimum(lap_n[t], s.shape[1] - 1)]
        if budget is not None:
            out[t] = np.where(lap_n[t] >= np.asarray(budget), RETIRED, out[t])
    return out


def host_switch_index(lap_n, schedule):
    """The set_of_instance a host re-installs to mimic a schedule from lap_n: row_of_lap[b][min(lap_n[b], L - 1)]."""
    s = np.asarray(schedule)
    return s[np.arange(s.shape[0]), np.minimum(np.asarray(lap_n), s.shape[1] - 1)].astype(np.int32)
