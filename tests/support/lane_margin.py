"""The lane-margin rule of the device closed loop (lmpc_set_lane_margins, DESIGN.md "Lane margins") restated on the host.

``lap_left_lane`` is the verdict of a mode 2 hand-over: the lap's recorded rows leave the lane Fx x <= bx when a row has a
non-finite entry or d_i > 0, d_i computed as the lap reports compute it (tests/support/lap_reports.lane_margins: in order, float64,
no fused multiply-adds).  ``adapt`` is the update of the margin after such a lap; ``planning_bx`` the lane a margin plans in.
Python floats round every operation once, as the device's __dadd_rn / __dsub_rn do, so the results match bit for bit."""
import numpy as np

from lap_reports import lane_margins


def lap_left_lane(x, Fx, bx):
    """Do the rows x [T, >= 6] (their first 6 entries) leave the lane Fx x <= bx?"""
    for row in np.asarray(x, np.float64):
        v = [float(e) for e in row[:6]]
        if not all(np.isfinite(v)):
            return True
        if any(d > 0.0 for d in lane_margins(Fx, bx, v)):
            return True
    return False


def adapt(row, m, left):
    """The margin after a lap under a mode 2 row (objects with margin0, margin_max, step_up, step_down)."""
    if left:
        return float(np.fmin(float(m) + float(row.step_up), float(row.margin_max)))
    return float(np.fmax(float(m) - float(row.step_down), float(row.margin0)))


def start(row):
    """m_b at the install and at every seeding: 0 under mode 0, margin0 under modes 1 and 2."""
    return 0.0 if int(row.mode) == 0 else float(row.margin0)


def hand_over(row, m, x, Fx, bx):
    """m_b after an own-lap hand-over of the rows x: adapted under mode 2, unchanged otherwise."""
    return adapt(row, m, lap_left_lane(x, Fx, bx)) if int(row.mode) == 2 else float(m)


def planning_bx(bx, m):
    """The lane rows a margin m plans with: bx_i - m, rounded once."""
    return np.array([float(v) - float(m) for v in bx])
