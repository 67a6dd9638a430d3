"""Test-side restatement of Map (Track.py) for any circuit.

oracle/track.py restates the reference's one L-shaped track, built in its constructor; ``from_table`` gives the same object for
any Map.PointAndTangent, so that Map.curvature / Map.getGlobalPosition (oracle.track.TrackTable.curvature / global_position) and
everything that takes a track object (vehicle_model.dyn_model / closed_loop, oracle.ltv_model.LocalLTVModel) work on any circuit.
Checked against the reference's own Map on the three circuits of Track.py (tests/golden/track_golden.npz).
"""
import numpy as np

from oracle.track import TrackTable


def from_table(table6):
    """A TrackTable whose PointAndTangent is ``table6`` ([nseg, 6]: x_end, y_end, psi_end, s_start, length, curvature) and whose
    TrackLength is start + length of its last row (Track.py:133).  The half-width and slack are the L track's (Track.py:31-32);
    the device takes the lane width through Fx / bx, not through the track."""
    t = TrackTable.__new__(TrackTable)
    t.halfWidth, t.slack = 0.4, 0.45
    t.PointAndTangent = np.array(table6, dtype=float).reshape(-1, 6)
    t.TrackLength = t.PointAndTangent[-1, 3] + t.PointAndTangent[-1, 4]
    return t
