"""The reference's tuning constants, values only (src/initControllerParameters.py:4-58, src/main.py:43-50).
They define the benchmark configurations of BASELINE.json; nothing here is executed by the reference."""
from dataclasses import dataclass
from types import SimpleNamespace
import numpy as np

HALF_WIDTH = 0.4          # Track.py:31
TRACK_LENGTH = 19.22957795130823   # Map(0.4).TrackLength (tests/golden pins it)


def _common():
    Fx = np.array([[0., 0., 0., 0., 0., 1.], [0., 0., 0., 0., 0., -1.]])
    Fu = np.kron(np.eye(2), np.array([1, -1])).T
    bu = np.array([0.5, 0.5, 10.0, 10.0])
    return Fx, Fu, bu


def mpc_params(N=12, vt=0.8):
    """initMPCParams (initControllerParameters.py:4-26): path-following MPC / LTV-MPC."""
    Fx, Fu, bu = _common()
    return SimpleNamespace(n=6, d=2, N=N, A=None, B=None, Q=np.diag([1.0, 1.0, 1, 1, 0.0, 100.0]),
                           R=np.diag([1.0, 10.0]), Qf=np.zeros((6, 6)), dR=np.zeros(2),
                           Qslack=np.array([0.0, 50.0]), Fx=Fx, bx=np.array([2.0, 2.0]), Fu=Fu, bu=bu,
                           xRef=np.array([vt, 0, 0, 0, 0, 0.0]), slacks=True, timeVarying=False)


def lmpc_params(N=12):
    """initLMPCParams (initControllerParameters.py:28-58).  Returns (numSS_it, numSS_Points, Laps,
    TimeLMPC, QterminalSlack, params)."""
    Fx, Fu, bu = _common()
    p = SimpleNamespace(n=6, d=2, N=N, A=None, B=None, Q=np.zeros((6, 6)), R=np.zeros((2, 2)),
                        Qf=np.zeros((6, 6)), dR=5 * np.array([1.0, 10.0]), Qslack=np.array([5.0, 25.0]),
                        Fx=Fx, bx=np.array([HALF_WIDTH, HALF_WIDTH]), Fu=Fu, bu=bu, xRef=np.zeros(6),
                        slacks=True, timeVarying=True)
    return 4, 48, 44, 400, 500 * np.eye(6), p


@dataclass(frozen=True)
class VehicleParams:
    """The vehicle of Simulator.dynModel (SysModel.py:61-70): mass, CoG to front / rear axle, yaw inertia and the Pacejka
    coefficients of the front and rear tyre, Fy = D sin(C atan(B alpha)).  The device simulator takes one per controller
    (BatchedController.set_vehicles)."""
    m: float
    lf: float
    lr: float
    Iz: float
    Df: float
    Cf: float
    Bf: float
    Dr: float
    Cr: float
    Br: float

    @classmethod
    def reference(cls):
        """The reference's car: friction coefficient 0.8."""
        return cls.from_friction(0.8)

    @classmethod
    def from_friction(cls, mu, m=1.98, lf=0.125, lr=0.125, Iz=0.024, Cf=1.25, Bf=1.0, Cr=1.25, Br=1.0):
        """Peak tyre force D = mu * m * 9.81 / 2.0 on both axles, in the reference's operation order (mu = 0.8 gives its D bit
        for bit)."""
        D = mu * m * 9.81 / 2.0
        return cls(m, lf, lr, Iz, D, Cf, Bf, D, Cr, Br)


def _wrap(a):
    if a < -np.pi:
        return 2 * np.pi + a
    if a > np.pi:
        return a - 2 * np.pi
    return a


class TrackParams:
    """A circuit as Map builds it (Track.py:54-133) from a spec of [length, radius] rows (radius 0: straight; negative: a right
    turn), closed by a straight back to the origin.  ``table6`` = Map.PointAndTangent (x_end, y_end, psi_end, s_start, length,
    curvature per row), ``seg_table`` = its columns 3:6 (what the device reads), ``TrackLength``.  The device takes one per
    controller (BatchedController.set_tracks)."""

    def __init__(self, table6):
        self.table6 = np.array(table6, dtype=float).reshape(-1, 6)
        self.seg_table = np.ascontiguousarray(self.table6[:, 3:6])
        self.TrackLength = self.table6[-1, 3] + self.table6[-1, 4]

    @classmethod
    def from_spec(cls, spec):
        """Map.__init__'s construction, operation for operation, so that the table equals the reference's bit for bit."""
        spec = np.asarray(spec, dtype=float).reshape(-1, 2)
        P = np.zeros((spec.shape[0] + 1, 6))
        for i in range(spec.shape[0]):
            length, r = spec[i, 0], spec[i, 1]
            # where the segment starts: the origin heading along x, or the end of the previous segment
            ang, x0, y0 = (0, 0, 0) if i == 0 else (P[i - 1, 2], P[i - 1, 0], P[i - 1, 1])
            s0 = P[i, 3] if i == 0 else P[i - 1, 3] + P[i - 1, 4]
            if r == 0.0:
                P[i] = [x0 + length * np.cos(ang), y0 + length * np.sin(ang), ang, s0, length, 0]
            else:
                d = 1 if r >= 0 else -1
                cx = x0 + np.abs(r) * np.cos(ang + d * np.pi / 2)
                cy = y0 + np.abs(r) * np.sin(ang + d * np.pi / 2)
                span = length / np.abs(r)
                psi = _wrap(ang + span * np.sign(r))
                normal = _wrap(d * np.pi / 2 + ang)
                a = -(np.pi - np.abs(normal)) * (1 if normal >= 0 else -1)
                P[i] = [cx + np.abs(r) * np.cos(a + d * span), cy + np.abs(r) * np.sin(a + d * span), psi, s0, length, 1 / r]
        xs, ys = P[-2, 0], P[-2, 1]
        P[-1] = [0, 0, 0, P[-2, 3] + P[-2, 4], np.sqrt((0 - xs) ** 2 + (0 - ys) ** 2), 0]
        return cls(P)

    @staticmethod
    def l_shaped_spec():
        """The track the reference drives (Track.py:30-40)."""
        lc = 4.5
        return np.array([[1.0, 0], [lc, lc / np.pi], [lc / 2, -lc / np.pi], [lc, lc / np.pi], [lc / np.pi * 2, 0],
                         [lc / 2, lc / np.pi]])

    @staticmethod
    def goggle_spec():
        """The goggle-shaped track (Track.py:15-28, commented out in the reference)."""
        return np.array([[60 * 0.03, 0], [80 * 0.03, -80 * 0.03 * 2 / np.pi], [20 * 0.03, 0], [80 * 0.03, -80 * 0.03 * 2 / np.pi],
                         [40 * 0.03, +40 * 0.03 * 10 / np.pi], [60 * 0.03, -60 * 0.03 * 5 / np.pi],
                         [40 * 0.03, +40 * 0.03 * 10 / np.pi], [80 * 0.03, -80 * 0.03 * 2 / np.pi], [20 * 0.03, 0],
                         [80 * 0.03, -80 * 0.03 * 2 / np.pi]])

    @staticmethod
    def oval_spec():
        """A right-turning oval (Track.py:43-48, commented out in the reference).  Its closing straight is 6.3e-16 long."""
        return np.array([[1.0, 0], [4.5, -4.5 / np.pi], [2.0, 0], [4.5, -4.5 / np.pi], [1.0, 0]])

    @classmethod
    def l_shaped(cls):
        return cls.from_spec(cls.l_shaped_spec())

    @classmethod
    def goggle(cls):
        return cls.from_spec(cls.goggle_spec())

    @classmethod
    def oval(cls):
        return cls.from_spec(cls.oval_spec())
