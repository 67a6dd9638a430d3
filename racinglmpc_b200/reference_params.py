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
