"""The reference's tuning constants, values only (src/initControllerParameters.py:4-58, src/main.py:43-50).
They define the benchmark configurations of BASELINE.json; nothing here is executed by the reference."""
import math
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


@dataclass(frozen=True)
class NoiseParams:
    """The noise of the closed loop: Simulator.dynModel adds sim_gain * clip(z_j * sim_sigma_j, +-sim_clip_j) to (vx, vy, wz)
    (SysModel.py:139-145), the PID path follower adds clip(z_j * pid_sigma_j, +-pid_clip_j) to (steering, acceleration)
    (Utilities.py:42-68), z_j standard normal.  The device closed loop takes one per controller (BatchedController.set_noise)."""
    sim_sigma: tuple
    sim_clip: tuple
    sim_gain: float
    pid_sigma: tuple
    pid_clip: tuple

    @classmethod
    def reference(cls):
        """The reference's constants."""
        return cls((0.01, 0.01, 0.005), (0.05, 0.05, 0.05), 0.01, (0.25, 0.10), (0.9, 0.2))

    @classmethod
    def scaled(cls, sim=1.0, pid=1.0):
        """The reference's noise with sigma and clip of the simulator multiplied by ``sim`` and those of the PID by ``pid`` (the
        gain stays): 1 gives the reference's values bit for bit, 0 a noise-free plant or PID."""
        r = cls.reference()
        return cls(tuple(v * sim for v in r.sim_sigma), tuple(v * sim for v in r.sim_clip), r.sim_gain,
                   tuple(v * pid for v in r.pid_sigma), tuple(v * pid for v in r.pid_clip))


@dataclass(frozen=True)
class MeasurementParams:
    """The sensor noise of the closed loop (no reference counterpart: the reference's controllers read the simulator's exact
    state): a controller sees y_j = x_j + clip(z_j * sigma_j, +-clip_j) on the six curvilinear channels (vx, vy, wz, epsi, s, ey),
    z_j standard normal, in the form of the process noise.  The device closed loop takes one per controller
    (BatchedController.set_measurement_noise)."""
    sigma: tuple
    clip: tuple

    @classmethod
    def zero(cls):
        """No measurement noise: installed, it gives every controller the plant state bit for bit."""
        return cls((0.0,) * 6, (0.0,) * 6)

    @classmethod
    def scaled(cls, k, base):
        """``base`` with every sigma and clip multiplied by ``k``: 1 gives ``base`` bit for bit, 0 no noise."""
        return cls(tuple(v * k for v in base.sigma), tuple(v * k for v in base.clip))


@dataclass(frozen=True)
class ObserverParams:
    """A fixed-gain state observer (no reference counterpart): a mode 1 controller reads x_hat_j = p_j + gain_j (y_j - p_j) on
    the six curvilinear channels (vx, vy, wz, epsi, s, ey) in place of the state y it is given (measured or true), p being its own
    one-step prediction xPred[1] of the previous step.  Gain 1 trusts the measurement, gain 0 the prediction.  Mode 0 reads y.
    The device closed loop takes one per controller (BatchedController.set_observers)."""
    mode: int = 0
    gain: tuple = (1.0,) * 6

    @classmethod
    def off(cls):
        """No observer: installed, the controllers read the state they are given, bit for bit."""
        return cls(0, (1.0,) * 6)

    @classmethod
    def uniform(cls, l):
        """An observer with gain ``l`` on every channel (1 reads y bit for bit)."""
        return cls(1, (float(l),) * 6)

    @classmethod
    def gains(cls, vx, vy, wz, epsi, s, ey):
        """An observer with one gain per channel."""
        return cls(1, tuple(float(v) for v in (vx, vy, wz, epsi, s, ey)))

    @classmethod
    def from_noise(cls, model_sigma, meas_sigma):
        """Per channel, the steady-state Kalman gain of a scalar random walk x_{k+1} = x_k + w (w of standard deviation
        model_sigma) measured as y = x + v (v of standard deviation meas_sigma): with q = model_sigma^2 and r = meas_sigma^2 the
        prior variance solves P = P r / (P + r) + q, so P = (q + sqrt(q^2 + 4 q r)) / 2, and l = P / (P + r).  meas_sigma == 0
        gives l = 1 (a perfect sensor), and model_sigma == 0 with meas_sigma > 0 gives l = 0.  Each argument is one value for
        every channel or six."""
        ms = np.broadcast_to(np.asarray(model_sigma, float), (6,))
        rs = np.broadcast_to(np.asarray(meas_sigma, float), (6,))
        if not (np.all(np.isfinite(ms)) and np.all(np.isfinite(rs)) and np.all(ms >= 0) and np.all(rs >= 0)):
            raise ValueError("model_sigma and meas_sigma must be finite and >= 0")
        out = []
        for m, s in zip(ms, rs):
            q, r = float(m) * float(m), float(s) * float(s)
            if r == 0.0:
                out.append(1.0)
                continue
            P = (q + math.sqrt(q * q + 4.0 * q * r)) / 2.0
            out.append(P / (P + r))
        return cls(1, tuple(out))


@dataclass(frozen=True)
class RegressionParams:
    """The constants of the local regression model (PredictiveModel.py:18-31): the laps used (the trToUse shortest stored laps),
    the neighbour count, the Epanechnikov bandwidth h, the ridge term and the diagonal of the feature scaling of the 1-norm
    distance over (vx, vy, wz, delta, a).  K1 takes one per controller (BatchedController.set_regression)."""
    trToUse: int
    MaxNumPoint: int
    h: float
    lamb: float
    scaling: tuple

    @classmethod
    def reference(cls, trToUse=4):
        """The reference's constants: PredictiveModel(n, d, map, trToUse) builds 1 for the LTV-MPC and 4 for LMPC
        (main.py:88,102)."""
        return cls(int(trToUse), 7, 5.0, 0.0, (0.1, 1.0, 1.0, 1.0, 1.0))


@dataclass(frozen=True)
class LapWindowParams:
    """How many of its most recent laps a controller's safe set and learned model draw from (0 = unbounded, the reference's
    rule): the safe set selects its numSS_it fastest laps among lap numbers [it - ss_window, it), the model regresses on the
    trToUse shortest laps among the last model_window it filed.  The device takes one per controller
    (BatchedController.set_lap_windows)."""
    ss_window: int = 0
    model_window: int = 0

    @classmethod
    def unbounded(cls):
        """Both windows unbounded: installed, the controllers select and store exactly what they do without a table."""
        return cls(0, 0)


@dataclass(frozen=True)
class LaneRuleParams:
    """Whether a controller's safe set ranks a lap that left the lane behind every lap that kept to it: mode 0 is the
    reference's rule (laps ranked by lap time alone), mode 1 judges every lap the controller files and ranks one whose rows leave
    a lane row by more than lane_tol behind the others.  The device takes one per controller
    (BatchedController.set_lane_rules)."""
    mode: int = 0
    lane_tol: float = 0.0

    @classmethod
    def reference(cls):
        """The reference's rule: installed, the controllers rank and store exactly what they do without a table."""
        return cls(0, 0.0)


@dataclass(frozen=True)
class LaneMarginParams:
    """The margin a controller's QPs narrow its lane by, while its reports and lane rules judge the lane it was given: mode 0
    none (the reference), mode 1 the fixed margin0, mode 2 a margin adapted after every own lap within [margin0, margin_max] --
    up by step_up after a lap that left the lane, down by step_down after one that kept to it.  The device takes one per
    controller (BatchedController.set_lane_margins)."""
    mode: int = 0
    margin0: float = 0.0
    margin_max: float = 0.0
    step_up: float = 0.0
    step_down: float = 0.0

    @classmethod
    def reference(cls):
        """No margin: installed, the controllers plan in the lane they are judged against."""
        return cls(0, 0.0, 0.0, 0.0, 0.0)


@dataclass(frozen=True)
class PredictionModelParams:
    """Where rows 0..2 (vx, vy, wz) of a controller's LTV model come from: mode 0 the k-NN regression of its stored laps (the
    reference), mode 1 the exact linearisation of the simulator's one-period map for ``vehicle`` (a car the controller believes
    it drives), mode 2 the same for the plant's own vehicle row (``vehicle`` is not read).  The device takes one per controller
    (BatchedController.set_prediction_models)."""
    mode: int = 0
    vehicle: VehicleParams = VehicleParams.reference()

    @classmethod
    def learned(cls):
        """The k-NN regression: installed, the controllers identify exactly what they do without a table."""
        return cls(0)

    @classmethod
    def plant(cls):
        """The exact linearisation of the car the simulator drives for the controller."""
        return cls(2)

    @classmethod
    def believes(cls, vehicle):
        """The exact linearisation of ``vehicle``, whatever the plant drives."""
        return cls(1, vehicle)


@dataclass(frozen=True)
class ObserverPrior:
    """Where a state observer (ObserverParams mode 1) takes its prior from (no reference counterpart): source 0 the controller's
    own plan (its previous QP's xPred[1]), source 1 the estimate of the previous step carried over one control period under the
    input applied, by the simulator's noise-free map for ``vehicle`` (a car the controller believes it drives, no surface),
    source 2 the same map for the plant's own vehicle and surface rows.  The device takes one per controller
    (BatchedController.set_observer_priors)."""
    source: int = 0
    vehicle: VehicleParams = VehicleParams.reference()

    @classmethod
    def plan(cls):
        """The controller's own plan: installed, the observers compute exactly what they compute without a table."""
        return cls(0)

    @classmethod
    def car(cls, vehicle):
        """The one-period map of ``vehicle``, whatever the plant drives."""
        return cls(1, vehicle)

    @classmethod
    def plant(cls):
        """The one-period map of the car and surface the plant drove the previous step with."""
        return cls(2)


def clipped_normal_variance(sigma, clip):
    """Var(clip(sigma Z, +-clip)) for a standard normal Z: with a = clip / sigma, sigma^2 [(1 - 2 Phi(-a)) - 2 a phi(a)] +
    2 clip^2 Phi(-a) (the variance of the noise the simulator and the sensor add).  0 when sigma or clip is 0."""
    sigma, clip = float(sigma), float(clip)
    if sigma == 0.0 or clip == 0.0:
        return 0.0
    if math.isinf(clip):
        return sigma * sigma
    a = clip / sigma
    tail = 0.5 * math.erfc(a / math.sqrt(2.0))                       # Phi(-a)
    dens = math.exp(-0.5 * a * a) / math.sqrt(2.0 * math.pi)          # phi(a)
    return sigma * sigma * ((1.0 - 2.0 * tail) - 2.0 * a * dens) + 2.0 * clip * clip * tail


@dataclass(frozen=True)
class ObserverGains:
    """The gains a state observer (ObserverParams mode 1) blends with (no reference counterpart): mode 0 its row's fixed gains,
    mode 1 the frozen-time Kalman gain K = P (P + R)^-1 of the linearised one-period map of its prior's car, P solving the filter
    DARE for diagonal Q = diag(q) (process covariance per control period) and R = diag(r) (measurement covariance) over (vx, vy,
    wz, epsi, s, ey).  Mode 1 needs a car prior (ObserverPrior.car or .plant).  The device takes one per controller
    (BatchedController.set_observer_gains)."""
    mode: int = 0
    q: tuple = (1.0,) * 6
    r: tuple = (1.0,) * 6

    @classmethod
    def fixed(cls):
        """The observer row's fixed gains: installed, the observers compute exactly what they compute without a table."""
        return cls(0)

    @classmethod
    def kalman(cls, q, r):
        """Model gains for the covariance diagonals ``q`` and ``r`` (one value for every channel or six, each finite and > 0)."""
        qs = np.broadcast_to(np.asarray(q, float), (6,))
        rs = np.broadcast_to(np.asarray(r, float), (6,))
        return cls(1, tuple(float(v) for v in qs), tuple(float(v) for v in rs))

    @classmethod
    def from_noise(cls, noise, measurement, model_sigma):
        """Model gains matched to the closed loop's noise: r_j the exact variance of the clipped sensor noise of ``measurement``
        (MeasurementParams), q on vx, vy, wz the variance of the simulator's process noise of ``noise`` (NoiseParams:
        sim_gain^2 Var(clip(sim_sigma Z, +-sim_clip))) plus model_sigma_j^2, q on epsi, s, ey model_sigma_j^2 alone.
        ``model_sigma`` (one value or six, finite and >= 0) is the standard deviation per control period of the model's own
        error, e.g. of the prior against the true state in a noise-free run.  Raises ValueError where a q_j or r_j would be 0 (a
        noise-free sensor channel, or a channel without process noise and model error) or is not finite."""
        ms = np.broadcast_to(np.asarray(model_sigma, float), (6,))
        if not (np.all(np.isfinite(ms)) and np.all(ms >= 0)):
            raise ValueError("model_sigma must be finite and >= 0")
        g = float(noise.sim_gain)
        q = [g * g * clipped_normal_variance(noise.sim_sigma[j], noise.sim_clip[j]) + float(ms[j]) ** 2 for j in range(3)]
        q += [float(ms[j]) ** 2 for j in range(3, 6)]
        r = [clipped_normal_variance(measurement.sigma[j], measurement.clip[j]) for j in range(6)]
        for name, v in (("q", q), ("r", r)):
            bad = [j for j in range(6) if not (math.isfinite(v[j]) and v[j] > 0.0)]
            if bad:
                raise ValueError("ObserverGains.from_noise: %s is not > 0 on channel(s) %s" % (name, bad))
        return cls(1, tuple(q), tuple(r))


@dataclass(frozen=True)
class SurfaceParams:
    """A track surface (no reference counterpart: the reference's grip is the same all round the lap): up to 16 zones
    (s_start, s_end, mu_f, mu_r), ascending without overlap, in the s-coordinate of the controller's track.  A simulator sub-step
    whose s (wrapped as the curvature lookup wraps it) lies in [s_start, s_end) of a zone drives with peak tyre forces mu_f Df and
    mu_r Dr of its car; elsewhere the car's own.  The device takes one per controller (BatchedController.set_surfaces)."""
    zones: tuple = ()

    def __post_init__(self):
        object.__setattr__(self, "zones", tuple(tuple(float(v) for v in z) for z in self.zones))

    @classmethod
    def dry(cls):
        """No zone: installed, the controllers drive exactly what they drive without a table."""
        return cls(())

    @classmethod
    def from_zones(cls, zones):
        """Zones given as (s_start, s_end, mu_f, mu_r) rows."""
        return cls(tuple(zones))

    @classmethod
    def on_segment(cls, track, row, mu_f, mu_r=None):
        """One zone covering segment ``row`` of ``track`` (a TrackParams): [s_start, s_start + length) of its seg_table row, the
        end rounded as the curvature lookup forms it; ``mu_r`` None takes ``mu_f``."""
        s0, ln = float(track.seg_table[row, 0]), float(track.seg_table[row, 1])
        return cls(((s0, float(np.float64(s0) + np.float64(ln)), float(mu_f), float(mu_f if mu_r is None else mu_r)),))


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
