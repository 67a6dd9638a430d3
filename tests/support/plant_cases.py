"""Case lists of the plant kernels' tests (tests/test_plant_reference.py on the CPU, tests/test_gpu_plant.py on the device).

Simulator cases cover the speeds, slips and steering angles of the closed loop and its edges: reverse and standstill (the atan2
branch cut at +-pi with signed zeros), every segment start, crossings of a segment boundary and of the finish line inside the
100 sub-steps, s in laps 2 and 3, ey at 0.9 / curvature on each circuit's tightest arc, all eight golden cars, all three golden
circuits (the oval with its empty closing segment) and the clip edges of the noise.  One case per controller: a batch of them is
one launch.  The noise sets all give the PID sigma 1 and clip 1e3, so that the PID's draw sets the input a case asks for.
"""
import os
from dataclasses import dataclass, field

import numpy as np

import plant_exact as pe
import track_model
from racinglmpc_b200.reference_params import NoiseParams, TrackParams, VehicleParams

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "golden")
CIRCUITS = ("l_shaped", "goggle", "oval")
TRACKS = [TrackParams.l_shaped(), TrackParams.goggle(), TrackParams.oval()]
VEHICLES = [VehicleParams(*row) for row in np.load(os.path.join(GOLD, "vehicle_golden.npz"))["vehicles"]]
CLIP = 0.05
_PID = dict(pid_sigma=(1.0, 1.0), pid_clip=(1e3, 1e3))
NOISES = [
    NoiseParams((0.01, 0.01, 0.005), (0.05, 0.05, 0.05), 0.01, **_PID),       # the reference's simulator noise
    NoiseParams((1.0, 1.0, 1.0), (CLIP, CLIP, CLIP), 1.0, **_PID),             # z itself, clipped: the clip edges
    NoiseParams((0.0, 0.0, 0.0), (0.05, 0.05, 0.05), 0.01, **_PID),            # sigma 0
    NoiseParams((0.01, 0.01, 0.005), (0.05, 0.05, 0.05), 0.0, **_PID),         # gain 0
]
VT = 1.0


@dataclass
class SimCase:
    name: str
    x: np.ndarray
    u: np.ndarray                 # the input the case asks for (the device applies it up to the PID's rounding)
    z: np.ndarray                 # simulator draws (vx, vy, wz)
    veh: int
    trk: int
    noise_idx: int = 0
    xg: np.ndarray = None
    boundary_case: bool = False   # a deliberate boundary case: its margin is not required
    crosses: bool = False         # a sub-step crosses a segment boundary or the finish line
    vehicle: object = field(init=False)
    noise: object = field(init=False)
    exact_track: object = field(init=False)
    track_model: object = field(init=False)

    def __post_init__(self):
        self.x = np.asarray(self.x, float)
        self.u = np.asarray(self.u, float)
        self.z = np.asarray(self.z, float)
        if self.xg is None:
            self.xg = np.array([self.x[0], self.x[1], self.x[2], 0.3, 1.5, -0.7])
        self.vehicle = VEHICLES[self.veh]
        self.noise = NOISES[self.noise_idx]
        t = TRACKS[self.trk]
        self.exact_track = pe.ExactTrack(t.seg_table, t.TrackLength)
        self.track_model = track_model.from_table(t.table6)

    def z_pid(self):
        """PID draws that make the device's PID (sigma 1, clip 1e3, target speed VT) apply about ``u``."""
        return np.array([self.u[0] - (-0.6 * self.x[5] - 0.9 * self.x[3]), self.u[1] - 1.5 * (VT - self.x[0])])


def _mid(trk, k):
    t = TRACKS[trk].seg_table
    return float(t[k, 0] + 0.37 * t[k, 1])


def _long_segments(trk):
    t = TRACKS[trk].seg_table
    return [k for k in range(t.shape[0]) if t[k, 1] > 0.5]


def sim_cases():
    rng = np.random.default_rng(20261016)
    cases = []

    def add(name, x, u, trk=None, **kw):
        k = len(cases)
        trk = k % 3 if trk is None else trk
        z = kw.pop("z", rng.standard_normal(3))
        cases.append(SimCase(name, x, u, z, veh=k % len(VEHICLES), trk=trk, **kw))

    # speed, slip and steering: slip angles up to the tyre peak and beyond
    for vx in (0.05, 0.3, 1.0, 2.0, 3.5):
        for j in range(4):
            trk = (len(cases)) % 3
            segs = _long_segments(trk)
            s = _mid(trk, segs[j % len(segs)])
            d = (0.45, -0.45, rng.uniform(-0.45, 0.45), rng.uniform(-0.45, 0.45))[j]
            a = (2.0, -2.0, rng.uniform(-2, 2), rng.uniform(-2, 2))[j]
            vy = rng.uniform(-1, 1) * 0.4 * max(vx, 0.25)
            wz = rng.uniform(-1, 1) * (1.0 + vx)
            add("slip vx=%g #%d" % (vx, j), [vx, vy, wz, rng.uniform(-0.3, 0.3), s, rng.uniform(-0.2, 0.2)], [d, a], trk=trk)
    # reverse
    for vx in (-0.5, -1.5):
        trk = len(cases) % 3
        add("reverse vx=%g" % vx, [vx, 0.1, -0.4, 0.05, _mid(trk, _long_segments(trk)[1]), 0.1], [0.2, -1.0], trk=trk)
    # standstill and reverse with vy +- lf wz a signed zero: atan2 at its branch cut
    for vx, y, a in ((0.0, 0.0, 1.0), (0.0, -0.0, -1.0), (-0.0, 0.0, -1.0), (-0.0, -0.0, 1.0), (-0.5, 0.0, 0.5), (-0.5, -0.0, 0.5)):
        trk = len(cases) % 3
        add("zero vx=%r y=%r" % (vx, y), [vx, y, y, 0.0, _mid(trk, 0), 0.0], [0.0 if a > 0 else 0.1, a], trk=trk)
    for trk in range(3):
        t, L = TRACKS[trk].seg_table, TRACKS[trk].TrackLength
        # every segment start (the empty closing segment of the oval has none: its start is the finish line)
        for k in range(t.shape[0]):
            if t[k, 1] > 0 and t[k, 0] < L:
                add("segment start %s/%d" % (CIRCUITS[trk], k), [1.0, 0.05, 0.2, 0.02, t[k, 0], 0.05], [0.05, 0.3], trk=trk)
        # a boundary crossed inside the period
        for k in range(t.shape[0] - 1):
            b = float(t[k, 0] + t[k, 1])
            if 0 < b < L:
                add("cross %s/%d" % (CIRCUITS[trk], k), [1.2, -0.03, 0.3, -0.02, b - 0.051 * 1.2, -0.04], [0.1, 0.5], trk=trk,
                    crosses=True)
        # the finish line inside the period, laps 2 and 3, and a finish line in lap 2
        add("finish %s" % CIRCUITS[trk], [1.3, 0.02, -0.1, 0.01, L - 0.047 * 1.3, 0.02], [0.0, 0.4], trk=trk, crosses=True)
        add("lap 2 %s" % CIRCUITS[trk], [1.0, 0.02, 0.3, 0.01, _mid(trk, 1) + L, -0.1], [0.1, 0.2], trk=trk)
        add("lap 3 %s" % CIRCUITS[trk], [2.0, -0.05, 0.6, -0.02, _mid(trk, 0) + 2 * L, 0.1], [0.2, -0.5], trk=trk)
        add("finish lap 2 %s" % CIRCUITS[trk], [0.9, 0.0, 0.1, 0.0, 2 * L - 0.033, 0.0], [0.0, 0.1], trk=trk, crosses=True)
        # ey at 0.9 / curvature on the tightest arc: 1 - c ey = 0.1
        k = int(np.argmax(np.abs(t[:, 2])))
        add("lane %s" % CIRCUITS[trk], [1.0, 0.05, 0.5, 0.0, float(t[k, 0] + 0.5 * t[k, 1]), 0.9 / t[k, 2]], [0.0, 0.0], trk=trk)
    # noise at the clip edges (sigma 1, gain 1: the draw is z clipped), sigma 0 and gain 0
    c, inside, outside = CLIP, np.nextafter(CLIP, 0.0), np.nextafter(CLIP, 1.0)
    for z in ((c, -c, inside), (outside, -outside, -inside), (-c, c, outside), (0.7, -3.0, 1e-3)):
        trk = len(cases) % 3
        add("clip z=%r" % (z,), [1.0, 0.0, 0.1, 0.0, _mid(trk, 0), 0.0], [0.0, 0.2], trk=trk, noise_idx=1, z=np.array(z))
    for n in (2, 3):
        trk = len(cases) % 3
        add("noise set %d" % n, [1.0, 0.0, 0.1, 0.0, _mid(trk, 0), 0.0], [0.0, 0.2], trk=trk, noise_idx=n)
    return cases


@dataclass
class PidCase:
    name: str
    x: np.ndarray
    vt: float
    z: np.ndarray
    noise_idx: int
    ulps: float = 1.0
    noise: object = field(init=False)

    def __post_init__(self):
        self.noise = PID_NOISES[self.noise_idx]


_SIM = dict(sim_sigma=(0.01, 0.01, 0.005), sim_clip=(0.05, 0.05, 0.05), sim_gain=0.01)
PID_NOISES = [
    NoiseParams(pid_sigma=(0.25, 0.10), pid_clip=(0.9, 0.2), **_SIM),        # the reference's PID noise
    NoiseParams(pid_sigma=(1.0, 1.0), pid_clip=(0.9, 0.2), **_SIM),          # z itself, clipped: the clip edges
    NoiseParams(pid_sigma=(0.0, 0.0), pid_clip=(0.9, 0.2), **_SIM),          # sigma 0
    NoiseParams(pid_sigma=(0.5, 2.0), pid_clip=(0.3, 0.7), **_SIM),
]


def pid_cases():
    """States without cancellation between the PID's terms (-0.6 ey - 0.9 epsi and the steering draw share a sign, as do
    1.5 (vt - vx) and the acceleration draw), so that one ulp of the result bounds every correct fp64 evaluation."""
    rng = np.random.default_rng(42)
    out = []
    c0, c1 = 0.9, 0.2
    edges = [(-c0, c1), (-np.nextafter(c0, 0), np.nextafter(c1, 0)), (-np.nextafter(c0, 1), np.nextafter(c1, 1))]
    for k in range(48):
        x = np.array([rng.uniform(0.3, 0.95), rng.uniform(-0.2, 0.2), rng.uniform(-1, 1), rng.uniform(0.01, 0.2),
                      rng.uniform(0, 19), rng.uniform(0.05, 0.3)])
        nidx = k % len(PID_NOISES)
        if nidx == 1:
            z = np.array(edges[(k // 4) % 3])
        else:
            z = np.array([-abs(rng.standard_normal()) * 3, abs(rng.standard_normal()) * 3])
        out.append(PidCase("pid #%d" % k, x, VT, z, nidx))
    return out


def sysid_records():
    """(x, u, lamb) records of the sysid calibration: the golden PID lap with three ridges (lambda 0 on well-posed data), its
    first 12, 13 and 300 rows, and a rank-deficient record (constant vx, zero input) with lambda > 0."""
    g = np.load(os.path.join(GOLD, "reference_golden.npz"))
    x, u = g["pid_x"], g["pid_u"]
    recs = [(x, u, 1e-7), (x, u, 0.0), (x, u, 1e3), (x[:12], u[:12], 1e-7), (x[:13], u[:13], 1e-7), (x[:300], u[:300], 1e-7)]
    xr, ur = rank_deficient_record(40)
    recs += [(xr, ur, 1e-7), (xr, ur, 1e3)]
    return recs


def rank_deficient_record(T, vx=1.0, dt=0.1):
    """Constant vx on a straight, no input: columns vy, wz, epsi, ey and both inputs are zero."""
    x = np.zeros((T, 6))
    x[:, 0] = vx
    x[:, 4] = np.arange(T) * (vx * dt)
    return x, np.zeros((T, 2))


COST_T = (1, 2, 255, 256, 257, 511, 512, 513)


def cost_cases(L, Tmax):
    """(s column, T) of the lap-cost cases: for every T in COST_T and Tmax, a lap that stays below the finish line, and one with
    rows at or past it at rows 0, 255, 256 and T-1, two more crossings, a NaN and an s exactly at TrackLength."""
    out = []
    for T in COST_T + (Tmax,):
        s = np.linspace(0.0, 0.99 * L, T)
        out.append((s.copy(), T))
        for r in (0, 255, 256, T - 1):
            if r < T:
                s[r] = L + 0.25
        if T > 8:
            s[T // 3] = L + 1.0
            s[(2 * T) // 3] = 2 * L
            s[T // 2] = np.nan
            s[T // 4] = L
        elif T == 2:
            s[0] = L
        out.append((s, T))
    return out
