"""Adversarial inputs for the k-NN regression kernel (K1, csrc/safeset.cuh knn_ltv_regress_kernel), a NumPy emulation of its
fp32 pre-filter and an exact reference of what it must compute.

K1 ranks every stored row with an fp32 distance packed into a key (the distance with its low 7 mantissa bits replaced by the row
counter j = t // 32 of lane t % 32), keeps the 3 smallest keys per lane, bounds the k-th nearest distance by the k-th smallest lane
minimum G and re-scores in exact fp64 every row under thr = G (1 + 3.2e-5) + (G + 2 qsum) 1.3e-6 (at most 32 of them; more sets
flag 32).  When a lane's third key is under thr it re-collects the candidates from global memory.  The fixtures below put rows
where that argument is tight: distances equal to 1e-9 relative across the k-th neighbour, many of the nearest rows in one lane,
more rows within fp32 resolution of the k-th distance than the re-scoring buffer holds, features of magnitude 50 whose fp32
rounding exceeds the differences that decide the selection, rows at the bandwidth h to the last bit, tile edges and the last row
counter of a 4096-row lap.

* ``prefilter``: which branch of the pre-filter a query takes on one lap, and how far every decision is from flipping.
* ``ExactLTVModel``: the oracle's arithmetic (oracle/ltv_model.py) with ties to the lowest row (np.argsort kind="stable", as
  the kernel documents) and the three 5 x 5 Gram systems solved in mpmath at 60 digits from the fp64 rows and weights.
* ``groups()``: the fixtures, grouped by what one controller handle shares (horizon, laps used, model constants, Tmax).
"""
from dataclasses import dataclass, field
from functools import lru_cache

import mpmath
import numpy as np

from oracle import ltv_model
from oracle.track import TrackTable

JBITS = 7
JMASK = (1 << JBITS) - 1
LOCAL = 3                      # entries of a lane's candidate list
CAND = 32                      # exact re-scoring buffer
FAR = np.float32(1e18)         # feature value of the padding rows of the last batch
EMPTY = np.uint32(0xFFFFFFFF)
MARGIN = 2.0 ** -20            # every pre-filter decision of a fixture is at least this far (relative) from flipping
DEFAULT = dict(MaxNumPoint=7, h=5.0, lamb=0.0, dt=0.1, scaling=(0.1, 1.0, 1.0, 1.0, 1.0))
DIGITS = 60


# ---------------------------------------------------------------------------------------------------------------- emulation
def _fma32(a, b, c):
    """fmaf emulated as the fp64 product (exact for fp32 inputs) plus c, rounded to fp64 and then to fp32."""
    return (np.float64(a) * np.float64(b) + np.float64(c)).astype(np.float32) if np.ndim(c) else \
        np.float32(np.float64(a) * np.float64(b) + np.float64(c))


def _dist32(F, f, s):
    """The scan's fp32 distance of feature rows F[n,5] (fp32) to the query f[5] (fp32) with scalings s[5] (fp32)."""
    D = np.abs(F - f[None, :])
    d = (s[0] * D[:, 0]).astype(np.float32)
    for k in range(1, 5):
        d = (np.float64(s[k]) * D[:, k].astype(np.float64) + d.astype(np.float64)).astype(np.float32)
    return d


def _bits(v):
    return np.asarray(v, np.float32).view(np.uint32)


def _flt(b):
    return np.asarray(b, np.uint32).view(np.float32)


def _bucket(d):
    """[lo, hi) of the fp32 values whose key has the same high 25 bits as d."""
    b = int(_bits(np.float32(d))) & ~JMASK
    return float(_flt(np.uint32(b))), float(_flt(np.uint32(b + JMASK + 1)))


def _key_flip(d, thr):
    """Smallest relative perturbation of d or thr that flips `key(d) <= thr | JMASK` (keys compare on the bucket)."""
    lo_t, hi_t = _bucket(thr)
    lo_d, hi_d = _bucket(d)
    if lo_d <= lo_t:                                   # in: d must rise above thr's bucket, or thr fall below its own
        return min(hi_t / d - 1.0, max(1.0 - lo_t / thr, lo_t / d - 1.0))
    hi2 = _bucket(hi_t)[1]                             # out: d must fall into thr's bucket, or thr rise into d's
    return max(min(1.0 - hi_t / d, max(hi_t / thr - 1.0, 1.0 - hi2 / d)), 0.0)


@dataclass
class Prefilter:
    branch: str            # "fast" | "recollect" | "overflow" (more than CAND candidates: flag 32) | "open"
    nc: int                # candidates re-scored (before the CAND cap)
    cand: np.ndarray       # their rows (first CAND)
    margins: dict          # decision -> relative distance from flipping


def prefilter(x, u, q5, consts, c_abs=1.3e-6, recollect=True):
    """Emulate K1's scan of one lap (x[T,6], u[T,2]) for the query q5 = (vx, vy, wz, delta, a) (csrc/safeset.cuh, steps 1-3).

    c_abs (the factor of the (G + 2 qsum) term of the threshold) and recollect=False (the fast path even when a lane list is
    full of candidates) describe weakened kernels: the fixtures must make those lose rows of the exact selection."""
    kk = int(consts["MaxNumPoint"])
    s = np.abs(np.asarray(consts["scaling"], np.float64)).astype(np.float32)
    f = np.asarray(q5, np.float64).astype(np.float32)
    T = x.shape[0]
    nrow = T - 1
    rows32 = (nrow + 31) & ~31
    F = np.full((rows32, 5), FAR, np.float32)
    F[:nrow] = np.hstack((x[:nrow, 0:3], u[:nrow])).astype(np.float32)
    d = _dist32(F, f, s)
    t = np.arange(rows32)
    key = (_bits(d) & np.uint32(~JMASK & 0xFFFFFFFF)) | (t >> 5).astype(np.uint32)
    lanes = np.sort(key.reshape(-1, 32), axis=0)                  # [blocks, 32]: each lane's keys, ascending
    lists = np.full((LOCAL, 32), EMPTY, np.uint32)
    n = min(LOCAL, lanes.shape[0])
    lists[:n] = lanes[:n]
    qsum = np.float32(s[0] * abs(f[0]))
    for k in range(1, 5):
        qsum = _fma32(s[k], abs(f[k]), qsum)
    cur = lists[0].copy()
    G = EMPTY
    for _ in range(max(kk, 2)):                  # at least two rounds (flag 4 needs both nearest rows as candidates)
        G = cur.min()
        cur[cur == G] = EMPTY
    row = ((lists & np.uint32(JMASK)).astype(np.int64) << 5) + np.arange(32)[None, :]
    open_thr = np.float32(FAR * np.float32(1e-3))

    def select(Gb):
        """Branch, candidates and decision margins for the lane-minimum key bucket Gb."""
        Gf = _flt(np.uint32(Gb))
        is_open = not (Gf < open_thr)
        margins = {}
        if is_open:
            thr = np.float32(3.0e38)
        else:
            a = _fma32(Gf, np.float32(3.2e-5), Gf)
            b = _fma32(np.float32(2.0), qsum, Gf)
            thr = _fma32(b, np.float32(c_abs), a)
            margins["open"] = abs(float(Gf) / float(open_thr) - 1.0)
        thrk = np.uint32(int(_bits(thr)) | JMASK)
        inl = (lists <= thrk) & (row < nrow) & (lists != EMPTY)
        if not is_open:
            real = (lists != EMPTY) & (row < nrow)
            m = [_key_flip(float(d[r]), float(thr)) for r in row[real]]
            margins["select"] = min(m) if m else np.inf
        if inl[2].any() and recollect:
            cand = np.nonzero(d[:nrow] <= thr)[0]
            if not is_open:
                margins["recollect"] = float(np.min(np.abs(d[:nrow].astype(np.float64) / float(thr) - 1.0)))
            branch = "recollect"
        else:
            cand = np.concatenate([row[0][inl[0]], row[1][inl[1]]])
            branch = "fast"
        if is_open:
            branch = "open"
        elif len(cand) > CAND:
            branch = "overflow"
        return branch, np.sort(cand), margins

    Gb = int(G) & ~JMASK
    branch, cand, margins = select(Gb)
    if branch != "open":
        # G is the bucket of one row's distance: a row within MARGIN of its bucket's edge may land in the neighbouring bucket;
        # that decision only counts when the neighbouring G changes the branch or the candidates
        lane_g = int(np.nonzero(lists[0] == G)[0][0])
        dg = float(d[((int(G) & JMASK) << 5) + lane_g])
        lo, hi = _bucket(dg)
        margins["G"] = min(dg - lo, hi - dg) / dg
        if margins["G"] < MARGIN:
            alt = [select(Gb + s * (JMASK + 1)) for s in (-1, 1)]
            if all(a[0] == branch and np.array_equal(a[1], cand) for a in alt):
                margins["G"] = np.inf
    return Prefilter(branch, len(cand), cand[:CAND], margins)


def min_margin(pf):
    return min(pf.margins.values()) if pf.margins else np.inf


# ------------------------------------------------------------------------------------------------------------ exact reference
class ExactLTVModel(ltv_model.LocalLTVModel):
    """The oracle's regression with ties to the lowest row and the Gram systems solved exactly.

    ``exact=True``: rows 0..2 of A, B, C come from the mpmath solution of the Gram systems built from the fp64 rows and the
    oracle's fp64 weights; ``systems`` then holds per solve (kappa_2(Q), theta*, np.linalg.solve's theta).  ``override``
    {lap position: rows} replaces the selection in those laps (the wrong selections of the discrimination check)."""

    def __init__(self, track, trToUse, consts, exact=True):
        super().__init__(6, 2, track, trToUse)
        self.MaxNumPoint = int(consts["MaxNumPoint"])
        self.h, self.lamb, self.dt = float(consts["h"]), float(consts["lamb"]), float(consts["dt"])
        self.scaling = np.diag(np.asarray(consts["scaling"], float))
        self.exact = exact
        self.override = None
        self.systems, self.dists = [], {}

    def knn(self, q, lap):
        xs, us = self.xStored[lap], self.uStored[lap]
        data = np.hstack((xs[0:-1, ltv_model.STATE_FEATS], us[0:-1, :]))
        dist = np.linalg.norm(np.dot(data - q[None, :], self.scaling), 1, axis=1)
        self.dists[lap] = dist
        pos = self.usedIt.index(lap)
        if self.override is not None and pos in self.override:
            idx = np.asarray(self.override[pos], int)
        else:
            near = np.squeeze(np.where(dist < self.h))
            if near.shape[0] >= self.MaxNumPoint:      # a 0-d squeeze raises like the reference (PM.py:189)
                idx = np.argsort(dist, kind="stable")[0:self.MaxNumPoint]
            else:
                idx = near
        return idx, (1 - (dist[idx] / self.h) ** 2) * 3 / 4

    def _rhs(self, y_index, idxs, M, Kt):
        y = np.concatenate([np.atleast_1d(np.squeeze(self.xStored[lap][idxs[c] + 1, y_index])) for c, lap in enumerate(self.usedIt)])
        self._sys = (M, Kt, y)
        return -np.dot(np.dot(M.T, np.diag(Kt)), y)

    def _fit(self, Q, b):
        th = np.linalg.solve(Q, -b)                    # raises LinAlgError where the oracle does
        if self.exact:
            M, Kt, y = self._sys
            with mpmath.workdps(DIGITS):
                Mm = [[mpmath.mpf(float(v)) for v in r] for r in M]
                Km = [mpmath.mpf(float(k)) for k in Kt]
                ym = [mpmath.mpf(float(v)) for v in y]
                n = M.shape[1]
                Qm = mpmath.matrix(n, n)
                bm = mpmath.matrix(n, 1)
                for r in range(n):
                    for c in range(n):
                        Qm[r, c] = mpmath.fsum(Km[p] * Mm[p][r] * Mm[p][c] for p in range(len(Km))) + \
                            (mpmath.mpf(self.lamb) if r == c else 0)
                    bm[r] = mpmath.fsum(Km[p] * Mm[p][r] * ym[p] for p in range(len(Km)))
                ts = mpmath.lu_solve(Qm, bm)
                star = np.array([float(v) for v in ts])
                Qf = np.array([[float(Qm[r, c]) for c in range(n)] for r in range(n)])
            self.systems.append((float(np.linalg.cond(Qf)), star, th))
            th = star
        return th[0:3], th[3:4], th[-1]

    def model(self, x6, u2):
        self.systems = []
        A, B, C = self.regressionAndLinearization(np.asarray(x6, float), np.asarray(u2, float))
        return A, B, C


def rows012(A, B, C):
    """The regression rows 0..2 of (A | B | C) as K1 writes them."""
    return np.concatenate([A[0:3].ravel(), B[0:3].ravel(), C[0:3]])


def rows345(A, B, C):
    return np.concatenate([A[3:6].ravel(), B[3:6].ravel(), C[3:6]])


def abc_split(abc):
    A = abc[0:36].reshape(6, 6); B = abc[36:48].reshape(6, 2); C = abc[48:54]
    return A, B, C


def tolerance(systems):
    """Bound of the GPU test on rows 0..2: 1e-9 where kappa_2(Q) <= 1e6, else 32 kappa_2 2^-53 |theta*|_inf."""
    kap = max(s[0] for s in systems)
    if kap <= 1e6:
        return 1e-9, kap
    return 32.0 * kap * 2.0 ** -53 * max(np.max(np.abs(s[1])) for s in systems), kap


# ------------------------------------------------------------------------------------------------------------------ fixtures
@dataclass
class Fixture:
    name: str
    laps: list                      # [(x[T,6], u[T,2])] in the order they are added
    xLin: np.ndarray                # [N+1, 6]
    uLin: np.ndarray                # [N, 2]
    branch: list                    # per query: the pre-filter branch it must take on every used lap (None: any)
    flags: int = 0                  # expected K1 flags of the instance
    raises: type = None             # the exception the reference raises (flags 1, 2, 4)
    discriminate: bool = False      # selection-sensitive: a wrong selection must move the model far beyond the tolerance
    note: str = ""
    kappa: float = None             # conditioning fixtures: the kappa_2 of the Gram matrices they are built for


@dataclass
class Group:
    """Instances that share one controller handle."""
    name: str
    N: int
    trToUse: int
    consts: dict
    Tmax: int
    model_cap: int
    fixtures: list = field(default_factory=list)


def used_laps(fx, trToUse):
    """The trToUse laps the reference regresses on: the shortest, ties in order of arrival (PM.py:35-46)."""
    m = ltv_model.LocalLTVModel(6, 2, None, trToUse)
    for x, u in fx.laps:
        m.addTrajectory(x, u)
    return list(zip(m.xStored, m.uStored))[:trToUse]


def exact_model(fx, group, exact=True):
    m = ExactLTVModel(TRACK, group.trToUse, group.consts, exact)
    for x, u in fx.laps:
        m.addTrajectory(x, u)
    return m


TRACK = TrackTable(0.4)
SEG_STARTS = TRACK.PointAndTangent[:, 3].copy()
TL = TRACK.TrackLength


def _q32(v):
    """Round to a multiple of 2^-12: exact in fp32 for the magnitudes used here."""
    return np.round(np.asarray(v, float) * 4096.0) / 4096.0


def mid_bucket(D):
    """D moved to the middle of its fp32 key bucket: 64 ulps from both edges."""
    b = (int(_bits(np.float32(D))) & ~JMASK) | 64
    return float(_flt(np.uint32(b)))


class _Lap:
    """A lap of far-away background rows; designed rows are put at row t with the regression target x[t+1, 0:3]."""

    def __init__(self, T, rng):
        self.T = T
        self.x = np.zeros((T, 6))
        self.x[:, 0:3] = rng.normal(0.0, 0.5, (T, 3))
        self.x[:, 3] = 0.05 * rng.standard_normal(T)
        self.x[:, 4] = np.linspace(0.0, 18.0, T)
        self.x[:, 5] = 0.05 * rng.standard_normal(T)
        self.u = 300.0 + 100.0 * rng.random((T, 2))          # scaled distance > 500 from every query
        self.busy = np.zeros(T, bool)
        self.rng = rng

    def free(self, t):
        return 0 <= t < self.T - 1 and not self.busy[t] and not self.busy[t + 1]

    def put(self, t, feat, y):
        assert self.free(t), t
        self.x[t, 0:3] = feat[0:3]
        self.u[t] = feat[3:5]
        self.x[t + 1, 0:3] = y
        self.busy[t] = self.busy[t + 1] = True

    def spot(self, lane=None, avoid_lanes=()):
        """A free row, in `lane` when given, else in a lane not in avoid_lanes."""
        for _ in range(10000):
            b = int(self.rng.integers(0, (self.T - 2) // 32 + 1))
            ln = lane if lane is not None else int(self.rng.integers(0, 32))
            if lane is None and ln in avoid_lanes:
                continue
            t = 32 * b + ln
            if self.free(t):
                return t
        raise RuntimeError("lap full")

    def lap(self):
        return self.x.copy(), self.u.copy()


def _target(rng, feat):
    """Next-row (vx, vy, wz) of a designed row: a smooth function of its features plus noise, so the regression has signal."""
    W = np.array([[0.9, 0.05, 0.0], [0.02, 0.8, 0.1], [0.0, 0.1, 0.7], [0.0, 0.3, 0.4], [0.1, 0.0, 0.0]])
    return feat @ W + np.array([0.01, -0.02, 0.03]) + 0.05 * rng.standard_normal(3)


def _sphere(rng, q5, D, scaling):
    """Rows at scaled 1-norm distance D[i] from q5 in random directions (features with scaling 0 get random offsets)."""
    s = np.asarray(scaling, float)
    act = np.nonzero(s != 0)[0]
    out = np.tile(np.asarray(q5, float), (len(D), 1))
    for i, d in enumerate(D):
        w = rng.dirichlet(np.ones(len(act)))
        sg = rng.choice([-1.0, 1.0], len(act))
        out[i, act] += sg * w * d / np.abs(s[act])
        out[i, s == 0] += rng.normal(0.0, 0.5, int(np.sum(s == 0)))
    return out


def _centre(i, base, S):
    """Query centre of variant i: a grid of pitch S over (wz, delta, a) so the variants' neighbourhoods do not overlap."""
    g = np.array([i % 4, (i // 4) % 4, i // 16], float)
    c = np.array(base, float)
    c[2:5] += S * g
    return _q32(c)


def _state(rng, q5, s=None):
    """xLin / uLin rows of a query: its features, small heading / lateral errors and a valid s."""
    x = np.array([q5[0], q5[1], q5[2], 0.05 * rng.standard_normal(), rng.uniform(0.3, 18.5) if s is None else s,
                  0.1 * rng.standard_normal()])
    return x, np.array(q5[3:5])


def _finish(name, rng, laps, qs, branch, N, s_list=None, **kw):
    xs, us = [], []
    for i in range(N):
        x, u = _state(rng, qs[i], None if s_list is None else s_list[i])
        xs.append(x); us.append(u)
    xs.append(xs[-1].copy())
    return Fixture(name, laps, np.array(xs), np.array(us), list(branch), **kw)


def _put_rows(rng, lap, feats, lanes="spread", lane=None):
    used = set()
    for f in feats:
        if lanes == "lane":
            t = lap.spot(lane=lane)
        else:
            t = lap.spot(avoid_lanes=used if len(used) < 32 else ())
        used.add(t % 32)
        lap.put(t, f, _target(rng, f))


# --- the cases of one query: rows around its centre q5 ---------------------------------------------------------------------
BASE = (1.0, 0.1, 0.0, 0.0, 0.0)


def case_near_ties(rng, lap, q5, consts, n=10):
    """n rows on a 1-norm sphere, distances D (1 + eps_i) with distinct eps_i ~ 1e-9: the k-th cut is inside fp32 resolution."""
    D = mid_bucket(0.75)
    eps = rng.permutation(np.linspace(-4e-9, 5e-9, n))
    _put_rows(rng, lap, _sphere(rng, q5, D * (1 + eps), consts["scaling"]))
    return "fast"


def case_exact_ties(rng, lap, q5, consts):
    """Five distinct nearer rows and 10 identical rows (a car at rest) with different next rows: the lowest 2 of them are used."""
    near = _sphere(rng, q5, [mid_bucket(v) for v in (0.3, 0.4, 0.5, 0.55, 0.6)], consts["scaling"])
    _put_rows(rng, lap, near)
    tie = _sphere(rng, q5, [mid_bucket(0.8)], consts["scaling"])[0]
    used = set()
    for _ in range(10):                           # next rows far apart: which 2 of the 10 are used shows in the model
        t = lap.spot(avoid_lanes=used)
        used.add(t % 32)
        lap.put(t, tie, _target(rng, tie) + 0.5 * rng.standard_normal(3))
    return "fast"


def case_lane_packing(rng, lap, q5, consts, m=4):
    """The m (4..7) nearest rows congruent mod 32: their lane's list of 3 overflows and the warp re-collects."""
    D = [mid_bucket(0.2 + 0.05 * j) for j in range(10)]
    rows = _sphere(rng, q5, D, consts["scaling"])
    lane = int(rng.integers(0, 32))
    _put_rows(rng, lap, rows[:m], lanes="lane", lane=lane)
    used = {lane}
    for f in rows[m:]:
        t = lap.spot(avoid_lanes=used)
        used.add(t % 32)
        lap.put(t, f, _target(rng, f))
    return "recollect"


def case_ties_many(rng, lap, q5, consts, n):
    """n rows within fp32 resolution of the k-th distance: more than 32 cannot all be re-scored (flag 32)."""
    D = mid_bucket(0.9)
    eps = rng.permutation(np.linspace(-3e-9, 3e-9, n))
    _put_rows(rng, lap, _sphere(rng, q5, D * (1 + eps), consts["scaling"]))
    return "overflow" if n > CAND else "fast"


def case_magnitude(rng, lap, q5, consts):
    """vx ~ 50: the fp32 rounding of the features (1.9e-7 in the distance) exceeds the 1e-9 differences at the k-th cut."""
    q = np.array(q5, float)
    q[0] = _q32(50.0 + 0.37)
    D = mid_bucket(0.6)
    eps = rng.permutation(np.linspace(-5e-9, 4e-9, 10))
    _put_rows(rng, lap, _sphere(rng, q, D * (1 + eps), consts["scaling"]))
    return "fast", q


def case_magnitude_margin(rng, lap, q5, consts):
    """vx ~ 50 and a ~ 40 with neighbours at D ~ 0.02: rounding the features to fp32 moves a distance by up to ~4e-6, a dozen key
    buckets at that D, so rows of the exact top 7 get keys well above G.  Only the (G + 2 qsum) 1.3e-6 term of the threshold
    keeps them candidates."""
    q = np.array(q5, float)
    q[0] = _q32(50.0 + 0.37)
    q[4] = _q32(40.0 + q5[4])
    eps = rng.permutation(np.linspace(-4e-9, 5e-9, 10))
    _put_rows(rng, lap, _sphere(rng, q, 0.02 * (1 + eps), consts["scaling"]))
    return "fast", q


def case_cluster(rng, lap, q5, consts, n=10, r=(0.2, 1.0)):
    """n rows at distinct distances in [r0, r1) (an ordinary neighbourhood)."""
    D = [mid_bucket(v) for v in np.sort(rng.uniform(r[0], r[1], n))]
    _put_rows(rng, lap, _sphere(rng, q5, D, consts["scaling"]))
    return "fast"


def case_affine(rng, lap, q5, consts, sigma, n=12):
    """Neighbours near the affine subspace vy = 0.7 wz - 0.2 (+ sigma noise): the Gram matrices are ill-conditioned."""
    P = _sphere(rng, q5, rng.uniform(0.2, 1.0, n), consts["scaling"])
    P[:, 1] = 0.7 * P[:, 2] - 0.2 + sigma * rng.standard_normal(n)
    _put_rows(rng, lap, P)
    q = np.array(q5, float)
    q[1] = _q32(0.7 * q[2] - 0.2)
    return None, q


# --- fixtures -------------------------------------------------------------------------------------------------------------
def _variants(name, seed, N, consts, T, cases, S=4.0, flags=0, raises=None, discriminate=True, nudge=True, s_list=None, note=""):
    """One instance, one lap: query i gets case cases[i % len(cases)] around its own centre."""
    rng = np.random.default_rng(seed)
    lap = _Lap(T, rng)
    qs, br = [], []
    for i in range(N):
        q5 = _centre(i, BASE, S)
        out = cases[i % len(cases)](rng, lap, q5, consts)
        b, q5 = (out if isinstance(out, tuple) else (out, q5))
        qs.append(q5); br.append(b)
    fx = _finish(name, rng, [lap.lap()], qs, br, N, s_list=s_list, flags=flags, raises=raises, discriminate=discriminate,
                 note=note)
    if nudge:
        _settle(fx, consts, rng)
    return fx


def _settle(fx, consts, rng, laps=None):
    """Move each query by a few fp32 buckets until every pre-filter decision is MARGIN away from flipping (ordinary data only)."""
    laps = laps or [l for l in fx.laps]
    for i in range(fx.uLin.shape[0]):
        for _ in range(200):
            q5 = np.concatenate([fx.xLin[i, 0:3], fx.uLin[i]])
            if all(min_margin(prefilter(x, u, q5, consts)) >= MARGIN for x, u in laps):
                break
            k = int(rng.integers(0, 5))
            if k < 3:
                fx.xLin[i, k] += rng.choice([-1, 1]) * 2.0 ** -14
            else:
                fx.uLin[i, k - 3] += rng.choice([-1, 1]) * 2.0 ** -14
        else:
            raise RuntimeError("%s: query %d could not be settled" % (fx.name, i))


def _bandwidth(name, seed, N, consts, at_h, n_well=5, **kw):
    """at_h: n_well rows well inside, one at computed distance nextafter(h, 0) (inside), one at exactly h (outside: vy offset
    0.25 + 5 - 0.25 == 5 exactly) and 3 at 1.5 h.  Otherwise 5 rows at h (1 - 1e-12) and 10 at h (1 + 1e-12).  The weight of a
    row is 0 at h, so only the flags see the rows at h; the rows at h (1 +- 1e-12) have weights of equal size and opposite sign."""
    rng = np.random.default_rng(seed)
    h = consts["h"]
    lap = _Lap(1200, rng)
    qs = []
    for i in range(N):
        q5 = _centre(i, (1.0, 0.25, 0.0, 0.0, 0.0), 24.0)
        qs.append(q5)
        if at_h:
            rows = list(_sphere(rng, q5, [mid_bucket(v) for v in (1.0, 1.8, 2.6, 3.4, 4.2)[:n_well]], consts["scaling"]))
            for off in (np.nextafter(h, 0.0), h):
                r = q5.copy(); r[1] = q5[1] + off
                assert np.linalg.norm((r - q5) * np.asarray(consts["scaling"]), 1) == off
                rows.append(r)
            rows += list(_sphere(rng, q5, [mid_bucket(1.5 * h * (1 + 0.1 * j)) for j in range(3)], consts["scaling"]))
        else:
            rows = list(_sphere(rng, q5, h * (1 - 1e-12) * np.ones(5), consts["scaling"]))
            rows += list(_sphere(rng, q5, h * (1 + 1e-12) * np.ones(10), consts["scaling"]))
        _put_rows(rng, lap, rows)
    return _finish(name, rng, [lap.lap()], qs, [None] * N, N, **kw)


def _few_inside(name, seed, N, consts, n_inside, T=1200, S=24.0):
    """n_inside rows inside the bandwidth, the others between 1.1 h and 1.4 h."""
    rng = np.random.default_rng(seed)
    h = consts["h"]
    lap = _Lap(T, rng)
    qs = []
    for i in range(N):
        q5 = _centre(i, BASE, S)
        qs.append(q5)
        D = [mid_bucket(v) for v in rng.uniform(0.2, 0.8, n_inside) * h] + \
            [mid_bucket(v) for v in rng.uniform(1.1, 1.4, 8) * h]
        _put_rows(rng, lap, _sphere(rng, q5, D, consts["scaling"]))
    return rng, lap, qs


def _lengths(seed, Tm1, consts, N=12):
    """A lap of T = Tm1 + 1 rows; the neighbourhood sits on the tile edges (256-row and 512-row tiles) and in the padded last
    batch; the last row (not a candidate, PM.py:183) is an exact copy of the first query."""
    rng = np.random.default_rng(seed)
    T = Tm1 + 1
    c = _q32(np.array([1.0, 0.1, 0.2, 0.05, 0.1]))
    if Tm1 <= 31:                                 # every row in the neighbourhood: a short smooth trajectory
        x = np.zeros((T, 6)); u = np.zeros((T, 2))
        P = c + rng.normal(0.0, 0.3, (T, 5)) * np.array([3.0, 1.0, 1.0, 1.0, 1.0]) / 5
        x[:, 0:3] = P[:, 0:3]; u[:] = P[:, 3:5]
        x[:, 4] = np.linspace(0.0, 1.0, T)
        qs = [_q32(c + rng.normal(0.0, 0.05, 5)) for _ in range(N)]
        fx = _finish("lengths_T-1=%d" % Tm1, rng, [(x, u)], qs, ["open" if Tm1 < 7 else None] * N, N,
                     discriminate=Tm1 >= 7)
    else:
        lap = _Lap(T, rng)
        spots = [t for e in range(256, Tm1 + 1, 256) for t in (e - 3, e - 1, e + 1) if t < Tm1 - 1]
        spots += [t for t in (Tm1 - 2, Tm1 - 4, Tm1 - 6) if t >= 0]
        spots = sorted(set(spots))
        rows = _sphere(rng, c, [mid_bucket(v) for v in rng.uniform(0.3, 1.2, len(spots) + 6)], consts["scaling"])
        for t, f in zip(spots, rows):
            if lap.free(t):
                lap.put(t, f, _target(rng, f))
        _put_rows(rng, lap, rows[len(spots):])
        x, u = lap.lap()
        qs = [_q32(c + rng.normal(0.0, 0.08, 5)) for _ in range(N)]
        x[T - 1, 0:3] = qs[0][0:3]; u[T - 1] = qs[0][3:5]       # the decoy
        fx = _finish("lengths_T-1=%d" % Tm1, rng, [(x, u)], qs, [None] * N, N, discriminate=True)
    _settle(fx, consts, rng)
    return fx


def _tmax4096(seed, consts, N=12):
    """One lap of 4096 rows: the neighbourhood among rows 4064..4094 (row counter j = 127), an exact-match decoy at row 4095."""
    rng = np.random.default_rng(seed)
    T = 4096
    lap = _Lap(T, rng)
    c = _q32(np.array([1.0, 0.1, 0.2, 0.05, 0.1]))
    rows = _sphere(rng, c, [mid_bucket(v) for v in rng.uniform(0.3, 1.2, 14)], consts["scaling"])
    for t, f in zip(range(4064, 4094, 2), rows):
        lap.put(t, f, _target(rng, f))
    x, u = lap.lap()
    qs = [_q32(c + rng.normal(0.0, 0.08, 5)) for _ in range(N)]
    for q in qs:
        assert np.linalg.norm(q - c, 1) < 1.0
    x[T - 1, 0:3] = qs[0][0:3]; u[T - 1] = qs[0][3:5]
    fx = _finish("tmax4096_j127", rng, [(x, u)], qs, [None] * N, N, discriminate=True)
    _settle(fx, consts, rng)
    return fx


def _multi_lap(name, seed, N, consts, lengths, special=None, **kw):
    """Laps added out of length order (equal-length ties included), each with its own rows around every query centre; `special`
    = (lap position in arrival order, n_inside) gives one lap only n_inside rows inside h."""
    rng = np.random.default_rng(seed)
    h = consts["h"]
    laps, qs = [], [_centre(i, BASE, 24.0 if special else 4.0) for i in range(N)]
    for li, T in enumerate(lengths):
        lap = _Lap(T, rng)
        for q5 in qs:
            if special and special[0] == li:
                D = [mid_bucket(v) for v in rng.uniform(0.2, 0.8, special[1]) * h] + \
                    [mid_bucket(v) for v in rng.uniform(1.1, 1.4, 6) * h]
            else:
                hi = 0.8 * h if special else min(1.0, 0.8 * h)
                D = [mid_bucket(v) for v in np.sort(rng.uniform(0.2 * hi, hi, 9))]
            _put_rows(rng, lap, _sphere(rng, q5, D, consts["scaling"]))
        laps.append(lap.lap())
    fx = _finish(name, rng, laps, qs, [None] * N, N, **kw)
    _settle(fx, consts, rng)
    return fx


def _curvature(name, seed, s_list, flags=0, raises=None):
    rng = np.random.default_rng(seed)
    N = len(s_list)
    fx = _variants(name, seed, N, DEFAULT, 800, [case_cluster], flags=flags, raises=raises, discriminate=False,
                   s_list=s_list, nudge=True)
    return fx


def _conditioning(seed, kappa, consts, N=12):
    """Neighbours near vy = 0.7 wz - 0.2 with the noise sigma calibrated so that kappa_2 of the Gram matrices ~ kappa."""
    def build(sigma):
        rng = np.random.default_rng(seed)
        lap = _Lap(800, rng)
        c = _q32(np.array([1.0, 0.7 * 0.3 - 0.2, 0.3, 0.05, 0.1]))
        P = _sphere(rng, c, rng.uniform(0.1, 1.0, 30), consts["scaling"])
        P[:, 1] = 0.7 * P[:, 2] - 0.2 + sigma * rng.standard_normal(30)
        _put_rows(rng, lap, P)
        qs = []
        for _ in range(N):                            # one neighbourhood, N queries inside it
            q = _q32(c + rng.normal(0.0, 0.1, 5))
            q[1] = _q32(0.7 * q[2] - 0.2)
            qs.append(q)
        fx = _finish("conditioning_k%.0e" % kappa, rng, [lap.lap()], qs, [None] * N, N)
        _settle(fx, consts, rng)
        return fx

    sigma = 1e-1
    for _ in range(8):
        fx = build(sigma)
        g = Group("", N, 1, consts, 0, 0)
        m = exact_model(fx, g, exact=False)
        ks = []
        for i in range(N):
            q = query(fx, i)
            idxs, Ks = zip(*[m.knn(q, lap) for lap in m.usedIt])
            ks.append(max(np.linalg.cond(m._normal_eq(f, idxs, Ks)[0]) for f in (ltv_model.IN_FEATS_VX, ltv_model.IN_FEATS_LAT)))
        k = float(np.median(ks))
        if abs(np.log10(k / kappa)) < 0.25:
            break
        sigma = min(sigma * np.sqrt(k / kappa), 1.0)     # beyond 1 the rows leave the bandwidth
    fx.note = "median kappa_2 %.1e (sigma %.1e)" % (k, sigma)
    fx.kappa = kappa
    return fx


def _zero_steer(name, seed, consts, N=12, **kw):
    """Every neighbour has steering delta = 0 exactly: the lateral Gram matrices have a zero row and column."""
    def case(rng, lap, q5, c):
        q = np.array(q5, float); q[3] = 0.0
        P = _sphere(rng, q, [mid_bucket(v) for v in np.sort(rng.uniform(0.2, 1.0, 10))], c["scaling"])
        P[:, 3] = 0.0
        _put_rows(rng, lap, P)
        return None, q
    return _variants(name, seed, N, consts, 800, [case], discriminate=False, nudge=True, **kw)


def _horizon_cases():
    return [case_near_ties, lambda r, l, q, c: case_lane_packing(r, l, q, c, 5), case_magnitude, case_exact_ties, case_cluster]


@lru_cache(maxsize=None)
def groups():
    D = DEFAULT
    G = []
    # ---- N = 12, one lap, the reference's constants
    a = Group("default_N12", 12, 1, D, 2048, 2)
    a.fixtures += [
        _variants("near_ties", 1, 12, D, 600, [case_near_ties]),
        _variants("exact_ties", 2, 12, D, 800, [case_exact_ties]),
        _variants("lane_packing", 3, 12, D, 900, [lambda r, l, q, c, m=m: case_lane_packing(r, l, q, c, m) for m in (4, 5, 6, 7)]),
        _variants("candidates_40", 4, 12, D, 1500, [lambda r, l, q, c: case_ties_many(r, l, q, c, 40)], flags=32, discriminate=False),
        _variants("candidates_30", 5, 12, D, 1200, [lambda r, l, q, c: case_ties_many(r, l, q, c, 30)]),
        _variants("magnitude_vx50", 6, 12, D, 600, [case_magnitude]),
        _variants("magnitude_margin", 12, 12, D, 600, [case_magnitude_margin], discriminate=False,
                  note="kappa_2 ~ 1e12: the features sit at 40..50 with a spread of 0.02"),
        _bandwidth("bandwidth_at_h", 7, 12, D, True, note="6 points inside h per query"),
        _bandwidth("bandwidth_1e-12", 10, 12, D, False, discriminate=True, note="5 points inside h per query"),
        _bandwidth("one_inside_at_h", 11, 12, D, True, n_well=0, flags=5, raises=IndexError,
                   note="nextafter(h, 0) inside, h outside: one neighbour"),
    ]
    rng, lap, qs = _few_inside("none_inside_h", 8, 12, D, 0)
    a.fixtures.append(_finish("none_inside_h", rng, [lap.lap()], qs, [None] * 12, 12, flags=1, raises=np.linalg.LinAlgError))
    a.fixtures.append(_zero_steer("zero_steering", 9, D, flags=1, raises=np.linalg.LinAlgError))
    a.fixtures += [_lengths(100 + Tm1, Tm1, D) for Tm1 in (5, 31, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025)]
    a.fixtures += [_conditioning(20 + j, kap, D) for j, kap in enumerate((1e3, 1e6, 1e10, 1e12))]
    starts = list(SEG_STARTS)
    below = [float(np.nextafter(s, -np.inf)) for s in starts[1:]]
    a.fixtures += [
        _curvature("curvature_starts", 30, starts + below[:5]),
        _curvature("curvature_wraps", 31, below[5:] + [float(np.nextafter(TL, 0.0))] + [TL + s for s in starts[1:6]] +
                   [3 * TL + s for s in starts[1:6]]),
        _curvature("curvature_at_TrackLength", 32, [TL] * 12, flags=2, raises=ValueError),
        _curvature("curvature_negative", 33, list(np.linspace(-8.0, -1e-9, 12)), flags=2, raises=ValueError),
        _curvature("curvature_beyond_64_laps", 34, [64 * TL * (1 + 1e-9), 100 * TL, 1e6] * 4, flags=2),
    ]
    G.append(a)
    # ---- one 4096-row lap: the last row counter
    G.append(Group("tmax4096", 12, 1, D, 4096, 2, [_tmax4096(40, D)]))
    # ---- several laps: added out of order, equal-length ties; trToUse in {1, 4, 8}
    lengths = [900, 600, 900, 750, 600, 1200, 750, 900, 450, 1050]
    for tr in (1, 4, 8):
        g = Group("laps_trToUse%d" % tr, 12, tr, D, 1280, len(lengths))
        g.fixtures += [_multi_lap("laps_%d_seed%d" % (tr, s), 50 + 10 * tr + s, 12, D, lengths, discriminate=True) for s in range(2)]
        if tr == 4:
            g.fixtures.append(_multi_lap("one_inside_h_in_a_lap", 60, 12, D, lengths, special=(3, 1), flags=4, raises=IndexError))
            g.fixtures.append(_multi_lap("none_inside_h_in_one_lap", 61, 12, D, lengths, special=(3, 0)))
        G.append(g)
    # ---- model constants
    c1 = dict(D, MaxNumPoint=1, h=50.0, lamb=1e-6)
    rng, lap, qs = _few_inside("k1_one_inside_h", 75, 12, c1, 1, S=150.0)
    G.append(Group("k1_h50_ridge", 12, 1, c1, 2048, 2, [
        _variants("k1_h50_ridge", 70, 12, c1, 600, [case_cluster], nudge=True),
        _finish("k1_one_inside_h", rng, [lap.lap()], qs, [None] * 12, 12, flags=4, raises=IndexError,
                note="MaxNumPoint = 1, exactly one row inside h")]))
    c3 = dict(D, MaxNumPoint=3, h=0.5, lamb=0.0)
    G.append(Group("k3_h0.5", 12, 2, c3, 1024, 3, [_multi_lap("k3_h0.5", 71, 12, c3, [500, 400], discriminate=True)]))
    cz = dict(D, MaxNumPoint=7, h=50.0, lamb=1e-6, dt=0.05, scaling=(0.1, 1.0, 0.0, 1.0, 1.0))
    G.append(Group("k7_h50_ridge_dt0.05_zero_scaling", 12, 1, cz, 1024, 2, [
        _variants("zero_scaling_entry", 72, 12, cz, 600, [case_near_ties, case_cluster]),
        _zero_steer("zero_steering_ridge", 73, cz)]))
    cn = dict(D, scaling=(-0.1, 1.0, 1.0, 1.0, 1.0))
    G.append(Group("negative_scaling", 12, 1, cn, 1024, 2, [
        _variants("negative_scaling", 74, 12, cn, 600, [case_near_ties, case_cluster, case_lane_packing])]))
    # ---- horizons: 1..4 blocks of 12 warps, N = 14 is the reference's LMPC horizon
    for N in (4, 6, 12, 14, 24, 48):
        G.append(Group("horizon_N%d" % N, N, 1, D, 2048, 2, [_variants("horizon_N%d" % N, 80 + N, N, D, 1800, _horizon_cases())]))
    return G


def all_fixtures():
    return [(g, fx) for g in groups() for fx in g.fixtures]


# ------------------------------------------------------------------------------------------------------------ per-query checks
def query(fx, i):
    return np.concatenate([fx.xLin[i, 0:3], fx.uLin[i]])


def wrong_selections(m, k):
    """The nearest wrong selections of the regression m just evaluated: {lap position: rows} for
    (a) the k-th and (k+1)-th nearest swapped, (b) the highest-index rows of a tie at the cut instead of the lowest,
    (c) one row just outside h included when fewer than k are inside."""
    out = []
    for pos, lap in enumerate(m.usedIt):
        d = m.dists[lap]
        sel = list(m.last_indices[pos]) if np.ndim(m.last_indices[pos]) else [int(m.last_indices[pos])]
        order = np.argsort(d, kind="stable")
        inside = int(np.sum(d < m.h))
        if inside >= k:
            if inside > k:
                out.append({pos: list(order[:k - 1]) + [order[k]]})
            dk = d[order[k - 1]]
            tied = np.nonzero(d == dk)[0]
            if len(tied) > 1:
                n_in = int(np.sum(d[order[:k]] == dk))
                if n_in < len(tied):
                    out.append({pos: [r for r in order[:k] if d[r] != dk] + list(tied[-n_in:])})
        elif inside < len(d):
            out.append({pos: sel + [order[inside]]})
    return out


def discrimination(fx, group, i, tol):
    """min over the wrong selections of max |rows 0..2 (wrong) - rows 0..2 (true)| / tol (inf when none applies)."""
    m = exact_model(fx, group, exact=False)
    true = rows012(*m.model(fx.xLin[i], fx.uLin[i]))
    worst = np.inf
    for alt in wrong_selections(m, group.consts["MaxNumPoint"]):
        w = exact_model(fx, group, exact=False)
        w.override = alt
        try:
            r = rows012(*w.model(fx.xLin[i], fx.uLin[i]))
        except np.linalg.LinAlgError:
            continue
        worst = min(worst, float(np.max(np.abs(r - true))) / tol)
    return worst
